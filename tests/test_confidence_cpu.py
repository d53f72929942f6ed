"""Confidence without a GPU: NeMo's measures from the four statistics against their direct evaluation on log-prob vectors,
the kernel's slice-wise reduction and merge restated in torch, the oracle's statistics, and the host layer."""
import math

import numpy as np
import pytest
import torch

from confidence_oracle import direct_measure, follow_stats, stats_of_logprobs
from reazonspeech_b200.confidence import ConfidenceConfig, ConfidenceMethodConfig, aggregate, measure, word_confidence, word_spans

METHODS = [("max_prob", "gibbs", "lin")] + [("entropy", t, n) for t in ("gibbs", "tsallis", "renyi") for n in ("lin", "exp")]


def _vectors(V):
    g = torch.Generator().manual_seed(V)
    random = torch.randn(V, generator=g, dtype=torch.float64) * 3
    peaked = torch.randn(V, generator=g, dtype=torch.float64)
    peaked[7] += 25
    flat = 1e-3 * torch.randn(V, generator=g, dtype=torch.float64)
    return {"random": random, "peaked": peaked, "flat": flat}


@pytest.mark.parametrize("V", [3001, 128])
@pytest.mark.parametrize("alpha", [1.0, 0.33])
def test_measures_from_statistics_equal_the_direct_measures(V, alpha):
    for kind, logits in _vectors(V).items():
        x = torch.log_softmax(logits, -1)
        st = np.array(stats_of_logprobs(x, alpha))
        for name, etype, norm in METHODS:
            m = ConfidenceMethodConfig(name=name, entropy_type=etype, alpha=alpha, entropy_norm=norm)
            got = float(measure(st, V, m))
            ref = direct_measure(x, name if name == "max_prob" else f"entropy_{etype}_{norm}", alpha)
            # relative 1e-6; measures of a nearly flat distribution sit at 0, where the bar is absolute (1e-9)
            assert got == pytest.approx(ref, rel=1e-6, abs=1e-9), (kind, name, etype, norm)
            assert -1e-9 <= got <= 1 + 1e-9, (kind, name, etype, norm, got)


def _soft(l: torch.Tensor, alpha: float):
    """(m, s, g, a, ga) of a float32 logit set, as one lane of the kernel forms them (an empty set: m = -inf)."""
    if l.numel() == 0:
        return (-math.inf, 0.0, 0.0, 0.0, 0.0)
    m = l.max()
    d = l - m
    e, ea = torch.exp(d), torch.exp(alpha * d)
    return (float(m), float(e.sum()), float((e * d).sum()), float(ea.sum()), float((ea * d).sum()))


def _merge(x, y, alpha):
    """decode_spec.cu soft_merge: the smaller-maximum side rescaled to the larger maximum, in float32."""
    if y[0] > x[0]:
        x, y = y, x
    if y[0] == -math.inf:
        return x
    f = np.float32
    d = f(y[0]) - f(x[0])
    r, ra = f(np.exp(d)), f(np.exp(f(alpha) * d))
    return (x[0], f(x[1]) + r * f(y[1]), f(x[2]) + r * (f(y[2]) + f(y[1]) * d),
            f(x[3]) + ra * f(y[3]), f(x[4]) + ra * (f(y[4]) + f(y[3]) * d))


def _final(c, alpha):
    """The consume step: a merged tuple relative to the argmax logit -> (lp, H1, A_alpha, G_alpha)."""
    m, s, g, a, ga = c
    log_s = math.log(s)
    s_ma = math.exp(-alpha * log_s)
    return [-log_s, g / s - log_s, s_ma * a, s_ma * ga - log_s * s_ma * a]


@pytest.mark.parametrize("NC", [3001, 128])
@pytest.mark.parametrize("alpha", [1.0, 0.33])
def test_slice_merge_equals_the_direct_statistics(NC, alpha):
    """Slices cut like rows_j = ceil(NC / S) with S = 33 (with 128 classes the last slice holds no row), each reduced, then
    merged in a shuffled order as the lanes / warps / slices of the kernel merge them."""
    S = 33
    rows_j = (NC + S - 1) // S
    g = torch.Generator().manual_seed(NC)
    for scale in (0.1, 3.0, 20.0):
        l = (scale * torch.randn(NC, generator=g)).float()
        parts = [_soft(l[min(NC, s * rows_j):min(NC, s * rows_j + rows_j)], alpha) for s in range(S)]
        if NC == 128:
            assert parts[-1][0] == -math.inf
        order = torch.randperm(S, generator=g).tolist()
        c = (-math.inf, 0.0, 0.0, 0.0, 0.0)
        for s in order:
            c = _merge(c, parts[s], alpha)
        assert c[0] == float(l.max())
        got = _final(c, alpha)
        ref = stats_of_logprobs(torch.log_softmax(l.double(), -1), alpha)
        assert got == pytest.approx(ref, rel=1e-5, abs=1e-6), (scale, got, ref)


def test_oracle_statistics_agree_with_log_softmax(tiny_cfg, tiny_sd):
    """Along the oracle's own decisions, follow_stats records one tuple per emitted token, and each tuple equals the statistics
    of scipy's log_softmax of the logits recomputed here."""
    from scipy.special import log_softmax
    from oracle import nemo_restated as O
    g = torch.Generator().manual_seed(7)
    enc = torch.randn(12, tiny_cfg.d_model, generator=g)
    res = O.rnnt_greedy(enc, tiny_sd, tiny_cfg)
    st = follow_stats(enc, tiny_sd, tiny_cfg, res.decisions, [1.0, 0.33], emulate=False)
    assert len(st[1.0]) == len(res.tokens) > 0 and len(st[0.33]) == len(res.tokens)
    for a in (1.0, 0.33):
        for row in st[a]:
            assert row[0] <= 0 and row[1] <= 0 and row[3] <= 0
    # recompute the first emission's logits by hand
    sd = tiny_sd
    hp = tiny_cfg.pred_hidden
    h, c = O.lstm_step(torch.zeros(hp), torch.zeros(hp), torch.zeros(hp), sd)
    pp = torch.nn.functional.linear(h, sd["joint.pred.weight"], sd["joint.pred.bias"])
    ep = O.joint_enc_proj(enc, sd)
    t0 = res.frames[0]
    logits = torch.nn.functional.linear(torch.relu(ep[t0] + pp), sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"])
    x = log_softmax(logits.double().numpy())
    p = np.exp(x)
    for a in (1.0, 0.33):
        pa = np.exp(a * x)
        assert st[a][0] == pytest.approx([x.max(), (p * x).sum(), pa.sum(), (pa * x).sum()], rel=1e-9, abs=1e-12)


def test_word_grouping_and_aggregation():
    assert word_spans(["▁a", "b", "▁c", "▁", "▁d", "e", "f"]) == [(0, 2), (2, 3), (4, 7)]
    assert word_spans(["x", "y", "▁z"]) == [(0, 2), (2, 3)]
    assert word_spans(["▁"]) == [] and word_spans([]) == []
    tc = [0.9, 0.5, 0.7, 0.1, 0.8, 0.6, 0.4]
    pieces = ["▁a", "b", "▁c", "▁", "▁d", "e", "f"]
    assert word_confidence(tc, pieces, "min") == [0.5, 0.7, 0.4]
    assert word_confidence(tc, pieces, "max") == [0.9, 0.7, 0.8]
    assert word_confidence(tc, pieces, "mean") == pytest.approx([0.7, 0.7, 0.6])
    assert word_confidence(tc, pieces, "prod") == pytest.approx([0.45, 0.7, 0.8 * 0.6 * 0.4])
    assert aggregate([0.2], "prod") == pytest.approx(0.2)


def test_config_validation():
    assert ConfidenceConfig().validate().alpha == pytest.approx(0.33)
    c = ConfidenceConfig()
    assert (c.exclude_blank, c.aggregation, c.method_cfg.name, c.method_cfg.entropy_type, c.method_cfg.entropy_norm) == (
        True, "min", "entropy", "tsallis", "exp")
    for bad in (ConfidenceConfig(exclude_blank=False), ConfidenceConfig(aggregation="median"),
                ConfidenceConfig(method_cfg=ConfidenceMethodConfig(name="lowest")),
                ConfidenceConfig(method_cfg=ConfidenceMethodConfig(entropy_type="shannon")),
                ConfidenceConfig(method_cfg=ConfidenceMethodConfig(entropy_norm="log")),
                ConfidenceConfig(method_cfg=ConfidenceMethodConfig(alpha=0.0)),
                ConfidenceConfig(method_cfg=ConfidenceMethodConfig(alpha=float("nan")))):
        with pytest.raises(ValueError):
            bad.validate()


def test_load_model_rejects_alsd_and_exclude_blank_false():
    from reazonspeech_b200.nemo import asr
    with pytest.raises(ValueError, match="greedy"):
        asr.load_model(synthetic=True, decoding="alsd", confidence=ConfidenceConfig())
    with pytest.raises(ValueError, match="exclude_blank"):
        asr.load_model(synthetic=True, confidence=ConfidenceConfig(exclude_blank=False))


def test_subword_as_dict_unchanged_without_confidence():
    from reazonspeech_b200.nemo.asr.interface import Subword
    assert Subword(0.5, 3, "a").as_dict() == {"seconds": 0.5, "token_id": 3, "token": "a"}
    assert Subword(0.5, 3, "a", 0.25).as_dict() == {"seconds": 0.5, "token_id": 3, "token": "a", "confidence": 0.25}


def test_greedy_hypothesis_and_subword_confidence(tiny_cfg):
    """The host half: statistics rows -> token confidence, word confidence, score = sum lp; subwords keep the confidence of
    their token after the empty (bare word-boundary) pieces are dropped."""
    from types import SimpleNamespace
    from reazonspeech_b200.nemo.asr.decode import decode_hypothesis
    from reazonspeech_b200.nemo.asr.transcribe import Hypothesis, greedy_hypothesis
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    tok = PieceTableTokenizer(synthetic_pieces(tiny_cfg.vocab_size))
    conf = ConfidenceConfig(aggregation="mean", method_cfg=ConfidenceMethodConfig(name="max_prob", alpha=1.0))
    model = SimpleNamespace(cfg=tiny_cfg, tokenizer=tok, confidence=conf)
    ids = [1, 10, 11, 1, 12, 2]                                   # id 1 is the bare word-boundary mark
    frames = [0, 1, 1, 3, 4, 6]
    x = torch.log_softmax(torch.randn(6, tiny_cfg.vocab_size + 1, generator=torch.Generator().manual_seed(3), dtype=torch.float64), -1)
    stats = np.array([stats_of_logprobs(r, 1.0) for r in x], np.float32)
    hyp = greedy_hypothesis(model, (ids, frames, stats))
    V = tiny_cfg.vocab_size + 1
    expect = [(V * math.exp(float(s[0])) - 1) / (V - 1) for s in stats]
    assert hyp.token_confidence == pytest.approx(expect, rel=1e-9)
    assert hyp.score == pytest.approx(float(stats[:, 0].astype(np.float64).sum()))
    assert hyp.word_confidence == pytest.approx(word_confidence(expect, tok.ids_to_pieces(ids), "mean"))
    r = decode_hypothesis(model, hyp)
    kept = [c for c, t in zip(expect, ids) if tok.ids_to_text([t])]
    assert [w.confidence for w in r.subwords] == pytest.approx(kept) and len(kept) < len(ids)
    plain = decode_hypothesis(model, Hypothesis.from_greedy(ids, frames, tiny_cfg.blank))
    assert all(w.confidence is None for w in plain.subwords)
    assert [w.as_dict() for w in plain.subwords] == [{k: v for k, v in w.as_dict().items() if k != "confidence"} for w in r.subwords]
    off = greedy_hypothesis(SimpleNamespace(cfg=tiny_cfg, tokenizer=tok, confidence=None), (ids, frames))
    assert off.score == 0.0 and off.token_confidence is None and off.word_confidence is None
