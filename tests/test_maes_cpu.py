"""MAES beam search without a GPU: the oracle's pieces (prefix_search, select_k_expansions, the duplicate check, the LM terms) on
hand-built hypotheses and logits, MaesConfig, the checkpoint's maes_* keys, and the error paths of load_model and the CLI."""
import math

import pytest
import torch

from ngram_oracle import ArpaOracle, write_arpa
from oracle.maes_restated import MaesHyp, maes_beam, prefix_search, select_k_expansions, topk_stable
from reazonspeech_b200.config import MaesConfig, ModelConfig


def _hyp(y, score, dec_out=None):
    return MaesHyp(list(y), float(score), [-1] * len(y), None, dec_out or [torch.tensor([float(i)]) for i in range(len(y))])


def test_prefix_search_adds_the_prefix_paths_with_scores_before_the_frame():
    """Three hypotheses [b], [b, 3], [b, 3, 5]; logp depends on the dec_out value only, so every term is known by hand."""
    lp = {0.0: torch.log(torch.tensor([0.1, 0.2, 0.3, 0.25, 0.05, 0.1])), 1.0: torch.log(torch.tensor([0.3, 0.1, 0.1, 0.1, 0.1, 0.3]))}
    logp = lambda d: lp[float(d[0])]
    b = 9
    h0, h1, h2 = _hyp([b], -1.0), _hyp([b, 3], -2.0), _hyp([b, 3, 5], -3.0)
    hyps = prefix_search([h2, h1, h0], logp, prefix_alpha=2)
    la = lambda a, c: max(a, c) + math.log1p(math.exp(min(a, c) - max(a, c)))
    # h2 from h1: -2 + lp(dec_out_1[-1] = 1.0)[5]; from h0: -1 + lp(0.0)[3] + lp(h2.dec_out[1] = 1.0)[5]  (old scores throughout)
    want2 = la(la(-3.0, -2.0 + float(lp[1.0][5])), -1.0 + float(lp[0.0][3]) + float(lp[1.0][5]))
    want1 = la(-2.0, -1.0 + float(lp[0.0][3]))
    assert hyps[0].score == pytest.approx(want2, abs=1e-12) and hyps[1].score == pytest.approx(want1, abs=1e-12) and hyps[2].score == -1.0
    # prefix_alpha = 1: the two-token gap is out of reach
    h0, h1, h2 = _hyp([b], -1.0), _hyp([b, 3], -2.0), _hyp([b, 3, 5], -3.0)
    prefix_search([h2, h1, h0], logp, prefix_alpha=1)
    assert h2.score == pytest.approx(la(-3.0, -2.0 + float(lp[1.0][5])), abs=1e-12)
    # not a prefix, or equal: untouched
    h0, h1 = _hyp([b, 4], -1.0), _hyp([b, 3, 5], -3.0)
    prefix_search([h1, h0], logp, prefix_alpha=4)
    assert h1.score == -3.0


def test_select_k_expansions_gamma_order_and_fallback():
    h = _hyp([1], -1.0)
    out = select_k_expansions([h], [[4, 2, 7]], [[-0.1, -1.0, -3.0]], gamma=2.3)
    assert out == [[(2, -2.0), (4, -1.1)]]                        # within 2.3 of the best, ascending by score
    tie = select_k_expansions([h], [[4, 2]], [[-0.5, -0.5]], gamma=1.0)
    assert [k for k, _ in tie[0]] == [4, 2]                       # equal scores keep the candidates' order (stable)
    nan = select_k_expansions([h], [[4, 2]], [[float("nan"), float("nan")]], gamma=1.0)
    assert len(nan[0]) == 1 and nan[0][0][0] == 4                 # nothing passes: the best alone
    k, v = topk_stable(torch.tensor([0.5, 0.9, 0.9, 0.1]), 3)
    assert k == [1, 2, 0] and v[0] == pytest.approx(0.9)          # ties -> lower class index


def test_duplication_check_is_built_once_per_frame(tiny_cfg, tiny_sd):
    """An expansion whose sequence is a kept hypothesis is dropped; one equal to another expansion of the same frame is kept
    (and recombined): no search sequence ever holds the same token sequence twice in one kept list when the recombination
    merges, and a kept list can hold duplicates when it returns its input."""
    enc = torch.randn(12, tiny_cfg.d_model, generator=torch.Generator().manual_seed(4)) * 0.3
    merged = maes_beam(enc, tiny_sd, tiny_cfg, beam=4, recombine_returns_input=False)
    ys = [tuple(h.y) for h in merged.nbest]
    assert len(ys) == len(set(ys))
    for h in merged.nbest:
        assert h.y[0] == tiny_cfg.blank and all(0 <= f < 12 for f in h.timestamp[1:])
        assert h.timestamp[1:] == sorted(h.timestamp[1:])


def test_oracle_lm_terms_equal_the_arpa_oracle(tmp_path, tiny_cfg, tiny_sd):
    path = str(tmp_path / "t3.arpa")
    write_arpa(path, tiny_cfg.vocab_size, 3, n_sentences=200, seed=7)
    lm = ArpaOracle(path, tiny_cfg.vocab_size, 0.1)
    calls = []

    def fn(state, k):
        calls.append((state, k))
        return lm.score(state, k), lm.next(state, k)

    enc = torch.randn(10, tiny_cfg.d_model, generator=torch.Generator().manual_seed(2))
    plain = maes_beam(enc, tiny_sd, tiny_cfg, beam=2)
    fused = maes_beam(enc, tiny_sd, tiny_cfg, beam=2, lm=fn, lm_start=lm.start)
    assert calls and calls[0][0] == lm.start
    # the fused winner's score is its acoustic path plus the LM terms along its tokens: recompute the terms independently
    state, total = lm.start, 0.0
    for k in fused.tokens:
        total += lm.score(state, k)
        state = lm.next(state, k)
        assert lm.score(state, 0) == pytest.approx(0.1 * math.log(10) * lm.log10p(tuple(state), 0))
    assert total < 0.0 and fused.score != plain.score


def test_maes_config_validation_and_limits():
    assert MaesConfig().validate() == MaesConfig(2, 1, 2, 2.3)
    for bad in (dict(num_steps=1), dict(num_steps=5), dict(prefix_alpha=-1), dict(prefix_alpha=5), dict(expansion_beta=5),
                dict(expansion_gamma=0.0), dict(expansion_gamma=float("nan")), dict(num_steps=2.5)):
        with pytest.raises(ValueError):
            MaesConfig(**bad).validate()
    MaesConfig().check_beam(8, 3000)                                 # 8 * 10^2 = 800 rows
    with pytest.raises(ValueError, match="1024"):
        MaesConfig(num_steps=3).check_beam(8, 3000)
    with pytest.raises(ValueError, match="vocabulary"):
        MaesConfig(expansion_beta=4).check_beam(4, 6)
    with pytest.raises(ValueError, match="1..8"):
        MaesConfig().check_beam(9, 3000)


def test_checkpoint_maes_keys():
    block = {"beam_size": 4, "search_type": "maes", "maes_num_steps": 3, "maes_prefix_alpha": 2, "maes_expansion_beta": 1,
             "maes_expansion_gamma": 1.5}
    assert MaesConfig.from_beam_block(block) == MaesConfig(3, 2, 1, 1.5)
    assert MaesConfig.from_beam_block({"beam_size": 4, "maes_num_steps": 3}) == MaesConfig(num_steps=3)
    assert MaesConfig.from_beam_block({"beam_size": 4, "search_type": "alsd"}) is None
    assert ModelConfig().checkpoint_maes is None


def test_load_model_error_paths():
    from reazonspeech_b200.confidence import ConfidenceConfig
    from reazonspeech_b200.boosting import PhraseBoostingConfig
    from reazonspeech_b200.ngram_lm import NgramLMConfig
    from reazonspeech_b200.nemo import asr
    with pytest.raises(ValueError, match="decoding"):
        asr.load_model("cuda", synthetic=True, decoding="beam")
    with pytest.raises(ValueError, match="maes="):
        asr.load_model("cuda", synthetic=True, decoding="alsd", maes=MaesConfig())
    with pytest.raises(ValueError):
        asr.load_model("cuda", synthetic=True, decoding="maes", maes=MaesConfig(num_steps=1))
    with pytest.raises(ValueError, match="confidence"):
        asr.load_model("cuda", synthetic=True, decoding="maes", confidence=ConfidenceConfig())
    with pytest.raises(ValueError, match="boosting"):
        asr.load_model("cuda", synthetic=True, decoding="maes", boosting=PhraseBoostingConfig(["a"]))
    with pytest.raises(ValueError, match="ALSD"):
        asr.load_model("cuda", synthetic=True, decoding="alsd", lm=NgramLMConfig("x.arpa", 0.3))
    with pytest.raises(ValueError, match="1024"):
        asr.load_model("cuda", synthetic=True, decoding="maes", beam_size=8, maes=MaesConfig(num_steps=3))


def test_cli_options():
    from reazonspeech_b200.nemo.asr.cli import parse
    assert parse(["a.wav"]).decoding == "greedy" and parse(["a.wav"]).beam is None
    o = parse(["--decoding=maes", "--beam=6", "--lm=x.arpa", "--lm-alpha=0.3", "a.wav"])
    assert (o.decoding, o.beam, o.lm, o.lm_alpha) == ("maes", 6, "x.arpa", 0.3)
    assert parse(["--decoding=alsd", "a.wav"]).decoding == "alsd"
    for bad in (["--decoding=beam", "a.wav"], ["--beam=4", "a.wav"], ["--decoding=maes", "--beam=0", "a.wav"],
                ["--decoding=alsd", "--lm=x.arpa", "--lm-alpha=0.3", "a.wav"], ["--decoding=maes", "--phrases=p.txt", "a.wav"],
                ["--decoding=maes", "--stream", "a.wav"]):
        with pytest.raises(ValueError):
            parse(bad)
