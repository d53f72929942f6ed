"""n-gram LM shallow fusion in the greedy decode kernel (kLM) on the GPU: the kernel's lookup seam against the numpy emulation,
the decisions against the fused oracle (tests/ngram_oracle.py) fed the same encoder output, fusion with boosting and with
confidence, off means off, batch invariance, and the Python / CLI / C surfaces."""
import os

import numpy as np
import pytest
import torch

from boosting_oracle import follow_stats_emitted
from ngram_oracle import ArpaOracle, greedy_fused, write_arpa
from parity import decisions_from
from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables, lookup

pytestmark = pytest.mark.gpu

NEAR_TIE = 1e-3
# The seeded synthetic joints' logits lie close together and every LM term is negative while blank gets none, so a large
# alpha makes blank win everywhere.  At these weights the fused decodes still emit plenty of tokens.
ALPHA = 0.1


def _tiny_enc(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(lens), max(lens), cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc, torch.tensor(lens, dtype=torch.int32)


@pytest.fixture(scope="module")
def tiny_lm(tmp_path_factory, tiny_cfg):
    path = str(tmp_path_factory.mktemp("lm") / "tiny3.arpa")
    write_arpa(path, tiny_cfg.vocab_size, 3, n_sentences=200, seed=7)
    return path


def _greedy(eng, enc, lens, tables=None, U=None, alpha=None, boost=None):
    eng.set_ngram_lm(tables)
    if boost is not None:
        eng.set_phrase_boosting(boost.bonus, boost.next)
    try:
        return [a.cpu() for a in eng.greedy(enc.cuda().contiguous(), lens.cuda(), U, alpha=alpha)]
    finally:
        eng.set_ngram_lm(None)
        eng.set_phrase_boosting(None)


def _check_against_oracle(eng, cfg, sd, enc, lens, path, alpha, tag, boost=None, min_tok=0.2, min_deep=0.1, min_changed=0.1):
    """The engine's fused decisions vs the fused oracle teacher-forced along them: only a fused near-tie may differ (at most
    one per utterance).  The comparison must exercise the LM state: tokens are emitted (each moves the state through the
    kernel's LM ring), a share of the decisions is made in contexts of order >= 2 (tiles filled for states reached by
    emissions), and fusion changes a share of the unfused argmaxes."""
    tables = build_lm_tables(NgramLMConfig(path, alpha), cfg.vocab_size)
    lm = ArpaOracle(path, cfg.vocab_size, alpha)
    tk, fr, nt = _greedy(eng, enc, lens, tables, boost=boost)
    n_dec = n_changed = n_deep = 0
    for b in range(enc.shape[0]):
        n, T = int(nt[b]), int(lens[b])
        dec = decisions_from(tk[b, :n].tolist(), fr[b, :n].tolist(), T, cfg.max_symbols, cfg.blank)
        r = greedy_fused(enc[b, :T], sd, cfg, lm, None if boost is None else (boost.bonus, boost.next), follow=dec)
        assert r.complete, f"{tag} b={b}: the decision sequence does not cover the utterance's {T} frames"
        assert all(g[4] < NEAR_TIE for g in r.gaps) and len(r.gaps) <= 1, f"{tag} b={b}: {r.gaps[:4]}"
        n_dec += len(dec); n_changed += r.changed; n_deep += sum(o >= 2 for o in r.orders)
    n_tok = int(nt.sum())
    print(f"{tag}: {n_dec} decisions, {n_tok} tokens, {n_deep} decisions in contexts of order >= 2; fusion changed {n_changed} "
          f"({100.0 * n_changed / n_dec:.1f} %) of the unfused argmaxes")
    assert n_tok >= min_tok * n_dec, f"{tag}: only {n_tok} tokens in {n_dec} decisions"
    assert n_deep >= max(10, min_deep * n_dec), f"{tag}: only {n_deep} of {n_dec} decisions in contexts of order >= 2"
    assert n_changed >= min_changed * n_dec, f"{tag}: fusion changed only {n_changed} of {n_dec} decisions"


def test_seam_matches_numpy_lookup(tmp_path):
    """rs_ngram_lm_eval (the decode kernel's own lookup) == ngram_lm.lookup on 1e5 random pairs of a ~1 M n-gram 4-gram at V = 3000."""
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    path = str(tmp_path / "big.arpa")
    n = write_arpa(path, cfg.vocab_size, 4, 40000, seed=0)
    t = build_lm_tables(NgramLMConfig(path, 0.5), cfg.vocab_size)
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    eng.set_ngram_lm(t)
    rng = np.random.default_rng(1)
    N = 100000
    states = rng.integers(0, t.n_states, N)
    states[: N // 4] = rng.choice(np.flatnonzero(t.level == 3), N // 4)    # deep states: the longest chains
    tokens = rng.integers(0, cfg.vocab_size, N)
    score, nxt = eng.ngram_lm_eval(torch.from_numpy(states), torch.from_numpy(tokens))
    ref_s, ref_n = lookup(t, states, tokens)
    got_s = score.cpu().numpy()
    assert np.array_equal(nxt.cpu().numpy(), ref_n)
    ulp = np.abs(got_s.view(np.int32).astype(np.int64) - ref_s.view(np.int32).astype(np.int64))
    print(f"seam: {n} n-grams, {t.n_states} states; {int((ulp == 0).sum())} of {N} scores bit-identical, max {int(ulp.max())} ulp")
    assert ulp.max() <= 1
    eng.set_ngram_lm(None)


def test_tiny_against_fused_oracle(tiny_cfg, tiny_sd, tiny_engine, tiny_lm):
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13, 2, 31, 9], seed=21)
    _check_against_oracle(tiny_engine, tiny_cfg, tiny_sd, enc, lens, tiny_lm, ALPHA, "tiny")


def test_production_geometry_against_fused_oracle(tmp_path):
    """32 x 30 s clips of the bench in one batch, 619 M model, a 4-gram over its 3000 tokens: the decode alone, fed the encoder
    output the oracle decodes too.  alpha = 0.01: the fused decode still emits about half the unfused decode's tokens on
    these weights (at 0.1, under 3 per clip)."""
    from test_gpu_boosting import _full_model_encoder
    cfg, sd, eng, x, lens, enc, enc_len = _full_model_encoder()
    path = str(tmp_path / "lm4.arpa")
    write_arpa(path, cfg.vocab_size, 4, 3000, seed=3)
    _check_against_oracle(eng, cfg, sd, enc.cpu(), enc_len.cpu(), path, 0.01, "32 x 30 s", min_tok=0.05, min_deep=0.0, min_changed=0.05)


def test_fusion_with_boosting(tiny_cfg, tiny_sd, tiny_engine, tiny_lm):
    from reazonspeech_b200.boosting import PhraseBoostingConfig, build_tables
    rng = np.random.default_rng(5)
    phrases = [[int(v) for v in rng.integers(0, tiny_cfg.vocab_size, int(rng.integers(1, 4)))] for _ in range(12)]
    boost = build_tables(PhraseBoostingConfig(phrases, 0.5), tiny_cfg.vocab_size)
    enc, lens = _tiny_enc(tiny_cfg, [37, 6, 23, 40, 13, 31], seed=22)
    _check_against_oracle(tiny_engine, tiny_cfg, tiny_sd, enc, lens, tiny_lm, ALPHA, "tiny + boosting", boost=boost)


@pytest.mark.parametrize("alpha", (1.0, 0.33))
def test_confidence_with_fusion(tiny_cfg, tiny_sd, tiny_engine, tiny_lm, alpha):
    """Statistics of the unfused softmax at the fused decisions, within 1e-3 of float64 log_softmax; the decisions are those
    of the fused decode without statistics."""
    tables = build_lm_tables(NgramLMConfig(tiny_lm, ALPHA), tiny_cfg.vocab_size)
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13], seed=23)
    plain = _greedy(tiny_engine, enc, lens, tables)
    tk, fr, nt, st = _greedy(tiny_engine, enc, lens, tables, alpha=alpha)
    assert torch.equal(tk, plain[0]) and torch.equal(fr, plain[1]) and torch.equal(nt, plain[2])
    worst = 0.0
    for b in range(enc.shape[0]):
        n, T = int(nt[b]), int(lens[b])
        if n == 0:
            continue
        dec = decisions_from(tk[b, :n].tolist(), fr[b, :n].tolist(), T, tiny_cfg.max_symbols, tiny_cfg.blank)
        ref = torch.tensor(follow_stats_emitted(enc[b, :T], tiny_sd, tiny_cfg, dec, alpha), dtype=torch.float64)
        d = (st[b, :n].double() - ref).abs()
        worst = max(worst, float(d.max()))
        assert float(d.max()) <= 1e-3, f"b={b}: |delta| per column {d.max(0).values.tolist()}"
    assert int(nt.sum()) > 0
    print(f"confidence with fusion, alpha {alpha}: {int(nt.sum())} tokens, largest |delta stats| {worst:.3e}")


def test_off_means_off(tiny_cfg, tiny_engine, tiny_lm):
    tables = build_lm_tables(NgramLMConfig(tiny_lm, ALPHA), tiny_cfg.vocab_size)
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13, 2, 31, 9], seed=24)
    for alpha in (None, 0.33):
        never = _greedy(tiny_engine, enc, lens, alpha=alpha)
        on = _greedy(tiny_engine, enc, lens, tables, alpha=alpha)
        cleared = _greedy(tiny_engine, enc, lens, alpha=alpha)       # _greedy clears the table after each call
        assert all(torch.equal(a, b) for a, b in zip(never, cleared)), f"alpha={alpha}"
        assert not torch.equal(on[0], never[0])


def test_batch_invariance(tiny_cfg, tiny_engine, tiny_lm):
    """At a small alpha, so the utterance still emits tokens (the untrained joint's logits are close together, and every LM term
    is negative while blank gets none)."""
    tables = build_lm_tables(NgramLMConfig(tiny_lm, ALPHA), tiny_cfg.vocab_size)
    enc, lens = _tiny_enc(tiny_cfg, [29, 17, 40, 8], seed=25)
    first = _greedy(tiny_engine, torch.cat([enc[2:3], enc[:2], enc[3:]]), torch.cat([lens[2:3], lens[:2], lens[3:]]), tables)
    third = _greedy(tiny_engine, enc, lens, tables)
    alone = _greedy(tiny_engine, enc[2:3], lens[2:3], tables)
    n = int(alone[2][0])
    assert n > 0 and int(first[2][0]) == n and int(third[2][2]) == n
    for i in range(2):
        assert torch.equal(alone[i][0, :n], first[i][0, :n]) and torch.equal(alone[i][0, :n], third[i][2, :n])


def test_batch_beyond_one_state_per_thread(tiny_cfg, tiny_engine, tiny_lm):
    """300 utterances in one decode: the LM states of utterances 256.. are advanced by the kernel's second pass over the
    batch; they decode as they do alone."""
    tables = build_lm_tables(NgramLMConfig(tiny_lm, ALPHA), tiny_cfg.vocab_size)
    rng = np.random.default_rng(27)
    enc, lens = _tiny_enc(tiny_cfg, [int(n) for n in rng.integers(4, 20, 300)], seed=27)
    tk, fr, nt = _greedy(tiny_engine, enc, lens, tables)
    for b in (0, 255, 256, 270, 299):
        a = _greedy(tiny_engine, enc[b:b + 1], lens[b:b + 1], tables)
        n = int(a[2][0])
        assert int(nt[b]) == n and torch.equal(a[0][0, :n], tk[b, :n]) and torch.equal(a[1][0, :n], fr[b, :n]), b
    assert int(nt[256:].sum()) > 0


def test_python_api_and_cli(tiny_cfg, tiny_lm, tmp_path):
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    audios = [AudioData(synth_clip(90 + i, s).astype(np.float32), 16000) for i, s in enumerate((1.5, 3.0, 2.2, 0.7))]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    plain = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3)
    fused = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, lm=NgramLMConfig(tiny_lm, ALPHA))
    base = [r.hypothesis.y_sequence.tolist() for r in asr.transcribe_batch(plain, audios, cfg)]
    got = [r.hypothesis.y_sequence.tolist() for r in asr.transcribe_batch(fused, audios, cfg)]
    # the same decode through the engine directly, with the same tables
    plain.set_ngram_lm(NgramLMConfig(tiny_lm, ALPHA))
    assert [r.hypothesis.y_sequence.tolist() for r in asr.transcribe_batch(plain, audios, cfg)] == got
    assert got != base
    fused.set_ngram_lm(None)
    assert [r.hypothesis.y_sequence.tolist() for r in asr.transcribe_batch(fused, audios, cfg)] == base
    # CLI on a WAV with the full synthetic model
    import scipy.io.wavfile
    from reazonspeech_b200.nemo.asr.cli import main
    wav = tmp_path / "a.wav"
    scipy.io.wavfile.write(str(wav), 16000, (synth_clip(3, 2.0) * 20000).astype(np.int16))
    from reazonspeech_b200.config import ModelConfig
    big = str(tmp_path / "big.arpa")
    write_arpa(big, ModelConfig().vocab_size, 3, 500, seed=9)
    os.environ["REAZONSPEECH_B200_SYNTHETIC"] = "1"
    out = tmp_path / "out.txt"
    assert main(["--lm=" + big, "--lm-alpha=0.5", "-o", str(out), str(wav)]) is None
    assert out.exists()


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu_fusion(tiny_cfg, tiny_lm):
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    lm = NgramLMConfig(tiny_lm, ALPHA)
    one = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, lm=lm)
    two = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, devices=[0, 1], lm=lm)
    audios = [AudioData(synth_clip(80 + i, 1.0 + 0.4 * i).astype(np.float32), 16000) for i in range(6)]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    for a, b in zip(asr.transcribe_batch(one, audios, cfg), asr.transcribe_batch(two, audios, cfg)):
        assert a.hypothesis.y_sequence.tolist() == b.hypothesis.y_sequence.tolist()
    two.set_ngram_lm(None)
    one.set_ngram_lm(None)
    for a, b in zip(asr.transcribe_batch(one, audios, cfg), asr.transcribe_batch(two, audios, cfg)):
        assert a.hypothesis.y_sequence.tolist() == b.hypothesis.y_sequence.tolist()


def test_bad_arguments_rejected_before_any_launch(tiny_cfg, tiny_engine, tiny_lm):
    from reazonspeech_b200.engine import RsNgramLM
    import ctypes as C
    eng = tiny_engine
    t = build_lm_tables(NgramLMConfig(tiny_lm, ALPHA), tiny_cfg.vocab_size)
    eng.set_ngram_lm(t)                                             # the table that must stay set
    enc, lens = _tiny_enc(tiny_cfg, [12, 7], seed=26)
    ref = [a.cpu() for a in eng.greedy(enc.cuda(), lens.cuda())]
    buf = torch.zeros(4096, dtype=torch.int32, device="cuda")
    p = buf.data_ptr()
    good = dict(order=3, n_states=4, n_arcs=2, pitch=128, start_state=0)
    before = eng.launch_count
    bad = [dict(order=1), dict(order=7), dict(n_states=0), dict(n_arcs=-1), dict(start_state=4), dict(start_state=-1),
           dict(pitch=tiny_cfg.vocab_size - 1 - (tiny_cfg.vocab_size - 1) % 4), dict(pitch=130)]
    for change in bad + [dict(ptr=p + 4), dict(ptr=0)]:
        f = dict(good, **{k: v for k, v in change.items() if k != "ptr"})
        ptrs = [p] * 8
        if "ptr" in change:
            ptrs[3] = change["ptr"] or None
        lm = RsNgramLM(f["order"], f["n_states"], f["n_arcs"], f["pitch"], f["start_state"], *ptrs)
        assert eng.lib.rs_set_ngram_lm(eng.h, C.byref(lm)) == -1, change                   # RS_ERR_INVALID_ARG
        assert b"rs_set_ngram_lm" in eng.lib.rs_last_error(eng.h)
    assert eng.lib.rs_set_ngram_lm(None, None) == -1
    assert eng.launch_count == before
    again = [a.cpu() for a in eng.greedy(enc.cuda(), lens.cuda())]          # the previous table is still set
    assert all(torch.equal(a, b) for a, b in zip(ref, again))
    eng.set_ngram_lm(None)
    assert eng.lib.rs_ngram_lm_eval(eng.h, p, p, 1, p, p, None) == -1              # no table set
