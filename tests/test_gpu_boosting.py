"""Phrase boosting in the greedy decode kernel (kBoost) on the GPU: an empty phrase list changes nothing, the decisions follow
the boosted oracle (tests/boosting_oracle.py) fed the same encoder output, forcing, batch invariance, confidence with boosting,
and the Python / C surfaces."""
import numpy as np
import pytest
import torch

from boosting_oracle import follow_stats_emitted, greedy_boosted
from parity import decisions_from
from reazonspeech_b200.boosting import PhraseBoostingConfig, build_tables

pytestmark = pytest.mark.gpu

NEAR_TIE = 1e-3


def _tiny_enc(cfg, lens, seed, T=None):
    g = torch.Generator().manual_seed(seed)
    T = T or max(lens)
    enc = torch.randn(len(lens), T, cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc, torch.tensor(lens, dtype=torch.int32)


def _random_phrases(V, n, seed, max_len=4):
    rng = np.random.default_rng(seed)
    return [[int(x) for x in rng.integers(0, V, int(rng.integers(1, max_len + 1)))] for _ in range(n)]


def _greedy(eng, enc, lens, tables=None, U=None, alpha=None):
    eng.set_phrase_boosting(None if tables is None else tables.bonus, None if tables is None else tables.next)
    try:
        return [a.cpu() for a in eng.greedy(enc.cuda().contiguous(), lens.cuda(), U, alpha=alpha)]
    finally:
        eng.set_phrase_boosting(None)


def _check_against_oracle(eng, cfg, sd, enc, lens, tables, tag):
    """The engine's boosted decisions vs the boosted oracle, teacher-forced along them: only a boosted near-tie may differ
    (at most one per utterance).  Returns (decisions, decisions whose boosted argmax differs from the plain one)."""
    tk, fr, nt = _greedy(eng, enc, lens, tables)
    n_dec = n_changed = 0
    for b in range(enc.shape[0]):
        n, T = int(nt[b]), int(lens[b])
        dec = decisions_from(tk[b, :n].tolist(), fr[b, :n].tolist(), T, cfg.max_symbols, cfg.blank)
        r = greedy_boosted(enc[b, :T], sd, cfg, tables.bonus, tables.next, follow=dec)
        assert r.complete, f"{tag} b={b}: the decision sequence does not cover the utterance's {T} frames"
        assert all(g[4] < NEAR_TIE for g in r.gaps) and len(r.gaps) <= 1, f"{tag} b={b}: {r.gaps[:4]}"
        n_dec += len(dec); n_changed += r.changed
    print(f"{tag}: {n_dec} decisions, boosting changed {n_changed} ({100.0 * n_changed / n_dec:.1f} %) of the oracle's argmaxes")
    assert n_changed >= 0.01 * n_dec, f"{tag}: boosting changed only {n_changed} of {n_dec} decisions"
    return n_dec, n_changed


def _full_model_encoder():
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    sd = random_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, "cuda:0")
    waves = [np.pad(synth_clip(i, 30.0), 8000) for i in range(32)]
    x = torch.from_numpy(np.stack(waves)).float().cuda()
    lens = torch.full((32,), len(waves[0]), dtype=torch.int32).cuda()
    enc, enc_len = eng.encode(*eng.log_mel(x, lens))
    return cfg, sd, eng, x, lens, enc, enc_len


@pytest.fixture(scope="module")
def full():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return _full_model_encoder()


def test_empty_list_is_unset_tiny(tiny_cfg, tiny_engine):
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13, 2, 31, 9], seed=11)
    empty = build_tables(PhraseBoostingConfig([], 2.0), tiny_cfg.vocab_size)
    for alpha in (None, 0.33):
        off = _greedy(tiny_engine, enc, lens, alpha=alpha)
        on = _greedy(tiny_engine, enc, lens, empty, alpha=alpha)
        assert all(torch.equal(a, b) for a, b in zip(off, on)), f"alpha={alpha}"


def test_empty_list_is_unset_bench_geometry(full):
    cfg, sd, eng, x, lens, enc, enc_len = full
    empty = build_tables(PhraseBoostingConfig([], 2.0), cfg.vocab_size)
    for alpha in (None, 0.33):
        off = [a.cpu() for a in eng.transcribe_device(x, lens, alpha=alpha)]
        eng.set_phrase_boosting(empty.bonus, empty.next)
        on = [a.cpu() for a in eng.transcribe_device(x, lens, alpha=alpha)]
        eng.set_phrase_boosting(None)
        assert all(torch.equal(a, b) for a, b in zip(off, on)), f"alpha={alpha}"
        assert int(off[2].sum()) > 0


def test_tiny_against_boosted_oracle(tiny_cfg, tiny_sd, tiny_engine):
    """Ragged lengths, windows past the end, 1-frame utterance; phrases over the tiny vocabulary at lambda 2."""
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13, 2, 31, 9], seed=12)
    tables = build_tables(PhraseBoostingConfig(_random_phrases(tiny_cfg.vocab_size, 12, seed=1), 2.0), tiny_cfg.vocab_size)
    _check_against_oracle(tiny_engine, tiny_cfg, tiny_sd, enc, lens, tables, "tiny")


def test_production_geometry_against_boosted_oracle(full):
    """32 x 30 s clips of the bench in one batch, 619 M model: the decode alone with 1000 phrases at lambda 2, fed the encoder
    output the oracle decodes too."""
    cfg, sd, eng, x, lens, enc, enc_len = full
    tables = build_tables(PhraseBoostingConfig(_random_phrases(cfg.vocab_size, 1000, seed=2), 2.0), cfg.vocab_size)
    _check_against_oracle(eng, cfg, sd, enc.cpu(), enc_len.cpu(), tables, "32 x 30 s")


def test_forcing_single_token_phrase(tiny_cfg, tiny_engine):
    """[k] at lambda 1e4: k, max_symbols times on every valid frame, also past a U_max below the token count."""
    k = 17
    tables = build_tables(PhraseBoostingConfig([[k]], 1e4), tiny_cfg.vocab_size)
    enc, lens = _tiny_enc(tiny_cfg, [11, 5, 16, 1], seed=13)
    tk, fr, nt = _greedy(tiny_engine, enc, lens, tables)
    ms = tiny_cfg.max_symbols
    assert nt.tolist() == [int(n) * ms for n in lens]
    for b, n in enumerate(lens.tolist()):
        assert tk[b, : n * ms].tolist() == [k] * (n * ms)
        assert fr[b, : n * ms].tolist() == [t for t in range(n) for _ in range(ms)]
    U = 7
    tk2, fr2, nt2 = _greedy(tiny_engine, enc, lens, tables, U=U)
    assert torch.equal(nt2, nt) and torch.equal(tk2, tk[:, :U]) and torch.equal(fr2, fr[:, :U])


def test_batch_invariance(tiny_cfg, tiny_engine):
    """One utterance alone, first in a batch and third in a batch decodes to the same boosted tokens."""
    tables = build_tables(PhraseBoostingConfig(_random_phrases(tiny_cfg.vocab_size, 12, seed=3), 2.0), tiny_cfg.vocab_size)
    enc, lens = _tiny_enc(tiny_cfg, [29, 17, 40, 8], seed=14)
    first = _greedy(tiny_engine, torch.cat([enc[2:3], enc[:2], enc[3:]]), torch.cat([lens[2:3], lens[:2], lens[3:]]), tables)
    third = _greedy(tiny_engine, enc, lens, tables)
    alone = _greedy(tiny_engine, enc[2:3], lens[2:3], tables)
    n = int(alone[2][0])
    assert n > 0 and int(first[2][0]) == n and int(third[2][2]) == n
    for i in range(2):
        assert torch.equal(alone[i][0, :n], first[i][0, :n]) and torch.equal(alone[i][0, :n], third[i][2, :n])


@pytest.mark.parametrize("alpha", (1.0, 0.33))
def test_confidence_with_boosting(tiny_cfg, tiny_sd, tiny_engine, alpha):
    """Statistics of the unboosted softmax at the boosted decisions, within 1e-3 of the oracle's float64 log_softmax; the
    decisions are those of the boosted decode without statistics."""
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13], seed=15)
    tables = build_tables(PhraseBoostingConfig(_random_phrases(tiny_cfg.vocab_size, 12, seed=4), 2.0), tiny_cfg.vocab_size)
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
    print(f"confidence with boosting, alpha {alpha}: largest |delta stats| {worst:.3e}")


def test_transcribe_batch_text_phrases_and_set_clear(tiny_cfg):
    """Text phrases through the synthetic tokenizer at load time; set_phrase_boosting replaced and cleared between calls."""
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    audios = [AudioData(synth_clip(90 + i, s).astype(np.float32), 16000) for i, s in enumerate((1.5, 3.0, 2.2, 0.7))]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    plain = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3)
    forced = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, boosting=PhraseBoostingConfig(["あ"], 1e4))
    base = asr.transcribe_batch(plain, audios, cfg)
    a_id = forced.tokenizer.text_to_ids("あ")[0]
    for r in asr.transcribe_batch(forced, audios, cfg):
        ids = r.hypothesis.y_sequence.tolist()[1:]
        assert len(ids) > 0 and set(ids) == {a_id} and r.text == "あ" * len(ids)
    forced.set_phrase_boosting(PhraseBoostingConfig(["い"], 1e4))
    i_id = forced.tokenizer.text_to_ids("い")[0]
    assert all(set(r.hypothesis.y_sequence.tolist()[1:]) == {i_id} for r in asr.transcribe_batch(forced, audios, cfg))
    forced.set_phrase_boosting(None)
    again = asr.transcribe_batch(forced, audios, cfg)
    assert [r.text for r in again] == [r.text for r in base]
    assert [r.hypothesis.y_sequence.tolist() for r in again] == [r.hypothesis.y_sequence.tolist() for r in base]
    # boosting together with confidence
    from reazonspeech_b200.confidence import ConfidenceConfig
    both = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, confidence=ConfidenceConfig(),
                          boosting=PhraseBoostingConfig(["あ"], 1e4))
    for r in asr.transcribe_batch(both, audios, cfg):
        assert set(r.hypothesis.y_sequence.tolist()[1:]) == {a_id}
        assert all(0.0 <= c <= 1.0 for c in r.hypothesis.token_confidence)


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu_boosting(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    boosting = PhraseBoostingConfig(_random_phrases(tiny_cfg.vocab_size, 12, seed=5), 2.0)
    one = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, boosting=boosting)
    two = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, devices=[0, 1], boosting=boosting)
    audios = [AudioData(synth_clip(80 + i, 1.0 + 0.4 * i).astype(np.float32), 16000) for i in range(6)]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    for a, b in zip(asr.transcribe_batch(one, audios, cfg), asr.transcribe_batch(two, audios, cfg)):
        assert a.hypothesis.y_sequence.tolist() == b.hypothesis.y_sequence.tolist()
    two.set_phrase_boosting(None)
    one.set_phrase_boosting(None)
    for a, b in zip(asr.transcribe_batch(one, audios, cfg), asr.transcribe_batch(two, audios, cfg)):
        assert a.hypothesis.y_sequence.tolist() == b.hypothesis.y_sequence.tolist()


def test_bad_arguments_rejected_before_any_launch(tiny_cfg, tiny_engine):
    eng = tiny_engine
    V = tiny_cfg.vocab_size
    bonus = torch.zeros(4, 136, dtype=torch.float32, device="cuda")
    nxt = torch.zeros(4, 136, dtype=torch.int32, device="cuda")
    before = eng.launch_count
    set_ = lambda b, n, s, p: eng.lib.rs_set_phrase_boosting(eng.h, b, n, s, p)
    for args in ((bonus.data_ptr(), nxt.data_ptr(), 8193, 128), (bonus.data_ptr(), nxt.data_ptr(), -1, 128),
                 (bonus.data_ptr(), nxt.data_ptr(), 4, V - 1 - (V - 1) % 4), (bonus.data_ptr(), nxt.data_ptr(), 4, 130),
                 (bonus.data_ptr() + 4, nxt.data_ptr(), 4, 128), (bonus.data_ptr(), nxt.data_ptr() + 8, 4, 128),
                 (None, nxt.data_ptr(), 4, 128), (bonus.data_ptr(), None, 4, 128)):
        assert set_(*args) == -1, args                                           # RS_ERR_INVALID_ARG
        assert b"rs_set_phrase_boosting" in eng.lib.rs_last_error(eng.h)
    assert eng.lib.rs_set_phrase_boosting(None, None, None, 0, 0) == -1
    assert set_(None, None, 0, 0) == 0                                            # clearing needs no table
    assert eng.launch_count == before
    with pytest.raises(ValueError):
        eng.set_phrase_boosting(np.zeros((2, 128), np.float32), np.zeros((3, 128), np.int32))
    with pytest.raises(RuntimeError, match="pitch"):
        eng.set_phrase_boosting(np.zeros((2, 126), np.float32), np.zeros((2, 126), np.int32))
    # a rejected table leaves the decode unboosted
    enc, lens = _tiny_enc(tiny_cfg, [12, 7], seed=16)
    base = [a.cpu() for a in eng.greedy(enc.cuda(), lens.cuda())]
    again = _greedy(eng, enc, lens)
    assert all(torch.equal(a, b) for a, b in zip(base, again))
