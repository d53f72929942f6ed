"""ALSD N-best lists on the GPU (rs_rnnt_alsd_nbest): NeMo's `final` rebuilt by replaying the engine's trace through the
oracle's step (oracle/alsd_restated.py::alsd_step) and ranked as NeMo ranks it, at several N, on the tiny model and at
production size; n_best = 1 and entry 0 byte-identical to rs_rnnt_alsd; the crafted joints; the edges; and the Python API
(transcribe_nbest_batch against transcribe_batch and align_batch)."""

import numpy as np
import pytest
import torch

import alsd_cases as AC
import alsd_nbest_cases as NC
from reazonspeech_b200.synth import synth_clip

pytestmark = pytest.mark.gpu

_WAVES = [(300, 2.0), (301, 3.3), (302, 0.9), (303, 2.6), (304, 1.4)]
_CASES = [(1, True, True), (2, True, True), (4, True, True), (4, False, True), (4, True, False), (4, False, False), (8, True, True),
          (8, False, True)]
_IDS = [f"beam{b}-{'input' if r else 'merged'}-{'norm' if s else 'raw'}" for b, r, s in _CASES]

@pytest.fixture(scope="module")
def alsd_engine(tiny_cfg, tiny_sd):
    from reazonspeech_b200.engine import Engine
    return Engine(tiny_cfg, tiny_sd, "cuda:0", alsd=True)

def _encode(eng, waves):
    L = max(len(w) for w in waves)
    x = torch.zeros(len(waves), L)
    for i, w in enumerate(waves):
        x[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    mel, mel_len = eng.log_mel(x.cuda(), lens.cuda())
    return eng.encode(mel, mel_len)

@pytest.fixture(scope="module")
def tiny_enc(alsd_engine):
    return _encode(alsd_engine, [np.pad(synth_clip(s, d), 8000) for s, d in _WAVES])

def _cpu(xs):
    return [a.cpu() for a in xs]

def _check_against_replay(eng, enc, enc_len, beam, returns_input, score_norm, blank, Ns):
    """rs_rnnt_alsd_nbest at every N of Ns equals NeMo's list rebuilt from the trace; n_best = 1 and entry 0 at every N are
    byte-identical to rs_rnnt_alsd.  -> the pool sizes."""
    kw = dict(beam=beam, score_norm=score_norm, recombine_returns_input=returns_input)
    tr = eng.alsd_trace(enc, enc_len, **kw)
    plain = _cpu(eng.alsd(enc, enc_len, **kw))
    lens = enc_len.cpu()
    pools = []
    for N in Ns:
        out = _cpu(eng.alsd_nbest(enc, enc_len, N, **kw))
        for b in range(enc.shape[0]):
            T = int(lens[b])
            pool, from_final = NC.final_from_trace(tr, b, T, beam, int(2.0 * T), score_norm, returns_input, blank)
            NC.check_entries(out, b, pool, from_final, score_norm, N)
            if N == Ns[0]:
                pools.append(len(pool))
        for a, o in zip(plain, out[:4]):                         # entry 0 is rs_rnnt_alsd's result, byte for byte
            assert torch.equal(o[:, 0], a), N
        if N == 1:
            for a, o in zip(plain, out[:4]):
                assert torch.equal(o.reshape(a.shape), a)
    return pools

@pytest.mark.parametrize("case", _CASES, ids=_IDS)
def test_nbest_equals_the_replayed_final_list(alsd_engine, tiny_enc, tiny_cfg, case):
    """On the tiny model's five clips, N = 1, 3, beam and 64 equal sorted(final or last beam)[:N] rebuilt from the trace:
    sequences, steps and token counts identical, scores within 1e-12 relative, count / pool / from_final exact."""
    beam, returns_input, score_norm = case
    enc, enc_len = tiny_enc
    pools = _check_against_replay(alsd_engine, enc, enc_len, beam, returns_input, score_norm, tiny_cfg.blank, sorted({1, 3, beam, 64}))
    print(f"{case}: pool sizes {pools}")
    assert beam == 1 or max(pools) > 3                          # N = 3 cuts at least one list (beam 1: one finishes per clip here)

def test_nbest_production_size():
    """One 4 s clip at the production size (619 M, V = 3000), beam 4: the same checks."""
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0", alsd=True)
    enc, enc_len = _encode(eng, [np.pad(synth_clip(61, 4.0), 8000)])
    pools = _check_against_replay(eng, enc, enc_len, 4, True, True, cfg.blank, [1, 3, 4, 64])
    print(f"production size: pool size {pools}")

@pytest.mark.parametrize("case", NC.crafted_cases(), ids=[c[0] for c in NC.crafted_cases()])
def test_nbest_crafted_cases(tiny_cfg, tiny_sd, case):
    """On the crafted constant-row joints the N-best equals the oracle's list (tokens, scores to 1e-5; the steps of exactly
    tied entries may differ with the last bit of the row), and exactly the list the oracle's step builds from the engine's
    own row; the fallback case has from_final = 0."""
    from reazonspeech_b200.engine import Engine
    name, Tn, beam, ratio, score_norm, bias = case
    sd = AC.crafted_sd(tiny_sd, tiny_cfg, bias)
    eng = Engine(tiny_cfg, sd, "cuda:0", alsd=True)
    u_max = int(ratio * Tn)
    pool, from_final = NC.constant_row_pool(sd, tiny_cfg, Tn, beam, u_max)
    want = NC.ranked(pool, score_norm)
    enc = torch.zeros(1, 32, tiny_cfg.d_model, device="cuda")
    lens = torch.tensor([Tn], dtype=torch.int32, device="cuda")
    kw = dict(beam=beam, u_max_ratio=ratio, score_norm=score_norm, U_cap=200)
    tr = eng.alsd_trace(enc, lens, max_steps=1, **kw)
    lp = tr["cand_logp"][0, 0, 0]
    own_pool, own_ff = NC.constant_row_pool(sd, tiny_cfg, Tn, beam, u_max, row=(float(lp[0]), [float(x) for x in lp[1:1 + beam]],
                                                                               [int(x) for x in tr["cand_tok"][0, 0, 0, :beam]]))
    for N in (4, 64):
        out = _cpu(eng.alsd_nbest(enc, lens, N, **kw))
        y, steps, n, score, count, pool_n, ff = out
        assert int(count[0]) == min(N, len(pool)) and int(pool_n[0]) == len(pool) and int(ff[0]) == int(from_final)
        for e, h in enumerate(want[:N]):
            k = int(n[0, e])
            assert y[0, e, : k + 1].tolist() == h.y and AC.close(float(score[0, e]), h.score, 1e-5), (name, e)
            AC.assert_valid_alignment(h.y[1:], steps[0, e, :k].tolist(), Tn)
        NC.check_entries(out, 0, own_pool, own_ff, score_norm, N)
    assert from_final == (not name.startswith("fallback"))

def _nbest_raw(eng, enc, enc_len, N, U, fill, beam=4):
    """rs_rnnt_alsd_nbest into buffers prefilled with ``fill``."""
    B, T, _ = enc.shape
    bufs = [torch.full(s, fill, dtype=torch.int32, device="cuda") for s in ((B, N, U + 1), (B, N, U), (B, N))]
    score = torch.full((B, N), float(fill), dtype=torch.float64, device="cuda")
    sizes = [torch.full((B,), fill, dtype=torch.int32, device="cuda") for _ in range(3)]
    rc = eng.lib.rs_rnnt_alsd_nbest(eng.h, enc.data_ptr(), enc_len.data_ptr(), B, T, beam, 2.0, 1, 1, N, bufs[0].data_ptr(), bufs[1].data_ptr(),
                                    bufs[2].data_ptr(), score.data_ptr(), *[s.data_ptr() for s in sizes], U, None)
    assert rc == 0, eng.lib.rs_last_error(eng.h)
    return _cpu(bufs + [score] + sizes)

def test_nbest_edges(alsd_engine, tiny_enc, tiny_cfg):
    """Utterances of 0, 1 and 2 frames beside a long one equal the lists replayed from the trace (the empty one: [blank],
    n 0, score 0, pool 1, from_final 0); buffers past count, and past each entry's tokens, keep what they held; U_cap below
    an entry's length keeps its first U_cap tokens and its full n."""
    enc, enc_len = tiny_enc
    long_i = int(enc_len.argmax())
    e = torch.stack([enc[long_i], enc[0], enc[1], enc[2]]).contiguous()
    lens = torch.tensor([int(enc_len[long_i]), 1, 2, 0], dtype=torch.int32, device="cuda")
    N, U = 6, e.shape[1] * 3 + 1
    out = _nbest_raw(alsd_engine, e, lens, N, U, -7)
    y, steps, n, score, count, pool, ff = out
    tr = alsd_engine.alsd_trace(e, lens, beam=4)
    for b in range(4):
        T = int(lens[b])
        fin, from_final = NC.final_from_trace(tr, b, T, 4, int(2.0 * T), True, True, tiny_cfg.blank)
        NC.check_entries(out, b, fin, from_final, True, N)
        c = int(count[b])
        for j in range(c):
            k = int(n[b, j])
            assert (y[b, j, k + 1:] == -7).all() and (steps[b, j, k:] == -7).all(), (b, j)
        assert (y[b, c:] == -7).all() and (steps[b, c:] == -7).all() and (n[b, c:] == -7).all() and (score[b, c:] == -7).all()
    assert int(count[3]) == 1 and int(pool[3]) == 1 and int(ff[3]) == 0
    assert y[3, 0, 0] == tiny_cfg.blank and int(n[3, 0]) == 0 and float(score[3, 0]) == 0.0
    # U_cap below the entries' lengths
    full = _cpu(alsd_engine.alsd_nbest(enc, enc_len, 4))
    cap = 2
    assert int(full[2].max()) > cap
    capped = _cpu(alsd_engine.alsd_nbest(enc, enc_len, 4, U_cap=cap))
    for i in (2, 3, 4, 5, 6):
        assert torch.equal(capped[i], full[i])
    assert torch.equal(capped[0], full[0][:, :, : cap + 1]) and torch.equal(capped[1], full[1][:, :, :cap])

def test_nbest_batch_invariance(alsd_engine, tiny_enc):
    """An utterance's list is identical alone (its own T_max) and at another position of the batch."""
    enc, enc_len = tiny_enc
    B, N, U = enc.shape[0], 8, 200
    shifted = [(j + 2) % B for j in range(B)]
    batched = [(perm, _cpu(alsd_engine.alsd_nbest(enc[perm].contiguous(), enc_len[perm].contiguous(), N, U_cap=U)))
               for perm in (list(range(B)), shifted)]
    for i in range(B):
        Tp = (int(enc_len[i]) + 7) // 8 * 8
        alone = _cpu(alsd_engine.alsd_nbest(enc[i : i + 1, :Tp].contiguous(), enc_len[i : i + 1].contiguous(), N, U_cap=U))
        for perm, out in batched:
            p = perm.index(i)
            for a, o in zip(alone, out):
                assert torch.equal(o[p], a[0]), (i, p)

def test_bad_arguments_are_rejected_before_any_launch(alsd_engine, tiny_enc):
    enc, enc_len = tiny_enc
    n0 = alsd_engine.launch_count
    for N in (0, 65):
        with pytest.raises(RuntimeError, match="n_best"):
            alsd_engine.alsd_nbest(enc, enc_len, N)
    assert alsd_engine.launch_count == n0

# ------------------------------------------------------------------------------------------------ Python API
@pytest.fixture(scope="module")
def alsd_model(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    return asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=3, decoding="alsd")

@pytest.fixture(scope="module")
def audios():
    from reazonspeech_b200.nemo import asr
    return [asr.audio_from_numpy(synth_clip(300 + i, s), 16000) for i, s in enumerate((2.0, 0.8, 3.3, 1.5, 2.4))]

def test_transcribe_nbest_batch_entry0_and_log_likelihood(alsd_model, audios):
    """Entry 0 equals transcribe_batch on the same model (text, subwords, segments); every candidate's log_likelihood is
    bit-identical to align_batch of the same audio and token ids; a plain transcribe_batch after the N-best call is
    byte-identical to one before it."""
    from reazonspeech_b200.nemo import asr
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    before = asr.transcribe_batch(alsd_model, audios, cfg)
    lists = asr.transcribe_nbest_batch(alsd_model, audios, 5, log_likelihood=True)
    after = asr.transcribe_batch(alsd_model, audios, cfg)
    flat_audio, flat_ids, flat_ll = [], [], []
    for a, ref, rs in zip(audios, before, lists):
        assert 1 <= len(rs) <= 5
        r0 = rs[0]
        assert r0.text == ref.text and r0.subwords == ref.subwords and r0.segments == ref.segments
        assert r0.hypothesis.y_sequence.tolist() == ref.hypothesis.y_sequence.tolist() and r0.hypothesis.score == ref.hypothesis.score
        keys = [r.hypothesis.score / len(r.hypothesis.y_sequence) for r in rs]
        assert keys == sorted(keys, reverse=True)
        for r in rs:
            flat_audio.append(a)
            flat_ids.append(r.hypothesis.y_sequence.tolist()[1:])
            flat_ll.append(r.hypothesis.log_likelihood)
    assert sum(len(rs) for rs in lists) > len(audios)
    aligned = asr.align_batch(alsd_model, flat_audio, flat_ids)
    assert [r.hypothesis.log_likelihood for r in aligned] == flat_ll
    for x, y in zip(before, after):
        assert x.text == y.text and x.subwords == y.subwords and x.segments == y.segments
        assert x.hypothesis.y_sequence.tolist() == y.hypothesis.y_sequence.tolist() and x.hypothesis.timestamp == y.hypothesis.timestamp
        assert x.hypothesis.score == y.hypothesis.score
    one = asr.transcribe_nbest(alsd_model, audios[2], 5)
    assert [r.text for r in one] == [r.text for r in lists[2]] and all(r.hypothesis.log_likelihood is None for r in one)

def test_merged_beam_score_is_at_most_the_log_likelihood(alsd_engine, tiny_enc):
    """Two independent kernels agree: in merged recombination mode no two beam entries share a sequence, so a finished
    candidate's beam score sums a subset of its sequence's lattice paths and lies at or below log P(tokens | audio)."""
    from reazonspeech_b200.alignment import pack_labels
    enc, enc_len = tiny_enc
    y, steps, n, score, count, pool, ff = _cpu(alsd_engine.alsd_nbest(enc, enc_len, 16, recombine_returns_input=False))
    rows, ids, scores = [], [], []
    for b in range(enc.shape[0]):
        assert int(ff[b]) == 1
        for e in range(int(count[b])):
            rows.append(b)
            ids.append(y[b, e, 1 : int(n[b, e]) + 1].tolist())
            scores.append(float(score[b, e]))
    labels, label_len = pack_labels(ids)
    sel = torch.tensor(rows, device="cuda")
    ll = alsd_engine.align(enc.index_select(0, sel).contiguous(), enc_len.index_select(0, sel).contiguous(),
                           torch.from_numpy(labels).cuda(), torch.from_numpy(label_len).cuda())[3].cpu()
    worst = max(s - float(l) for s, l in zip(scores, ll))
    print(f"{len(scores)} candidates, max(beam score - log-likelihood) = {worst:.3e}")
    assert worst <= 1e-2

def test_nbest_rejects_greedy_models_and_bad_n_best(alsd_model, audios, tiny_cfg):
    """A greedy model and an n_best outside 1..64 are rejected before any launch."""
    from reazonspeech_b200.nemo import asr
    greedy = asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0)
    for model, N in ((greedy, 4), (alsd_model, 0), (alsd_model, 65)):
        n0 = model.engine.launch_count
        with pytest.raises(ValueError):
            asr.transcribe_nbest_batch(model, audios, N)
        assert model.engine.launch_count == n0
