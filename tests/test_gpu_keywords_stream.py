"""Streaming keyword spotting on the GPU (spot_stream.cu; keywords.py, "Streaming"): the lattice's independence of a frame's
place in its tile, rs_rnnt_spot_resume over chunked ranges against rs_rnnt_spot on the whole encoder output (E and S bit for
bit, the hits at an unbounded delay), the forced cuts against the CPU policy (tests/spot_stream_oracle.py) on the kernel's own
E, S and sigma, the transcriber against find_keywords at unlimited context, staggered streams batched against one at a time,
and the argument checks."""
import math
import random

import numpy as np
import pytest
import torch

import spot_oracle as K
import spot_stream_oracle as SS
from reazonspeech_b200.keywords import StreamKeywordsConfig
from reazonspeech_b200.streaming import StreamingConfig

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)


def _enc(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(lens), max(lens), cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc.cuda().contiguous(), torch.tensor(lens, dtype=torch.int32).cuda()


def _labels(kws):
    lab = torch.zeros(len(kws), max(len(x) for x in kws), dtype=torch.int32)
    for k, x in enumerate(kws):
        lab[k, : len(x)] = torch.tensor(x, dtype=torch.int32)
    return lab.cuda(), torch.tensor([len(x) for x in kws], dtype=torch.int32).cuda()


def _kws(cfg, lens, seed):
    rng = np.random.default_rng(seed)
    return [[int(k) for k in rng.integers(0, cfg.vocab_size, n)] for n in lens]


@pytest.fixture(scope="module")
def production():
    """The 619 M bench geometry (V = 3000, joint_hidden = 640), seeded weights."""
    from reazonspeech_b200.nemo.asr import load_model
    model = load_model("cuda:0", synthetic=True)
    return model.engine, model.cfg


@pytest.fixture(params=["tiny", "619M"])
def geometry(request, tiny_engine, tiny_cfg):
    """(engine, config, frames): the tiny model with short inputs, and the bench geometry, whose lattice spans many vocabulary
    tiles and whose gather copies several float4 rows per thread."""
    if request.param == "tiny":
        return tiny_engine, tiny_cfg, [40, 1, 23, 9, 64]
    eng, cfg = request.getfixturevalue("production")
    return eng, cfg, [120, 45, 1, 97]


def test_lattice_cell_does_not_depend_on_its_tile_position(geometry):
    eng, cfg, _ = geometry
    enc, lens = _enc(cfg, [45], 3)
    lab, ll = _labels(_kws(cfg, [3, 9], 4))
    whole = eng.spot_lattice(enc, lens, lab, ll)
    for a, b in ((3, 23), (7, 8), (1, 40), (17, 45)):
        part = eng.spot_lattice(enc[:, a:b].contiguous(), torch.tensor([b - a], dtype=torch.int32).cuda(), lab, ll)
        for k, U in enumerate(ll.tolist()):
            for w, p in zip(whole, part):
                assert torch.equal(w[k, a:b, :U + 1], p[k, :b - a, :U + 1]), (a, b, k)


def _ranges(rng, T, C):
    """Ranges covering [0, T) of at most C frames each, with empty and one-frame ranges."""
    out, t = [], 0
    while t < T:
        n = rng.choice([0, 1, C, rng.randint(0, C), rng.randint(1, C)])
        out.append((t, min(T, t + n)))
        t = min(T, t + n)
    return out


def _resume(eng, enc, lens, n_kw, C, seed):
    """Every row's ranges fed through rs_rnnt_spot_resume, rows joining at different calls, permuted slots, two records never
    used -> (E [B, n_kw, T], S, per (b, k): [(t, last, sigma, hits of that call)])."""
    B, T = enc.shape[0], enc.shape[1]
    rng = random.Random(seed)
    ranges = [_ranges(rng, int(lens[b]), C) for b in range(B)]
    start = [0 if b % 3 else rng.randint(0, 2) for b in range(B)]
    n_slots = B + 2
    slot_of = rng.sample(range(n_slots), B)
    rec = torch.zeros(n_slots, n_kw, eng.spot_state_bytes, dtype=torch.uint8, device="cuda")
    spare = [s for s in range(n_slots) if s not in slot_of]
    rec[spare] = torch.randint(0, 256, (len(spare), n_kw, eng.spot_state_bytes), dtype=torch.uint8, device="cuda")
    spare_before = rec[spare].clone()
    E = torch.full((B, n_kw, T), float("nan")); S = torch.full((B, n_kw, T), -1, dtype=torch.int32)
    log = {(b, k): [] for b in range(B) for k in range(n_kw)}
    for c in range(max(s + len(r) for s, r in zip(start, ranges))):
        rows = [b for b in range(B) if start[b] <= c < start[b] + len(ranges[b])]
        if not rows:
            continue
        rng.shuffle(rows)
        seg = [ranges[b][c - start[b]] for b in rows]
        last = [int(c - start[b] == len(ranges[b]) - 1) for b in rows]
        i32 = lambda v: torch.tensor(v, dtype=torch.int32)
        meta, val, fr, tl, e_, s_, sig = eng.spot_resume(enc[rows].contiguous(), i32([a for a, _ in seg]), i32([b for _, b in seg]),
                                                         i32([slot_of[b] for b in rows]), i32(last), rec, scores=True)
        e_, s_, sig = e_.cpu(), s_.cpu(), sig.cpu()
        assert [tuple(m[:2]) for m in meta] == sorted(tuple(m[:2]) for m in meta)
        for r, b in enumerate(rows):
            a0, a1 = seg[r]
            E[b, :, a0:a1], S[b, :, a0:a1] = e_[r, :, a0:a1], s_[r, :, a0:a1]
            for k in range(n_kw):
                sel = [i for i in range(len(meta)) if meta[i][0] == r and meta[i][1] == k]
                log[(b, k)].append((a1 - 1, last[r], int(sig[r, k]), [(meta[i], val[i], fr[i], tl[i]) for i in sel]))
    assert torch.equal(rec[spare], spare_before), "records outside the batch changed"
    return E, S, log


@pytest.mark.parametrize("U_lens", [[1, 3, 6], [32, 2]])
def test_resume_equals_offline_at_unbounded_delay(geometry, U_lens):
    eng, cfg, lens_ = geometry
    enc, lens = _enc(cfg, lens_, 11)
    kws = _kws(cfg, U_lens, 12)
    C = 20
    for thr in (-math.inf, -1.0):
        eng.set_spot_keywords(kws, thr, max(lens_), C)                  # D >= T: no cut is ever forced
        lab, ll = _labels(kws)
        span, score, conf, frames, token_lp, count, E0, S0 = [x.cpu() for x in eng.spot(enc, lens, lab, ll, thr, 256, scores=True)]
        E, S, log = _resume(eng, enc, lens, len(kws), C, seed=5)
        for b, T in enumerate(lens_):
            for k, U in enumerate(U_lens):
                p = b * len(kws) + k
                assert np.array_equal(E[b, k, :T].numpy().view(np.int32), E0[p, :T].numpy().view(np.int32)), (b, k)
                assert torch.equal(S[b, k, :T], S0[p, :T]), (b, k)
                n = int(count[p])
                assert n < 256
                want = sorted(range(n), key=lambda h: int(span[p, h, 1]))
                got = [h for *_, hs in log[(b, k)] for h in hs]
                assert len(got) == n, (b, k, thr)
                for (meta, val, fr, tl), h in zip(got, want):
                    assert tuple(meta[2:]) == (int(span[p, h, 0]), int(span[p, h, 1]), 0)
                    assert float(val[0]) == float(score[p, h]) and float(val[1]) == float(conf[p, h])
                    assert fr[:U].tolist() == frames[p, h, :U].tolist()
                    assert np.array_equal(tl[:U].view(np.int32), token_lp[p, h, :U].numpy().view(np.int32))
                    assert (fr[U:] == -1).all()


@pytest.mark.parametrize("D", [0, 2, 7])
def test_forced_cuts_follow_the_cpu_policy(tiny_engine, tiny_cfg, D):
    lens_ = [60, 33, 47]
    enc, lens = _enc(tiny_cfg, lens_, 21)
    kws = _kws(tiny_cfg, [2, 4, 8], 22)
    tiny_engine.set_spot_keywords(kws, -math.inf, D, 10)           # every frame a candidate: decisions are forced often
    E, S, log = _resume(tiny_engine, enc, lens, len(kws), 10, seed=D)
    n_forced = 0
    for (b, k), calls in log.items():
        Ek, Sk = E[b, k].numpy(), S[b, k].numpy()
        m = K.mean_lp(Ek, Sk)
        pending, barrier, t_prev = [], -1, -1
        for t, last, sigma, hits in calls:
            if t < 0 and t_prev < 0:
                assert sigma == -1 and not hits
                continue
            pending += [e for e in range(t_prev + 1, t + 1) if m[e] >= -np.inf]
            t_prev = max(t, t_prev)
            assert 0 <= sigma <= int(Sk[t_prev])                               # sigma <= start[t][U] = S(t)
            want, pending, barrier, _, _ = SS.decide(pending, Ek, Sk, sigma, t_prev, last, D, barrier)
            got = [(int(mt[2]), int(mt[3]), float(v[1]), bool(mt[4])) for mt, v, _, _ in hits]
            assert got == [(s, e, float(mm), f) for s, e, mm, f in want], (b, k, t)
            n_forced += sum(f for *_, f in got)
    assert n_forced > 0 or D > 2, "forced cuts are exercised"


def _stream(model, waves, config, kw, max_batch=None):
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    st = StreamingTranscriber(model, config, max_streams=len(waves), keywords=kw)
    ids = [st.open() for _ in waves]
    for sid, w in zip(ids, waves):
        st.feed(sid, w)
        st.close(sid)
    taken = {sid: [] for sid in ids}
    while not all(st.done(s) for s in ids):
        st.step()
        for sid, hs in st.take_hits().items():
            taken[sid] += hs
    return [st.result(s) for s in ids], [st.hits(s) if kw else None for s in ids], [taken[s] for s in ids]


def test_unlimited_context_equals_find_keywords(tiny_cfg):
    from reazonspeech_b200.nemo.asr import audio_from_numpy, find_keywords, load_model
    from reazonspeech_b200.synth import synth_clip
    model = load_model("cuda:0", synthetic=True, config=tiny_cfg, max_batch=3)
    waves = [synth_clip(60 + i, s).astype(np.float32) for i, s in enumerate((2.0, 3.3, 0.7, 5.1))]
    longest = max(len(w) for w in waves) / 16000 + 1.0
    ctx = 0.08 * int(longest / 0.08 + 1)
    config = StreamingConfig(1.6, ctx, ctx)
    kws = _kws(tiny_cfg, [1, 3, 5], 61)
    kw = StreamKeywordsConfig(kws, threshold=-math.inf, max_delay_seconds=0.08 * 200)
    plain, _, _ = _stream(model, waves, config, None)
    res, hits, taken = _stream(model, waves, config, kw)
    total = 0
    for i, w in enumerate(waves):
        assert res[i].text == plain[i].text and res[i].subwords == plain[i].subwords and res[i].segments == plain[i].segments
        want = find_keywords(model, audio_from_numpy(w, 16000), kws, threshold=-math.inf, max_hits=256)
        assert hits[i] == want, f"clip {i}"
        key = lambda h: (h.start_seconds, h.end_seconds, str(h.keyword), h.score)
        assert sorted(taken[i], key=key) == sorted(sum(want, []), key=key)
        total += sum(len(x) for x in want)
    assert total > 10


class _StepCheck:
    """Wraps the engine's stream_step_spot: every step's hits (and the records it leaves) must equal rs_rnnt_spot_resume's
    fed that step's buffer encoder output (the same staged batch through rs_logmel and rs_encode) from the records as they
    were before the step."""

    def __init__(self, eng):
        self.eng, self.real, self.steps, self.hits = eng, eng.stream_step_spot, 0, 0

    def __call__(self, wav, lens, dec_begin, dec_end, slot, states, U, out, last, records, alpha=None):
        eng, before = self.eng, records.clone()
        got = self.real(wav, lens, dec_begin, dec_end, slot, states, U, out, last, records, alpha=alpha)
        x = wav.to(torch.float32) * (1.0 / 32768.0) if wav.dtype == torch.int16 else wav
        enc, _ = eng.encode(*eng.log_mel(x.cuda().contiguous(), lens.to(torch.int32).cuda()))
        want = eng.spot_resume(enc, dec_begin, dec_end, slot, last, before)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2]), "hits: meta / frames"
        assert np.array_equal(got[1].view(np.int32), want[1].view(np.int32)) and np.array_equal(got[3].view(np.int32), want[3].view(np.int32))
        assert torch.equal(before, records), "records after the step"
        self.steps += 1
        self.hits += len(got[0])
        return got


@pytest.mark.parametrize("threshold,delay", [(-1.0, 10.0), (-math.inf, 0.8), (-math.inf, 0.0)])
def test_staggered_streams_batched_equal_one_at_a_time(tiny_cfg, threshold, delay):
    """Default StreamingConfig: seven staggered streams fed in irregular pieces over several max_batch calls equal the same
    schedule run one stream at a time, and every batched step's hits equal the device seam's on that step's buffer."""
    from reazonspeech_b200.nemo.asr import StreamingTranscriber, load_model
    from reazonspeech_b200.synth import synth_clip
    model = load_model("cuda:0", synthetic=True, config=tiny_cfg)
    rng = random.Random(3)
    sched = []
    for i in range(7):
        w = synth_clip(200 + i, rng.uniform(1.0, 12.0)).astype(np.float32)
        pieces, pos = [], 0
        while pos < len(w):
            n = rng.choice([5920, 3000, 12000, 20000]); pieces.append(w[pos:pos + n]); pos += n
        sched.append((rng.randint(0, 4), pieces))
    kw = StreamKeywordsConfig(_kws(tiny_cfg, [2, 4, 7], 201), threshold=threshold, max_delay_seconds=delay)

    def run(which, max_batch):
        model.max_batch = max_batch
        st = StreamingTranscriber(model, StreamingConfig(), max_streams=len(which), keywords=kw)
        sid, nxt, done, tick = {}, {i: 0 for i in which}, {}, 0
        while len(done) < len(which):
            for i in which:
                if tick == sched[i][0]:
                    sid[i] = st.open()
                if i in sid and nxt[i] < len(sched[i][1]):
                    st.feed(sid[i], sched[i][1][nxt[i]]); nxt[i] += 1
                    if nxt[i] == len(sched[i][1]):
                        st.close(sid[i])
            st.step()
            for i in [i for i, s in sid.items() if st.done(s)]:
                s = sid.pop(i)
                done[i] = (st.result(s).text, st.hits(s))
            tick += 1
            assert tick < 10000
        return done

    eng = model.engine
    check = _StepCheck(eng)
    eng.stream_step_spot = check
    try:
        batched = run(list(range(7)), 3)
    finally:
        del eng.stream_step_spot
    assert check.steps > 10
    n_hits = n_forced = 0
    for i in range(7):
        assert batched[i] == run([i], 1)[i], f"stream {i}"
        n_hits += sum(len(x) for x in batched[i][1]); n_forced += sum(h.forced for x in batched[i][1] for h in x)
    assert n_hits == check.hits
    if threshold == -math.inf:
        assert n_hits > 0
    if delay == 0.0:
        assert n_forced > 0, "with no delay every step whose frames hold a candidate forces a cut"
    print(f"threshold {threshold}, delay {delay} s: {n_hits} hits, {n_forced} forced")


def test_bad_arguments_are_rejected_before_any_launch(tiny_engine, tiny_cfg):
    eng = tiny_engine
    kws = _kws(tiny_cfg, [2, 3], 9)
    with pytest.raises(RuntimeError):
        eng.set_spot_keywords([[tiny_cfg.vocab_size]], -1.0, 10, 5)          # label outside the vocabulary
    with pytest.raises(RuntimeError):
        eng.set_spot_keywords([[1] * 33], -1.0, 10, 5)                      # U > 32
    with pytest.raises(RuntimeError):
        eng.set_spot_keywords(kws, -1.0, 20000, 5)                          # the ring does not fit
    with pytest.raises(RuntimeError):
        eng.set_spot_keywords(kws, float("nan"), 10, 5)
    eng.set_spot_keywords([], 0.0, 0, 1)
    assert eng.spot_state_bytes == 0
    enc, lens = _enc(tiny_cfg, [20, 20], 1)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32)
    rec = torch.zeros(3, 2, 4096, dtype=torch.uint8, device="cuda")
    z = i32(0, 0).cuda()
    out = [np.zeros((64, 8), np.int32) for _ in range(4)] + [np.zeros(1, np.int32)]
    rc = eng.lib.rs_rnnt_spot_resume(eng.h, enc.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), rec.data_ptr(), 3, 2, 20,
                                     64, *[a.ctypes.data for a in out], None, None, None, eng._stream())
    assert rc != 0 and "no keyword set" in eng.lib.rs_last_error(eng.h).decode()
    eng.set_spot_keywords(kws, -1.0, 10, 5)
    rec = torch.zeros(3, 2, eng.spot_state_bytes, dtype=torch.uint8, device="cuda")
    launches = eng.launch_count
    for db, de, sl in ((i32(0, 0), i32(5, 5), i32(1, 1)),                    # repeated slot
                       (i32(0, 0), i32(5, 5), i32(0, 3)),                     # slot outside the records
                       (i32(3, 0), i32(2, 5), i32(0, 1)),                     # dec_begin > dec_end
                       (i32(0, 0), i32(6, 5), i32(0, 1)),                     # more than C frames
                       (i32(0, 18), i32(5, 21), i32(0, 1))):                  # beyond T_max
        with pytest.raises(RuntimeError):
            eng.spot_resume(enc, db, de, sl, i32(0, 0), rec)
    assert eng.launch_count == launches and int(rec.sum()) == 0
    # the host step: bad slots, a range longer than the installed chunk, a small max_out, no installed set
    states = torch.zeros(4, eng.stream_state_bytes, dtype=torch.uint8, device="cuda")
    wav = torch.zeros(2, 32000)
    lens2 = i32(32000, 20000)
    out = (torch.zeros(2, 100, dtype=torch.int32), torch.zeros(2, 100, dtype=torch.int32), torch.zeros(2, dtype=torch.int32))
    for db, de, sl in ((i32(0, 0), i32(5, 5), i32(1, 1)), (i32(0, 0), i32(5, 5), i32(0, 3)), (i32(0, 0), i32(6, 5), i32(0, 1))):
        with pytest.raises(RuntimeError):
            eng.stream_step_spot(wav, lens2, db, de, sl, states, 100, out, i32(0, 0), rec)
    with pytest.raises(ValueError):                                           # records of another keyword count
        eng.stream_step_spot(wav, lens2, i32(0, 0), i32(5, 5), i32(0, 1), states, 100, out, i32(0, 0),
                             torch.zeros(3, 3, eng.spot_state_bytes, dtype=torch.uint8, device="cuda"))
    hits = [np.zeros((64, 8), np.int32) for _ in range(4)] + [np.zeros(1, np.int32)]
    args = [i32(0, 0), i32(5, 5), i32(0, 1), lens2, i32(0, 0)]
    ptrs = [a.data_ptr() for a in args]

    def raw(max_out):
        return eng.lib.rs_stream_step_spot(eng.h, wav.data_ptr(), 0, ptrs[3], ptrs[0], ptrs[1], ptrs[2], states.data_ptr(), 2, 32000,
                                           out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), 100, 0.0, None, ptrs[4],
                                           rec.data_ptr(), 3, max_out, *[a.ctypes.data for a in hits], eng._stream())
    assert raw(eng.lib.rs_spot_max_hits(eng.h, 2) - 1) != 0 and "max_out" in eng.lib.rs_last_error(eng.h).decode()
    eng.set_spot_keywords([], 0.0, 0, 1)
    assert raw(1 << 20) != 0 and "no keyword set" in eng.lib.rs_last_error(eng.h).decode()
    assert eng.launch_count == launches and int(rec.sum()) == 0 and int(states.sum()) == 0
