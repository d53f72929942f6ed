"""Streaming keyword spotting on the CPU (keywords.py, "Streaming"): the float64 streaming oracle (tests/spot_stream_oracle.py)
against the offline recursion and policy over every chunking of small random and integer-tied lattices, the frontier bound,
the forced cut's guarantees, the config's validation and record size, and the transcriber's calls without keywords."""
import itertools
import math

import numpy as np
import pytest

import spot_oracle as K
import spot_stream_oracle as SS
from reazonspeech_b200.keywords import KeywordHit, StreamKeywordsConfig, stream_record_bytes


def _lattice(rng, T, U, tied):
    if tied:
        return -rng.integers(0, 3, (T, U + 1)).astype(np.float64), -rng.integers(0, 3, (T, U + 1)).astype(np.float64)
    return np.log(rng.uniform(0.01, 1.0, (T, U + 1))), np.log(rng.uniform(0.01, 1.0, (T, U + 1)))


def _chunkings(T, rng, n):
    """Every composition of T for small T, else n random ones (with empty chunks)."""
    if T <= 6:
        for cuts in itertools.product([0, 1], repeat=T - 1):
            sizes, k = [], 1
            for c in cuts:
                if c:
                    sizes.append(k); k = 0
                k += 1
            yield sizes + [k]
        return
    for _ in range(n):
        cuts = sorted(rng.integers(0, T + 1, rng.integers(0, 6)).tolist())
        edges = [0] + cuts + [T]
        yield [b - a for a, b in zip(edges, edges[1:])]


CASES = [(T, U, tied, seed) for seed in range(4) for tied in (False, True) for T, U in ((1, 1), (5, 2), (6, 3), (17, 4), (40, 2), (40, 4))]


@pytest.mark.parametrize("T,U,tied,seed", CASES)
def test_frontier_bound_and_exact_scores(T, U, tied, seed):
    rng = np.random.default_rng(seed)
    lpb, lpe = _lattice(rng, T, U, tied)
    off = K.spot(lpb, lpe, T, U)
    for chunks in _chunkings(T, rng, 12):
        o = SS.stream(lpb, lpe, T, U, chunks, -np.inf, T)
        assert np.array_equal(o["E"], off["E"]) and np.array_equal(o["S"], off["S"]), chunks     # the carried column is exact
        ends = np.cumsum(chunks) - 1
        seen = [s for s, n in zip(o["sigma"], np.cumsum(chunks)) if n > 0]
        assert seen == sorted(seen), "sigma never decreases"
        for t, sig in zip(ends, o["sigma"]):
            if t >= 0:
                assert all(off["S"][e] >= sig for e in range(t + 1, T)), (chunks, t)


@pytest.mark.parametrize("T,U,tied,seed", CASES)
@pytest.mark.parametrize("thr", ["-inf", "-1", "median"])
def test_unbounded_delay_is_the_offline_policy(T, U, tied, seed, thr):
    rng = np.random.default_rng(seed + 100)
    lpb, lpe = _lattice(rng, T, U, tied)
    off = K.spot(lpb, lpe, T, U)
    m = K.mean_lp(off["E"], off["S"])
    threshold = {"-inf": -np.inf, "-1": -1.0, "median": float(np.median(m))}[thr]
    want = sorted(K.pick(off["E"], off["S"], T, threshold, 10 ** 6), key=lambda h: h[1])
    for chunks in _chunkings(T, rng, 8):
        o = SS.stream(lpb, lpe, T, U, chunks, threshold, T)
        got = sorted(o["hits"], key=lambda h: h[1])
        assert [(s, e, m) for s, e, m, *_ in got] == [(s, e, m) for s, e, m in want], chunks
        assert o["forced_cuts"] == 0 and not any(h[3] for h in got)
        for s, e, _, _, fr, tl in got:                                   # the forward traceback is the choice-byte backtrace
            bf, bl = K.backtrace(off["choice"], lpe, e, U)
            assert fr.tolist() == bf.tolist() and np.array_equal(tl, bl) and fr[0] == s


@pytest.mark.parametrize("T,U,tied,seed", [c for c in CASES if c[0] >= 17])
@pytest.mark.parametrize("D", [0, 1, 3, 8])
def test_bounded_delay(T, U, tied, seed, D):
    rng = np.random.default_rng(seed + 200)
    lpb, lpe = _lattice(rng, T, U, tied)
    off = K.spot(lpb, lpe, T, U)
    want = sorted(K.pick(off["E"], off["S"], T, -1.0, 10 ** 6), key=lambda h: h[1])
    for chunks in _chunkings(T, rng, 8):
        o = SS.stream(lpb, lpe, T, U, chunks, -1.0, D)
        hits = sorted(o["hits"], key=lambda h: h[1])
        for (s0, e0, *_), (s1, e1, *_) in zip(hits, hits[1:]):
            assert e0 < s1, "hits never overlap"
        for s, e, m, _, fr, tl in hits:                                   # each hit is a true segment path with its score
            assert fr[0] == s and np.isclose(sum(K.frame_lp(lpb, lpe, fr, e, U)), off["E"][e])
        for n, pend in zip(np.cumsum(chunks), o["pending_after"]):
            assert all(n - 1 - e < D for e in pend), "a candidate waits at most D frames"
        # forced exactly on the hits decided beyond their step's natural cut; without a forced cut, the offline list
        for (s, e, m, f, *_), i in zip(o["hits"], o["hit_step"]):
            assert f == (e >= o["natural"][i])
        if o["forced_cuts"] == 0:
            assert [(s, e) for s, e, *_ in hits] == [(s, e) for s, e, _ in want] and not any(h[3] for h in hits)


def test_small_delays_force_cuts():
    n_forced = 0
    for seed in range(30):
        lpb, lpe = _lattice(np.random.default_rng(seed), 30, 3, seed % 2 == 0)
        o = SS.stream(lpb, lpe, 30, 3, [3] * 10, -1.0, 2)
        n_forced += o["forced_cuts"]
        assert o["forced_cuts"] > 0 or not any(h[3] for h in o["hits"])
    assert n_forced > 0


def test_config_validation_and_record_size():
    c = StreamKeywordsConfig(["a"], max_delay_seconds=10.0)
    assert c.delay_frames() == 125 and c.threshold == -1.0
    assert StreamKeywordsConfig([[1, 2]], max_delay_seconds=0.0).delay_frames() == 0
    for bad in (dict(max_delay_seconds=0.1), dict(max_delay_seconds=-0.08), dict(threshold=math.nan), dict(threshold=math.inf),
                dict(threshold=True)):
        with pytest.raises(ValueError):
            StreamKeywordsConfig(["a"], **bad)
    with pytest.raises(ValueError):
        StreamKeywordsConfig([])
    assert stream_record_bytes(8, 125, 20) == 11664 and stream_record_bytes(32, 125, 20) == 47472
    assert stream_record_bytes(1, 0, 1) == 80 and all(stream_record_bytes(u, 5, 3) % 16 == 0 for u in range(1, 33))
    assert KeywordHit("a", 0.0, 1.0).forced is False and list(KeywordHit.__dataclass_fields__)[-1] == "forced"


def test_transcriber_without_keywords_makes_todays_calls(tiny_cfg):
    """A fixed schedule of three staggered streams on the stub engine: the (rows, slots) of every rs_stream_step call are the
    ones the transcriber made before keywords existed, and nothing else is called."""
    import test_streaming_cpu as TS
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    from reazonspeech_b200.streaming import StreamingConfig
    model = TS._model(tiny_cfg, 2)
    st = StreamingTranscriber(model, StreamingConfig(), max_streams=4)
    assert st.keywords is None and st.take_hits() == {}
    sig = [TS._signal(s) for s in (2.0, 3.1, 1.3)]
    pieces = [5920, 3000, 12000, 20000, 7000]
    sid, pos, tick = {}, [0, 0, 0], 0
    while len(sid) < 3 or not all(st.done(s) for s in sid.values()):
        for i in range(3):
            if tick == i and i not in sid:
                sid[i] = st.open()
            if i in sid and pos[i] < len(sig[i]):
                n = pieces[(tick + i) % len(pieces)]
                st.feed(sid[i], sig[i][pos[i]:pos[i] + n]); pos[i] += n
                if pos[i] >= len(sig[i]):
                    st.close(sid[i])
        st.step()
        tick += 1
    assert model.engine.calls == [(2, [0, 1]), (1, [0]), (1, [2]), (2, [1, 2]), (1, [1])]
    with pytest.raises(ValueError):
        st.hits(sid[0])
    with pytest.raises(ValueError):
        StreamingTranscriber(model, keywords=["a"])


@pytest.mark.parametrize("frames_cfg", [(20, 15, 15), (20, 0, 0), (1, 0, 0), (7, 3, 0), (3, 0, 1)])
def test_a_closed_stream_ends_with_a_step_that_decodes_its_last_frame(frames_cfg):
    """The transcriber marks a row ``last`` when it decodes frame F - 1 of a closed stream, and that is where everything
    pending is decided.  So a closed stream must never drain without such a step: before close() it has decoded at most
    rs_enc_valid(n) frames, and the 0.5 s of zeros that close() appends adds frames to F."""
    from reazonspeech_b200.streaming import PAD_SAMPLES, enc_valid, plan_row, stream_frames
    rng = np.random.default_rng(sum(frames_cfg))
    for _ in range(300):
        n, decoded, closed, rows = PAD_SAMPLES, 0, False, []
        total = int(rng.integers(0, 80000))
        while True:
            if not closed:
                add = int(rng.choice([0, 1, 159, 1280, 5920, 20000]))
                n += min(add, total)
                total -= min(add, total)
                if total == 0 and rng.random() < 0.5:
                    assert decoded <= enc_valid(n)
                    n += PAD_SAMPLES
                    closed = True
                    assert decoded < stream_frames(n, True)
            row = plan_row(n, decoded, closed, frames_cfg)
            if row is not None:
                decoded = row.dec_end + row.offset
                rows.append((closed, decoded))
            if closed and decoded >= stream_frames(n, True):
                break
        assert rows and rows[-1] == (True, stream_frames(n, True))
