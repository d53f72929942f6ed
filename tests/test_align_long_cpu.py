"""Long-form alignment on the CPU: the float64 banded oracle (tests/band_oracle.py) against forced alignment's oracle and brute
force, the band builder's properties (reazonspeech_b200/longform.py), the anchors, the widening loop on a stub, and the
argument checks that run before any GPU work."""
import numpy as np
import pytest

import align_oracle as A
import band_oracle as BO
from reazonspeech_b200 import longform as L


def _lattice(rng, T, U, integer=False):
    if integer:                                   # integer-valued: planted exact ties
        return -rng.integers(0, 3, (T, U + 1)).astype(np.float64), -rng.integers(0, 3, (T, U + 1)).astype(np.float64)
    return np.log(rng.uniform(0.05, 1.0, (T, U + 1))), np.log(rng.uniform(0.05, 1.0, (T, U + 1)))


def test_full_band_equals_forced_alignment():
    rng = np.random.default_rng(0)
    for T, U in ((1, 0), (1, 3), (5, 2), (7, 9), (12, 4)):
        for integer in (False, True):
            lpb, lpe = _lattice(rng, T, U, integer)
            r = A.align(lpb, lpe, T, U)
            q = BO.align(lpb, lpe, np.zeros(U + 1, int), np.full(U + 1, T), T, U)
            assert q["loglik"] == r["loglik"] and q["viterbi"] == r["viterbi"]
            assert q["frames"].tolist() == r["frames"].tolist() and q["edge"] == 0


def test_every_valid_band_equals_brute_force():
    rng = np.random.default_rng(1)
    n = 0
    for T in range(1, 6):
        for U in range(0, 4):
            for integer in (False, True):
                lpb, lpe = _lattice(rng, T, U, integer)
                full = A.align(lpb, lpe, T, U)
                for lo, hi in BO.valid_bands(T, U):
                    q = BO.align(lpb, lpe, lo, hi, T, U)
                    ll, best, frames = BO.brute_force(lpb, lpe, lo, hi, T, U)
                    assert abs(q["loglik"] - ll) <= 1e-12 * max(1.0, abs(ll)), (T, U, lo, hi)
                    assert q["viterbi"] == pytest.approx(best, abs=1e-12), (T, U, lo, hi)
                    assert q["frames"].tolist() == frames.tolist(), (T, U, lo, hi)
                    assert q["edge"] == BO.edge_count(frames.tolist(), lo, hi, T)
                    assert q["viterbi"] <= full["viterbi"] + 1e-12 and q["loglik"] <= full["loglik"] + 1e-12
                    L.check_band(lo, hi, T)
                    n += 1
    assert n > 1000


def test_band_containing_the_viterbi_path_keeps_it():
    rng = np.random.default_rng(2)
    for _ in range(30):
        T, U = int(rng.integers(5, 30)), int(rng.integers(1, 25))
        lpb, lpe = _lattice(rng, T, U)
        r = A.align(lpb, lpe, T, U)
        for k in (0, 1, 3):
            lo, hi = L.build_band(r["frames"], T, k)
            q = BO.align(lpb, lpe, lo, hi, T, U)
            assert q["frames"].tolist() == r["frames"].tolist() and q["viterbi"] == pytest.approx(r["viterbi"], abs=1e-9)


def _random_anchor(rng, U, T):
    a = np.sort(rng.integers(0, T, U))
    a[rng.random(U) < 0.3] = -1
    return a


def test_band_builder_properties():
    rng = np.random.default_rng(3)
    for _ in range(300):
        T, U, W = int(rng.integers(1, 200)), int(rng.integers(0, 60)), int(rng.integers(0, 20))
        a = _random_anchor(rng, U, T)
        lo, hi = L.build_band(a, T, W)
        L.check_band(lo, hi, T)
        assert lo.dtype == np.int32 and len(lo) == U + 1
        known = np.nonzero(a >= 0)[0]
        for k in known:                                   # token k joins rows k and k + 1: both hold anchor +- W
            for r in (k, k + 1):
                assert lo[r] <= max(a[k] - W, 0) and hi[r] >= min(a[k] + W + 1, T)
        for k in range(U):                                # an unmatched run spans its whole gap
            if a[k] >= 0:
                continue
            prev = [a[j] for j in known if j < k]
            nxt = [a[j] for j in known if j > k]
            f0 = prev[-1] if prev else 0
            f1 = nxt[0] if nxt else T - 1
            for r in (k, k + 1):
                assert lo[r] <= max(f0 - W, 0) and hi[r] >= min(f1 + W + 1, T)


def test_check_band_rejects_invalid_bands():
    good_lo, good_hi = np.array([0, 2, 4]), np.array([5, 6, 8])
    L.check_band(good_lo, good_hi, 8)
    for lo, hi in (([1, 2, 4], [5, 6, 8]), ([0, 2, 4], [5, 6, 7]), ([0, 2, 4], [5, 4, 8]), ([0, 5, 6], [5, 6, 8]),
                   ([0, 3, 2], [5, 6, 8]), ([0, 2, 8], [5, 6, 8]), ([0, -1, 4], [5, 6, 8])):
        with pytest.raises(ValueError):
            L.check_band(np.array(lo), np.array(hi), 8)


def test_anchors_are_the_matched_tokens():
    rng = np.random.default_rng(4)
    greedy = [int(x) for x in rng.integers(0, 50, 400)]
    frames = sorted(int(x) for x in rng.integers(0, 3000, 400))
    text, src = [], []                               # the greedy tokens with planted substitutions, deletions, insertions
    for j, k in enumerate(greedy):
        r = rng.random()
        if r < 0.05:
            text.append(1000 + j); src.append(-1)     # substitution by a token the greedy transcript lacks
        elif r < 0.10:
            continue                                  # deletion
        else:
            text.append(k); src.append(j)
        if rng.random() < 0.05:
            text.append(2000 + j); src.append(-1)     # insertion
    a = L.anchors(text, greedy, frames)
    for k, j in enumerate(src):
        assert a[k] == (frames[j] if j >= 0 else -1), k
    assert (L.anchors([1, 2, 3], [], []) == -1).all()


def test_widest_diagonal_and_extent_error():
    lo, hi = L.build_band([-1] * 20, 10, 2)           # nothing matched: every row spans every frame
    n, u0, u1 = L.widest_diagonal(lo, hi, 10)
    assert (n, u0, u1) == (10, 0, 9) or n == 10
    L.check_extent(lo, hi, 10)
    U = L.MAX_PITCH + 5
    lo, hi = np.zeros(U + 1, np.int32), np.full(U + 1, 2 * U, np.int32)
    with pytest.raises(ValueError, match="tokens 0\\.\\."):
        L.check_extent(lo, hi, 2 * U)


def test_widening_loop_on_a_stub():
    calls = []

    def stub(edges):
        def run(W):
            calls.append(W)
            return (None, None, None, None, edges[len(calls) - 1])
        return run

    calls.clear()
    res, W, n = L.align_widening(stub([0]), 50, 2)
    assert calls == [50] and (W, n) == (50, 1)
    calls.clear()
    res, W, n = L.align_widening(stub([3, 0]), 50, 2)
    assert calls == [50, 100] and (W, n) == (100, 2) and res[4] == 0
    calls.clear()
    res, W, n = L.align_widening(stub([3, 2, 1, 1]), 50, 2)
    assert calls == [50, 100, 200] and (W, n) == (200, 3) and res[4] == 1
    calls.clear()
    L.align_widening(stub([3]), 50, 0)
    assert calls == [50]


def test_arguments_rejected_before_gpu_work(tmp_path):
    for bad in (0, -1.0, float("nan"), float("inf"), "4", True):
        with pytest.raises(ValueError):
            L.band_frames(bad)
    assert L.band_frames(4.0) == 50
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError):
            L.check_widen(bad)

    class NoGpu:                                      # a model on several GPUs has no align_long_tokens
        cfg = None
    from reazonspeech_b200.nemo import asr
    with pytest.raises(ValueError, match="one GPU"):
        asr.align_long(NoGpu(), None, "x")


class _Tok:
    def sentence_to_ids(self, s):
        return [ord(c) % 7 for c in s]


class _Cfg:
    vocab_size = 7


class _Model:
    """align_long_tokens is present, so the checks under test are the ones before it is called."""
    cfg, tokenizer = _Cfg(), _Tok()

    def align_long_tokens(self, *a, **k):
        raise AssertionError("the GPU path was reached")


def test_bad_ids_and_counts_are_rejected():
    from reazonspeech_b200.nemo import asr
    m = _Model()
    with pytest.raises(ValueError, match="outside"):
        asr.align_long(m, None, [1, 7])
    with pytest.raises(ValueError, match="transcripts"):
        asr.align_long_batch(m, [None, None], ["a"])
    with pytest.raises(ValueError):
        asr.align_long(m, None, [1], band_seconds=-2)
    with pytest.raises(ValueError):
        asr.align_long(m, None, [1], max_widen=-1)


def test_cli_band_options(tmp_path):
    from reazonspeech_b200.nemo.asr import cli
    t = tmp_path / "t.txt"
    t.write_text("first line\n\n  second line \n", encoding="utf-8")
    with pytest.raises(ValueError, match="--text"):
        cli.parse(["--band=4", "a.wav"])
    with pytest.raises(ValueError, match="one AUDIO"):
        cli.parse([f"--text={t}", "--band=4", "a.wav", "b.wav"])
    with pytest.raises(ValueError):
        cli.parse([f"--text={t}", "--band=0", "a.wav"])
    opt = cli.parse([f"--text={t}", "--band=2.5", "a.wav"])
    assert opt.band == 2.5 and opt.text == str(t)
    assert cli.load_long_transcript(str(t)) == "first linesecond line"
    assert cli.parse([f"--text={t}", "a.wav"]).band is None


def test_row_oracle_equals_the_dense_one():
    rng = np.random.default_rng(5)
    for _ in range(40):
        T, U = int(rng.integers(1, 40)), int(rng.integers(0, 30))
        lpb, lpe = _lattice(rng, T, U)
        lo, hi = L.build_band(_random_anchor(rng, U, T), T, int(rng.integers(0, 6)))
        q = BO.align(lpb, lpe, lo, hi, T, U)
        r = BO.align_rows(BO.rows_of(lpb, lo, hi), BO.rows_of(lpe, lo, hi), lo, hi, T, U)
        assert r["viterbi"] == pytest.approx(q["viterbi"], abs=1e-9) and r["loglik"] == pytest.approx(q["loglik"], abs=1e-9)
        assert r["frames"].tolist() == q["frames"].tolist() and r["edge"] == q["edge"]
