"""Caption alignment without a GPU: the float64 segment oracle (tests/segment_oracle.py) against brute-force enumeration with
planted ties, its inequalities, what the free start and the free end buy, the confidence formula, the window and seconds
arithmetic, the TSV round trip, the CLI options and the host plumbing of ``align_captions`` on a stub model."""
import io
import math

import numpy as np
import pytest

import align_oracle as A
import segment_oracle as S
from reazonspeech_b200.captions import (AlignedCaption, Caption, caption_window, confidence, frame_seconds, read_captions_tsv,
                                        segment_seconds, window_samples)

PLANTED_BAR = S.PLANTED_BAR       # overlap share the segment DP must reach on planted lattices, and the variants must not


def _int_lattice(rng, T, U):
    """Integer-valued log-probabilities from a small range: exact ties between paths are common and exact in float64."""
    return -rng.integers(0, 3, (T, U + 1)).astype(np.float64), -rng.integers(0, 3, (T, U + 1)).astype(np.float64)


@pytest.mark.parametrize("T", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("U", [1, 2, 3])
def test_oracle_equals_brute_force(T, U):
    rng = np.random.default_rng(100 * T + U)
    cases = [_int_lattice(rng, T, U) for _ in range(12)]
    cases += [(np.log(rng.uniform(0.05, 1.0, (T, U + 1))), np.log(rng.uniform(0.05, 1.0, (T, U + 1)))) for _ in range(3)]
    cases.append((np.zeros((T, U + 1)), np.zeros((T, U + 1))))      # every path ties
    for lpb, lpe in cases:
        r = S.segment_align(lpb, lpe, T, U)
        score, s, e, frames = S.brute_force(lpb, lpe, T, U)
        assert abs(r["score"] - score) < 1e-12
        assert (r["s"], r["e"], r["frames"].tolist()) == (s, e, frames.tolist())
        assert r["token_lp"].tolist() == [lpe[f, u] for u, f in enumerate(frames)]
        assert abs(S.path_score(lpb, lpe, tuple(frames), e, U) - r["score"]) < 1e-12


def test_loglik_frame_lp_and_the_inequalities():
    rng = np.random.default_rng(7)
    for T, U in [(1, 1), (3, 5), (12, 4), (30, 9), (40, 1)]:
        for _ in range(5):
            lpb, lpe = np.log(rng.uniform(0.02, 1.0, (T, U + 1))), np.log(rng.uniform(0.02, 1.0, (T, U + 1)))
            r = S.segment_align(lpb, lpe, T, U)
            s, e = r["s"], r["e"]
            assert 0 <= s <= e < T and r["frames"][0] == s and r["frames"][-1] <= e
            assert abs(r["loglik"] - A.align(lpb[s:e + 1], lpe[s:e + 1], e - s + 1, U)["loglik"]) < 1e-12
            fl = r["frame_lp"]
            assert np.isnan(fl[:s]).all() and np.isnan(fl[e + 1:]).all() and not np.isnan(fl[s:e + 1]).any()
            assert abs(fl[s:e + 1].sum() - r["score"]) < 1e-9
            full = A.align(lpb, lpe, T, U)["viterbi"]
            assert r["loglik"] >= r["score"] - 1e-12 and r["score"] >= full - 1e-12


def _planted(rng, T, U):
    """A window of T frames whose caption (U tokens) is said over frames [a, a + 2U): its tokens are likely there (one per
    two frames).  Elsewhere other speech is going on: blank and the caption's tokens are both unlikely."""
    a = int(rng.integers(0, T - 2 * U + 1))
    lpb = np.log(rng.uniform(0.02, 0.1, (T, U + 1)))
    lpe = np.log(rng.uniform(0.001, 0.05, (T, U + 1)))
    lpb[a:a + 2 * U] = np.log(rng.uniform(0.4, 0.9, (2 * U, U + 1)))
    for u in range(U):
        lpe[a + 2 * u, u] = np.log(rng.uniform(0.5, 0.95))
    return lpb, lpe, a, a + 2 * U


def _overlap_rate(free_start, free_end, n=200):
    rng = np.random.default_rng(11)
    hit = 0
    for _ in range(n):
        T, U = int(rng.integers(60, 120)), int(rng.integers(3, 12))
        lpb, lpe, a, b = _planted(rng, T, U)
        r = S.segment_align(lpb, lpe, T, U, free_start=free_start, free_end=free_end)
        s = r["s"] if free_start else 0
        e = r["e"]
        hit += int(s < b and e >= a and (e - s + 1) <= 2 * (b - a))         # overlaps, and is not the whole window
    return hit / n


def test_free_start_and_free_end_are_needed():
    segment = _overlap_rate(True, True)
    no_start = _overlap_rate(False, True)
    no_end = _overlap_rate(True, False)
    print(f"planted overlap: segment {segment:.2f}, no free start {no_start:.2f}, no free end {no_end:.2f}")
    assert segment >= PLANTED_BAR > max(no_start, no_end)


def test_confidence_matches_a_direct_loop():
    rng = np.random.default_rng(3)
    for n in (1, 5, 15, 16, 40, 97):
        x = rng.normal(-1.0, 1.0, n)
        for L in (1, 4, 15, 30):
            direct = float(np.mean(x)) if n <= L else min(sum(x[i:i + L]) / L for i in range(n - L + 1))
            assert abs(confidence(x, L) - direct) < 1e-12
    with pytest.raises(ValueError):
        confidence([1.0], 0)
    assert math.isnan(confidence([], 15))


def test_window_and_seconds_arithmetic():
    c = Caption(40.0, 43.5, "x")
    assert caption_window(c, 100.0) == (15.0, 43.5)
    assert caption_window(c, 100.0, before=5.0, after=2.0) == (35.0, 45.5)
    assert caption_window(Caption(10.0, 12.0, "x"), 100.0) == (0.0, 12.0)                # clamped at 0
    assert caption_window(Caption(90.0, 120.0, "x"), 100.0, after=5.0) == (65.0, 100.0)  # clamped at the end
    assert caption_window(Caption(130.0, 140.0, "x"), 100.0, before=5.0) is None          # outside the audio
    assert caption_window(Caption(3.0, 3.0, "x"), 100.0, before=0.0) is None              # empty
    with pytest.raises(ValueError):
        caption_window(Caption(5.0, 4.0, "x"), 100.0)
    assert window_samples(15.0, 43.5, 16000) == (240000, 696000)
    # frame f of a padded window lies 0.08 f - 0.5 s into it, clamped at 0
    assert frame_seconds(0) == 0.0 and frame_seconds(6) == 0.0 and abs(frame_seconds(20) - 1.1) < 1e-12
    s, e = segment_seconds(20, 44, 15.0, 43.5)
    assert abs(s - 16.1) < 1e-9 and abs(e - (15.0 + 0.08 * 45 - 0.5)) < 1e-9
    assert segment_seconds(0, 3, 15.0, 43.5) == (15.0, 15.0)                           # inside the leading pad
    s, e = segment_seconds(300, 370, 15.0, 43.5)                                       # the trailing pad: clamped
    assert e == 43.5 and s <= e


def test_tsv_round_trip(tmp_path):
    from reazonspeech_b200.nemo.asr.interface import Segment
    from reazonspeech_b200.nemo.asr.writer import get_writer
    caps = [Caption(1.25, 3.5, "こんにちは"), Caption(4.0, 9.125, "今日は　晴れ"), Caption(12.0, 12.5, "a b")]
    buf = io.StringIO()
    w = get_writer(buf, "tsv")
    w.write_header()
    for c in caps:
        w.write(Segment(c.start_seconds, c.end_seconds, c.text))
    p = tmp_path / "c.tsv"
    p.write_text(buf.getvalue() + "\n", encoding="utf-8")
    assert read_captions_tsv(str(p)) == caps
    p.write_text("1.0\t2.0\n", encoding="utf-8")
    with pytest.raises(ValueError, match=":1:"):
        read_captions_tsv(str(p))


def test_cli_options():
    from reazonspeech_b200.nemo.asr import cli
    o = cli.parse(["--captions=c.tsv", "--before=10", "--after=1.5", "--to=srt", "a.wav"])
    assert (o.captions, o.before, o.after, o.fmt, o.audio) == ("c.tsv", 10.0, 1.5, "srt", ["a.wav"])
    o = cli.parse(["a.wav"])
    assert (o.captions, o.before, o.after) == (None, 25.0, 0.0)
    for bad in (["--captions=c.tsv", "a.wav", "b.wav"], ["--captions=c.tsv", "--stream", "a.wav"],
                ["--captions=c.tsv", "--text=t.txt", "a.wav"], ["--captions=c.tsv", "--before=-1", "a.wav"]):
        with pytest.raises(ValueError):
            cli.parse(bad)
    with pytest.raises(ValueError):
        cli.parse(["--captions=c.tsv", "--before=x", "a.wav"])


class _Tok:
    def sentence_to_ids(self, text):
        return [ord(ch) % 50 for ch in text if not ch.isspace()]

    def ids_to_text(self, ids):
        return "".join(chr(65 + i % 26) for i in ids)


class _Cfg:
    vocab_size = 50
    blank = 50


class _StubModel:
    """Records each window and places the tokens one per frame from frame 10 (the window's 0.3 s mark after the pad)."""
    tokenizer = _Tok()
    cfg = _Cfg()

    def __init__(self):
        self.calls = []

    def align_segment_tokens(self, waves, token_lists, pad=0):
        self.calls.append(([len(w) for w in waves], [list(t) for t in token_lists], pad))
        out = []
        for ids in token_lists:
            n = len(ids)
            out.append((10, 10 + n - 1, list(range(10, 10 + n)), [-0.1] * n, [-0.1] * n, -0.1 * n, -0.05 * n))
        return out


def test_align_captions_host_plumbing():
    from reazonspeech_b200.nemo.asr import align_captions
    from reazonspeech_b200.nemo.asr.interface import AudioData
    sr = 16000
    audio = AudioData(np.zeros(60 * sr, dtype=np.float32), sr)
    caps = [Caption(50.0, 52.0, "abc"), Caption(85.0, 90.0, "out"), Caption(10.0, 11.0, "  "), Caption(30.0, 33.0, "hello")]
    m = _StubModel()
    res = align_captions(m, audio, caps, before=20.0)
    assert res[1] is None and res[2] is None                       # beyond the audio; no token
    lens, ids, pad = m.calls[0]
    assert pad == sr // 2 and ids == [_Tok().sentence_to_ids("abc"), _Tok().sentence_to_ids("hello")]
    assert lens == [(52 - 30) * sr, (33 - 10) * sr]                 # the windows in input order
    for k, w0 in ((0, 30.0), (3, 10.0)):
        r = res[k]
        assert isinstance(r, AlignedCaption) and r.caption is caps[k] and r.text == caps[k].text
        n = len(_Tok().sentence_to_ids(caps[k].text))
        assert abs(r.start_seconds - (w0 + 0.08 * 10 - 0.5)) < 1e-9
        assert abs(r.end_seconds - (w0 + 0.08 * (10 + n) - 0.5)) < 1e-9
        assert [round(w.seconds - w0, 6) for w in r.subwords] == [round(0.08 * f - 0.5, 6) for f in range(10, 10 + n)]
        assert r.score == pytest.approx(-0.1 * n) and r.log_likelihood == pytest.approx(-0.05 * n)
        assert r.confidence == pytest.approx(-0.1) and r.asr is None and r.cer is None
    with pytest.raises(ValueError):
        align_captions(m, audio, [Caption(5.0, 4.0, "x")])
    assert align_captions(_StubModel(), audio, [Caption(100.0, 101.0, "x")]) == [None]
