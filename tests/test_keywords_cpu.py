"""Keyword spotting without a GPU: the spotting oracle (tests/spot_oracle.py) against brute-force enumeration with planted ties
and against the segment oracle, the hit policy against its sort-then-accept form, keyword validation and tokenisation, the
keyword groups, the seconds of a hit, the CLI options and the host plumbing of ``find_keywords_batch`` on a stub model."""
import math

import numpy as np
import pytest

import segment_oracle as SO
import spot_oracle as K
from reazonspeech_b200.captions import confidence
from reazonspeech_b200.keywords import (MAX_HITS, SCRATCH_CAP_BYTES, THRESHOLD, KeywordHit, check_search, hit_seconds,
                                        keyword_groups, keyword_ids, scratch_bytes)
from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces


def _int_lattice(rng, T, U):
    """Integer-valued log-probabilities from a small range: exact ties between paths are common and exact in float64."""
    return -rng.integers(0, 3, (T, U + 1)).astype(np.float64), -rng.integers(0, 3, (T, U + 1)).astype(np.float64)


@pytest.mark.parametrize("T", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("U", [1, 2, 3])
def test_oracle_equals_brute_force(T, U):
    rng = np.random.default_rng(300 + 10 * T + U)
    cases = [_int_lattice(rng, T, U) for _ in range(12)]
    cases += [(np.log(rng.uniform(0.05, 1.0, (T, U + 1))), np.log(rng.uniform(0.05, 1.0, (T, U + 1)))) for _ in range(3)]
    cases.append((np.zeros((T, U + 1)), np.zeros((T, U + 1))))      # every path ties
    for lpb, lpe in cases:
        r = K.spot(lpb, lpe, T, U)
        E, S, F = K.brute_force(lpb, lpe, T, U)
        assert np.abs(r["E"] - E).max() < 1e-12
        assert r["S"].tolist() == S.tolist()
        for e in range(T):
            frames, token_lp = K.backtrace(r["choice"], lpe, e, U)
            assert frames.tolist() == F[e].tolist(), (e, frames, F[e])
            assert token_lp.tolist() == [lpe[f, u] for u, f in enumerate(frames)]
            assert frames[0] == r["S"][e] and frames[-1] <= e


def test_best_end_is_the_segment_alignment():
    rng = np.random.default_rng(5)
    for T, U in [(1, 1), (3, 5), (12, 4), (30, 9), (40, 1), (25, 32)]:
        for _ in range(4):
            lpb, lpe = np.log(rng.uniform(0.02, 1.0, (T, U + 1))), np.log(rng.uniform(0.02, 1.0, (T, U + 1)))
            r = K.spot(lpb, lpe, T, U)
            seg = SO.segment_align(lpb, lpe, T, U)
            e = int(np.argmax(r["E"]))
            assert abs(r["E"][e] - seg["score"]) < 1e-12 and e == seg["e"] and r["S"][e] == seg["s"]


def test_float32_oracle_is_the_float64_recursion_rounded():
    rng = np.random.default_rng(9)
    T, U = 60, 6
    lpb, lpe = np.log(rng.uniform(0.02, 1.0, (T, U + 1))).astype(np.float32), np.log(rng.uniform(0.02, 1.0, (T, U + 1))).astype(np.float32)
    a, b = K.spot(lpb, lpe, T, U, np.float32), K.spot(lpb.astype(np.float64), lpe.astype(np.float64), T, U)
    assert a["E"].dtype == np.float32 and np.abs(a["E"] - b["E"]).max() <= 1e-5 * np.abs(b["E"]).max()
    agree = a["S"] == b["S"]
    assert agree.all() or (b["margin"][~agree] <= 1e-4).all()


def test_mean_is_the_caption_confidence_on_short_segments():
    rng = np.random.default_rng(13)
    for _ in range(20):
        T, U = int(rng.integers(5, 40)), int(rng.integers(1, 5))
        lpb, lpe = np.log(rng.uniform(0.02, 1.0, (T, U + 1))), np.log(rng.uniform(0.02, 1.0, (T, U + 1)))
        r = K.spot(lpb, lpe, T, U)
        m = K.mean_lp(r["E"], r["S"])
        for e in range(T):
            s = int(r["S"][e])
            if e - s + 1 > 15:
                continue
            frames, _ = K.backtrace(r["choice"], lpe, e, U)
            fl = K.frame_lp(lpb, lpe, frames, e, U)
            assert abs(fl.sum() - r["E"][e]) < 1e-9
            assert abs(confidence(fl) - float(m[e])) <= 1e-6 * abs(float(m[e])) + 1e-6


def _random_scores(rng, T, integer):
    """E and S arrays as the recursion leaves them: S(e) <= e, E < 0 (integer-valued ones tie often)."""
    S = np.array([int(rng.integers(max(0, e - 6), e + 1)) for e in range(T)], dtype=np.int64)
    E = (-rng.integers(1, 6, T) * (np.arange(T) - S + 1)).astype(np.float32) if integer else (-rng.uniform(0.1, 8.0, T)).astype(np.float32)
    return E, S


@pytest.mark.parametrize("integer", [False, True])
def test_policy_equals_the_sorted_scan(integer):
    rng = np.random.default_rng(17 + integer)
    for _ in range(150):
        T = int(rng.integers(1, 70))
        E, S = _random_scores(rng, T, integer)
        if rng.uniform() < 0.2:
            S[rng.integers(0, T)] = -1                                # a frame no segment ends at
        thr = float(rng.choice([-np.inf, -1.0, -2.5, -4.0]))
        H = int(rng.choice([1, 2, 5, 256]))
        got, ref = K.pick(E, S, T, thr, H), K.pick_sorted(E, S, T, thr, H)
        assert got == ref
        assert len(got) <= H
        m = K.mean_lp(E, S)
        for i, (s, e, mm) in enumerate(got):
            assert s == S[e] and mm == m[e] and mm >= np.float32(thr)
            for s2, e2, _ in got[i + 1:]:
                assert e2 < s or s2 > e                               # hits never overlap
        if H == 256 and thr == -np.inf:                               # every valid frame is covered by some hit
            for e in range(T):
                if S[e] >= 0:
                    assert any(S[e] <= he and e >= hs for hs, he, _ in got)


def test_policy_tie_takes_the_smaller_end():
    E = np.array([-2.0, -2.0, -1.0, -2.0], dtype=np.float32)
    S = np.array([0, 1, 1, 3])                                        # m: -2, -2, -0.5, -2
    assert [(s, e) for s, e, _ in K.pick(E, S, 4, -np.inf, 10)] == [(1, 2), (0, 0), (3, 3)]
    assert [(s, e) for s, e, _ in K.pick(E, S, 4, -np.inf, 2)] == [(1, 2), (0, 0)]
    assert [(s, e) for s, e, _ in K.pick(E, S, 4, -1.0, 10)] == [(1, 2)]


def test_keyword_validation_and_tokenisation():
    tok = PieceTableTokenizer(synthetic_pieces(3000))
    assert keyword_ids(["あい"], 3000, tok) == [tok.text_to_ids("あい")]
    assert tok.sentence_to_ids("あい")[0] == 1 and keyword_ids(["あい"], 3000, tok)[0] == tok.sentence_to_ids("あい")[1:]
    assert keyword_ids([[5, 6], (7,)], 3000) == [[5, 6], [7]]
    for bad in ([""], [[]], [[3000]], [[-1]], [[1] * 33]):
        with pytest.raises(ValueError):
            keyword_ids(bad, 3000, tok)
    with pytest.raises(ValueError, match="align_captions"):
        keyword_ids([[1] * 33], 3000)
    assert keyword_ids([[1] * 32], 3000) == [[1] * 32]
    with pytest.raises(ValueError):
        keyword_ids(["あ"], 3000)                                     # text without a tokenizer
    check_search(THRESHOLD, MAX_HITS)
    check_search(-math.inf, 256)
    check_search(np.float32(-2.0), np.int64(1))
    for thr, H in ((math.nan, 4), (math.inf, 4), ("x", 4), (-1.0, 0), (-1.0, 257), (-1.0, 2.0), (-1.0, True)):
        with pytest.raises(ValueError):
            check_search(thr, H)


def test_keyword_groups_stay_under_the_cap():
    rng = np.random.default_rng(3)
    for _ in range(50):
        lengths = [int(x) for x in rng.integers(1, 33, int(rng.integers(1, 120)))]
        n_rec, T = int(rng.integers(1, 4)), int(rng.integers(100, 50000))
        cap = int(rng.choice([1 << 20, 1 << 26, SCRATCH_CAP_BYTES]))
        groups = keyword_groups(lengths, n_rec, T, cap)
        assert sorted(k for g in groups for k in g) == list(range(len(lengths)))
        flat = [lengths[k] for g in groups for k in g]
        assert flat == sorted(flat)
        for g in groups:
            assert len(g) == 1 or scratch_bytes(n_rec, T, len(g), max(lengths[k] for k in g)) <= cap
    assert keyword_groups([], 1, 100) == []
    assert keyword_groups([3, 1, 2], 1, 100) == [[1, 2, 0]]


def test_hit_seconds():
    # frame f of a padded recording lies 0.08 f - 0.5 s into it, clamped at 0; a hit ends at the end of frame e
    s, e = hit_seconds(20, 44, 60.0)
    assert abs(s - 1.1) < 1e-9 and abs(e - (0.08 * 45 - 0.5)) < 1e-9
    assert hit_seconds(0, 3, 60.0) == (0.0, 0.0)
    assert hit_seconds(740, 760, 60.0)[1] == 60.0                      # the trailing pad: clamped to the recording


def test_cli_options(tmp_path):
    from reazonspeech_b200.nemo.asr import cli
    o = cli.parse(["--keywords=k.txt", "--keyword-threshold=-2.5", "--max-hits=8", "--to=srt", "a.wav", "b.wav"])
    assert (o.keywords, o.keyword_threshold, o.max_hits, o.fmt, o.audio) == ("k.txt", -2.5, 8, "srt", ["a.wav", "b.wav"])
    o = cli.parse(["a.wav"])
    assert (o.keywords, o.keyword_threshold, o.max_hits) == (None, None, None)
    assert cli.parse(["--keywords=k.txt", "--keyword-threshold=-inf", "a.wav"]).keyword_threshold == -math.inf
    for extra in (["--text=t.txt"], ["--captions=c.tsv"], ["--stream"], ["--decoding=alsd"], ["--decoding=greedy"],
                  ["--decoding=maes", "--beam=2"], ["--phrases=p.txt"], ["--phrase-score=1"], ["--lm=x.arpa", "--lm-alpha=0.3"]):
        with pytest.raises(ValueError):
            cli.parse(["--keywords=k.txt", *extra, "a.wav"])
    for bad in (["--max-hits=4", "a.wav"], ["--keyword-threshold=-1", "a.wav"], ["--keywords=k.txt", "--max-hits=0", "a.wav"],
                ["--keywords=k.txt", "--max-hits=257", "a.wav"], ["--keywords=k.txt", "--keyword-threshold=nan", "a.wav"],
                ["--keywords=k.txt", "--max-hits=x", "a.wav"]):
        with pytest.raises(ValueError):
            cli.parse(bad)
    p = tmp_path / "k.txt"
    p.write_text("東京\n\n  大阪 \n", encoding="utf-8")
    assert cli.load_keywords(str(p)) == ["東京", "大阪"]


class _Cfg:
    vocab_size = 50
    blank = 50


class _StubTok:
    def text_to_ids(self, text):
        return [ord(ch) % 50 for ch in text if not ch.isspace()]

    def ids_to_text(self, ids):
        return "".join(chr(65 + i % 26) for i in ids)


class _StubModel:
    """Records the call and reports, for keyword k of recording i, hits in pick order: [(40, 40 + n - 1), (10, 10 + n - 1)]."""
    tokenizer = _StubTok()
    cfg = _Cfg()
    decoding = "alsd"

    def __init__(self):
        self.calls = []

    def spot_tokens(self, waves, token_lists, pad=0, *, threshold, max_hits):
        self.calls.append(([len(w) for w in waves], [list(t) for t in token_lists], pad, threshold, max_hits))
        out = []
        for i, _ in enumerate(waves):
            row = []
            for ids in token_lists:
                n = len(ids)
                row.append([(s, s + n - 1, -0.5 * n - i, -0.5 - i / n, list(range(s, s + n)), [-0.5] * n) for s in (40, 10)])
            out.append(row)
        return out


def test_find_keywords_host_plumbing():
    from reazonspeech_b200.nemo.asr import find_keywords, find_keywords_batch
    from reazonspeech_b200.nemo.asr.interface import AudioData
    sr = 16000
    audios = [AudioData(np.zeros(10 * sr, dtype=np.float32), sr), AudioData(np.zeros(3 * sr, dtype=np.float32), sr)]
    m = _StubModel()
    res = find_keywords_batch(m, audios, ["ab", [7, 8, 9]], threshold=-3.0, max_hits=5)
    lens, ids, pad, thr, H = m.calls[0]
    assert lens == [10 * sr, 3 * sr] and pad == sr // 2 and ids == [_StubTok().text_to_ids("ab"), [7, 8, 9]] and (thr, H) == (-3.0, 5)
    assert len(res) == 2 and all(len(r) == 2 for r in res)
    for i, per_kw in enumerate(res):
        for kw, hits in zip(["ab", [7, 8, 9]], per_kw):
            n = 2 if kw == "ab" else 3
            assert [type(h) for h in hits] == [KeywordHit, KeywordHit] and all(h.keyword == kw for h in hits)
            assert [round(h.start_seconds, 6) for h in hits] == [round(0.08 * 10 - 0.5, 6), round(0.08 * 40 - 0.5, 6)]   # time order
            assert abs(hits[0].end_seconds - (0.08 * (10 + n) - 0.5)) < 1e-9
            assert [round(w.seconds, 6) for w in hits[0].subwords] == [round(0.08 * f - 0.5, 6) for f in range(10, 10 + n)]
            assert hits[0].score == pytest.approx(-0.5 * n - i) and hits[0].confidence == pytest.approx(-0.5 - i / n)
    assert find_keywords(_StubModel(), audios[0], ["ab"])[0][0].start_seconds == pytest.approx(0.3)
    assert find_keywords_batch(_StubModel(), audios, []) == [[], []]


def test_find_keywords_rejects_before_the_gpu():
    from reazonspeech_b200.nemo.asr import find_keywords
    from reazonspeech_b200.nemo.asr.interface import AudioData
    audio = AudioData(np.zeros(16000, dtype=np.float32), 16000)
    m = _StubModel()
    for kws, kw in (([""], {}), ([[50]], {}), ([[1] * 33], {}), (["a"], {"max_hits": 0}), (["a"], {"threshold": math.nan})):
        with pytest.raises(ValueError):
            find_keywords(m, audio, kws, **kw)
    assert m.calls == []

    class _NoSpot:
        tokenizer = _StubTok()
        cfg = _Cfg()
    with pytest.raises(ValueError, match="one GPU"):
        find_keywords(_NoSpot(), audio, ["a"])
