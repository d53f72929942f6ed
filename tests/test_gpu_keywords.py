"""Keyword spotting on the GPU (rnnt_lattice_kernel<true>, rnnt_spot_dp_kernel and rnnt_spot_pick_kernel; keywords.py): the
pair lattice against the forced alignment's, the recursion against the float64 oracle (tests/spot_oracle.py) on the kernel's
own lattice, the hits against the oracle's policy on the kernel's own E and S, every hit against a forced alignment of its
span, batch invariance, edge cases and argument checks, ``find_keywords`` end to end, the CLI, and recovery at the bench
geometry."""
import math

import numpy as np
import pytest
import torch

import spot_oracle as K
from reazonspeech_b200.synth import synth_clip

pytestmark = pytest.mark.gpu


def _enc(cfg, T_lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(T_lens), max(T_lens + [1]), cfg.d_model, generator=g)
    for b, n in enumerate(T_lens):
        enc[b, n:] = 0
    return enc, torch.tensor(T_lens, dtype=torch.int32)


def _labels(kws):
    lab = torch.zeros(len(kws), max(len(x) for x in kws), dtype=torch.int32)
    for k, x in enumerate(kws):
        lab[k, : len(x)] = torch.tensor(x, dtype=torch.int32)
    return lab, torch.tensor([len(x) for x in kws], dtype=torch.int32)


def _random_kws(cfg, lens, seed):
    rng = np.random.default_rng(seed)
    return [[int(k) for k in rng.integers(0, cfg.vocab_size, n)] for n in lens]


def _spot(eng, enc, T, lab, ll, threshold=-1.0, max_hits=64):
    return [x.cpu() for x in eng.spot(enc.cuda().contiguous(), T.cuda(), lab.cuda(), ll.cuda(), threshold, max_hits, scores=True)]


def _lattice(eng, enc, T, lab, ll):
    return [x.cpu() for x in eng.spot_lattice(enc.cuda().contiguous(), T.cuda(), lab.cuda(), ll.cuda())]


TINY_T = [40, 1, 23, 9, 64]
TINY_U = [3, 1, 6, 12, 32, 2]             # U = 1, U = 32, U > T


@pytest.fixture(scope="module")
def tiny_case(tiny_cfg):
    kws = _random_kws(tiny_cfg, TINY_U, 31)
    enc, T = _enc(tiny_cfg, TINY_T, 32)
    lab, ll = _labels(kws)
    return enc, T, lab, ll


def test_pair_lattice_is_the_forced_alignment_lattice(tiny_engine, tiny_case):
    enc, T, lab, ll = tiny_case
    R, Kn = len(TINY_T), len(TINY_U)
    lpb, lpe = _lattice(tiny_engine, enc, T, lab, ll)
    # the forced alignment of every pair, the encoder output copied per pair
    rb, re = [x.cpu() for x in tiny_engine.align_lattice(enc.repeat_interleave(Kn, 0).cuda().contiguous(), T.repeat_interleave(Kn).cuda(),
                                                          lab.repeat(R, 1).cuda(), ll.repeat(R).cuda())]
    for r in range(R):
        for k in range(Kn):
            p, Tr, U = r * Kn + k, TINY_T[r], TINY_U[k]
            assert torch.equal(lpb[p, :Tr, :U + 1], rb[p, :Tr, :U + 1]), (r, k)
            assert torch.equal(lpe[p, :Tr, :U + 1], re[p, :Tr, :U + 1]), (r, k)
            assert torch.isnan(lpb[p, Tr:]).all() and torch.isnan(lpb[p, :, U + 1:]).all()


def test_scores_against_the_float64_oracle(tiny_engine, tiny_case):
    enc, T, lab, ll = tiny_case
    Kn = len(TINY_U)
    lpb, lpe = _lattice(tiny_engine, enc, T, lab, ll)
    E, S = _spot(tiny_engine, enc, T, lab, ll)[6:]
    differ = 0
    for r, Tr in enumerate(TINY_T):
        for k, U in enumerate(TINY_U):
            p = r * Kn + k
            o = K.spot(lpb[p].double().numpy(), lpe[p].double().numpy(), Tr, U)
            e64 = o["E"]
            assert np.all(np.abs(E[p, :Tr].double().numpy() - e64) <= 1e-4 * np.abs(e64) + 1e-5), (r, k)
            bad = S[p, :Tr].numpy() != o["S"]
            assert np.all(o["margin"][bad] <= 1e-4), (r, k)
            differ += int(bad.sum())
            assert torch.isnan(E[p, Tr:]).all() and (S[p, Tr:] == -1).all()
    print(f"start frames differing from the float64 oracle at near-ties: {differ}")


@pytest.mark.parametrize("thr_kind,max_hits", [("-inf", 64), ("-inf", 256), ("median", 8), ("default", 64), ("-inf", 1)])
def test_hits_are_the_oracle_policy(tiny_engine, tiny_case, thr_kind, max_hits):
    enc, T, lab, ll = tiny_case
    Kn = len(TINY_U)
    lpb, lpe = _lattice(tiny_engine, enc, T, lab, ll)
    E, S = _spot(tiny_engine, enc, T, lab, ll, -math.inf)[6:]
    ms = np.concatenate([K.mean_lp(E[r * Kn + k, :Tr].numpy(), S[r * Kn + k, :Tr].numpy()) for r, Tr in enumerate(TINY_T) for k in range(Kn)])
    thr = {"-inf": -math.inf, "median": float(np.median(ms)), "default": -1.0}[thr_kind]
    span, score, conf, frames, token_lp, count, E2, S2 = _spot(tiny_engine, enc, T, lab, ll, thr, max_hits)
    assert torch.equal(E2.nan_to_num(7.0), E.nan_to_num(7.0)) and torch.equal(S2, S)
    total = 0
    for r, Tr in enumerate(TINY_T):
        for k, U in enumerate(TINY_U):
            p = r * Kn + k
            want = K.pick(E[p].numpy(), S[p].numpy(), Tr, thr, max_hits)
            n = int(count[p])
            total += n
            assert n == len(want), (r, k)
            assert [(int(span[p, h, 0]), int(span[p, h, 1])) for h in range(n)] == [(s, e) for s, e, _ in want]
            assert [float(conf[p, h]) for h in range(n)] == [float(m) for _, _, m in want]
            assert [float(score[p, h]) for h in range(n)] == [float(E[p, e]) for _, e, _ in want]
            # the kernel's fp32 recursion, step for step, gives its choices: the backtraces must match exactly
            o32 = K.spot(lpb[p].numpy(), lpe[p].numpy(), Tr, U, np.float32)
            assert np.array_equal(o32["E"].view(np.int32), E[p, :Tr].numpy().view(np.int32)) and np.array_equal(o32["S"], S[p, :Tr].numpy())
            for h, (s, e, _) in enumerate(want):
                fr, tl = K.backtrace(o32["choice"], lpe[p].numpy(), e, U)
                assert frames[p, h, :U].tolist() == fr.tolist() and fr[0] == s
                assert np.array_equal(token_lp[p, h, :U].numpy().view(np.int32), tl.astype(np.float32).view(np.int32))
                assert (frames[p, h, U:] == -1).all() and torch.isnan(token_lp[p, h, U:]).all()
    print(f"threshold {thr_kind} ({thr:.3f}), max_hits {max_hits}: {total} hits")
    if thr_kind == "-inf":
        assert total > 0


def test_every_hit_is_a_forced_alignment_of_its_span(tiny_engine, tiny_case):
    enc, T, lab, ll = tiny_case
    Kn = len(TINY_U)
    span, score, conf, frames, token_lp, count = _spot(tiny_engine, enc, T, lab, ll, -math.inf, 16)[:6]
    checked = 0
    for r, Tr in enumerate(TINY_T):
        for k, U in enumerate(TINY_U):
            p = r * Kn + k
            for h in range(int(count[p])):
                s, e = int(span[p, h, 0]), int(span[p, h, 1])
                fr, _, vit, _ = [x.cpu() for x in tiny_engine.align(enc[r:r + 1, s:e + 1].contiguous().cuda(),
                                                                    torch.tensor([e - s + 1], dtype=torch.int32).cuda(),
                                                                    lab[k:k + 1, :U].contiguous().cuda(), ll[k:k + 1].cuda())]
                assert abs(float(vit[0]) - float(score[p, h])) <= 1e-5 * abs(float(score[p, h])), (r, k, h)
                assert (fr[0] + s).tolist() == frames[p, h, :U].tolist(), (r, k, h)
                checked += 1
    assert checked > 0


def _same_pair(a, pa, b, pb, Tr, U):
    span, score, conf, frames, token_lp, count, E, S = a
    span2, score2, conf2, frames2, token_lp2, count2, E2, S2 = b
    n = int(count[pa])
    assert int(count2[pb]) == n
    assert torch.equal(span[pa, :n], span2[pb, :n]) and torch.equal(score[pa, :n], score2[pb, :n]) and torch.equal(conf[pa, :n], conf2[pb, :n])
    assert torch.equal(frames[pa, :n, :U], frames2[pb, :n, :U]) and torch.equal(token_lp[pa, :n, :U], token_lp2[pb, :n, :U])
    assert torch.equal(E[pa, :Tr], E2[pb, :Tr]) and torch.equal(S[pa, :Tr], S2[pb, :Tr])


def test_batch_invariance(tiny_engine, tiny_case):
    enc, T, lab, ll = tiny_case
    R, Kn = len(TINY_T), len(TINY_U)
    full = _spot(tiny_engine, enc, T, lab, ll, -math.inf, 32)
    perm = [3, 0, 4, 2, 1]
    moved = _spot(tiny_engine, enc[perm], T[perm], lab, ll, -math.inf, 32)
    kperm = [5, 2, 0, 4, 1, 3]
    kmoved = _spot(tiny_engine, enc, T, lab[kperm], ll[kperm], -math.inf, 32)
    for r, Tr in enumerate(TINY_T):
        alone_r = _spot(tiny_engine, enc[r:r + 1, :Tr], T[r:r + 1], lab, ll, -math.inf, 32)
        for k, U in enumerate(TINY_U):
            p = r * Kn + k
            _same_pair(full, p, moved, perm.index(r) * Kn + k, Tr, U)
            _same_pair(full, p, kmoved, r * Kn + kperm.index(k), Tr, U)
            _same_pair(full, p, alone_r, k, Tr, U)
            alone = _spot(tiny_engine, enc[r:r + 1, :Tr], T[r:r + 1], lab[k:k + 1, :U], ll[k:k + 1], -math.inf, 32)
            _same_pair(full, p, alone, 0, Tr, U)


def test_keyword_groups_at_different_caps(tiny_engine, tiny_cfg):
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.keywords import keyword_groups
    model = asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=2)
    waves = [np.pad(synth_clip(600 + i, s), 8000).astype(np.float32) for i, s in enumerate((3.0, 5.5, 1.2))]
    kws = _random_kws(tiny_cfg, [4, 1, 7, 2, 3, 12, 5], 33)
    ref = model.spot_tokens(waves, kws, threshold=-math.inf, max_hits=16)
    for cap in (1, 20_000, 60_000):
        T = model.engine.enc_frames((len(waves[1]) + 3) & ~3)
        if cap > 1:
            assert 1 < len(keyword_groups([len(k) for k in kws], 2, T, cap)) < len(kws)
        assert model.spot_tokens(waves, kws, threshold=-math.inf, max_hits=16, cap=cap) == ref
    assert any(hits for row in ref for hits in row)


def test_edges(tiny_engine, tiny_cfg):
    V = tiny_cfg.vocab_size
    T_lens = [1, 0, 5, 40]
    enc, T = _enc(tiny_cfg, T_lens, 34)
    kws = [[1], [2, 3], [4] * 12, [5, V, 6], [7, 8]]           # U > T, and a label outside [0, V)
    lab, ll = _labels(kws)
    ll2 = ll.clone(); ll2[4] = 0                              # label_len outside [1, U_max]
    out = _spot(tiny_engine, enc, T, lab, ll2, -math.inf, 256)
    span, score, conf, frames, token_lp, count, E, S = out
    Kn = len(kws)
    for r, Tr in enumerate(T_lens):
        for k in range(Kn):
            p = r * Kn + k
            if Tr == 0 or k >= 3:                             # an empty recording, a bad keyword: no hit, no segment end
                assert int(count[p]) == 0 and torch.isnan(E[p]).all() and (S[p] == -1).all(), (r, k)
                continue
            n = int(count[p])
            assert n >= 1
            hits = [(int(span[p, h, 0]), int(span[p, h, 1])) for h in range(n)]
            for i, (s, e) in enumerate(hits):                 # a non-overlapping tiling of the candidates
                assert 0 <= s <= e < Tr and all(e2 < s or s2 > e for s2, e2 in hits[i + 1:])
            for e in range(Tr):
                assert any(int(S[p, e]) <= he and e >= hs for hs, he in hits)
    good = [0, 1, 2]
    ref = _spot(tiny_engine, enc, T, lab[good], ll[good], -math.inf, 256)
    for r, Tr in enumerate(T_lens):
        for j, k in enumerate(good):
            _same_pair(out, r * Kn + k, ref, r * len(good) + j, Tr, len(kws[k]))
    # the max_hits cap: the first hits of the uncapped pick order
    capped = _spot(tiny_engine, enc, T, lab, ll2, -math.inf, 3)
    for p in range(len(T_lens) * Kn):
        n = min(int(count[p]), 3)
        assert int(capped[5][p]) == n and torch.equal(capped[0][p, :n], span[p, :n])


def test_bad_host_arguments_are_rejected_before_any_launch(tiny_engine, tiny_cfg):
    eng = tiny_engine
    enc, T = [x.cuda() for x in _enc(tiny_cfg, [6], 35)]
    lab, ll = [x.cuda() for x in _labels([[1, 2]])]
    H, U = 4, 2
    outs = [torch.zeros(1, H, 2, dtype=torch.int32, device="cuda"), torch.zeros(1, H, device="cuda"), torch.zeros(1, H, device="cuda"),
            torch.zeros(1, H, U, dtype=torch.int32, device="cuda"), torch.zeros(1, H, U, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")]
    p = [x.data_ptr() for x in outs]
    f = eng.lib.rs_rnnt_spot
    base = dict(R=1, Tm=6, K=1, U=U, thr=-1.0, H=H)

    def call(q=p, **kw):
        a = {**base, **kw}
        return f(eng.h, enc.data_ptr(), T.data_ptr(), a["R"], a["Tm"], lab.data_ptr(), ll.data_ptr(), a["K"], a["U"], a["thr"], a["H"],
                 *q, None, None, None)
    n0 = eng.launch_count
    for kw in (dict(U=33), dict(U=0), dict(H=0), dict(H=257), dict(K=0), dict(R=0), dict(Tm=0), dict(thr=math.nan), dict(thr=math.inf)):
        assert call(**kw) != 0, kw
        assert eng.lib.rs_last_error(eng.h)
    for i in range(6):                                          # each output missing in turn
        q = list(p); q[i] = None
        assert call(q) != 0
    assert f(eng.h, None, T.data_ptr(), 1, 6, lab.data_ptr(), ll.data_ptr(), 1, U, -1.0, H, *p, None, None, None) != 0
    assert eng.launch_count == n0
    assert call(thr=-math.inf) == 0 and call() == 0


# ---------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def model(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    return asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=2)


def _audios():
    from reazonspeech_b200.nemo import asr
    return [asr.audio_from_numpy(synth_clip(700 + i, s), 16000) for i, s in enumerate((4.0, 7.5, 2.0))]


def _keywords(model):
    pieces = model.tokenizer.pieces
    return [pieces[10] + pieces[11], [20, 21, 22], pieces[40]]


def test_find_keywords_batch_equals_one_audio_at_a_time(model):
    from reazonspeech_b200.nemo import asr
    audios, kws = _audios(), _keywords(model)
    batch = asr.find_keywords_batch(model, audios, kws, threshold=-math.inf, max_hits=5)
    assert len(batch) == len(audios)
    for a, lists in zip(audios, batch):
        one = asr.find_keywords(model, a, kws, threshold=-math.inf, max_hits=5)
        assert len(lists) == len(kws)
        for kw, hits, hits1 in zip(kws, lists, one):
            assert [(h.start_seconds, h.end_seconds, h.score, h.confidence) for h in hits] == \
                   [(h.start_seconds, h.end_seconds, h.score, h.confidence) for h in hits1]
            assert 1 <= len(hits) <= 5 and all(h.keyword == kw for h in hits)
            starts = [h.start_seconds for h in hits]
            assert starts == sorted(starts)
            for h in hits:
                assert 0.0 <= h.start_seconds <= h.end_seconds <= a.seconds and h.score <= 0 and math.isfinite(h.confidence)
                secs = [w.seconds for w in h.subwords]
                assert secs == sorted(secs) and len(secs) == (3 if isinstance(kw, list) else len(model.tokenizer.text_to_ids(kw)))
    with pytest.raises(ValueError):
        asr.find_keywords(model, audios[0], [[model.cfg.vocab_size]])
    alsd = asr.load_model("cuda:0", synthetic=True, config=model.engine.cfg, seed=0, decoding="alsd")
    again = asr.find_keywords(alsd, audios[0], kws, threshold=-math.inf, max_hits=5)
    assert [[(h.start_seconds, h.score) for h in row] for row in again] == [[(h.start_seconds, h.score) for h in row] for row in batch[0]]


def test_cli_keywords_writes_hits(tmp_path, monkeypatch, model, tiny_cfg):
    import sys
    import scipy.io.wavfile as wavfile
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr import cli
    audios = _audios()[:2]
    paths = []
    for i, a in enumerate(audios):
        paths.append(str(tmp_path / f"a{i}.wav"))
        wavfile.write(paths[-1], 16000, (np.asarray(a.waveform) * 20000).astype(np.int16))
    kw = model.tokenizer.pieces
    kfile = tmp_path / "k.txt"
    kfile.write_text(f"{kw[10]}{kw[11]}\n\n{kw[40]}\n", encoding="utf-8")
    out = tmp_path / "k.tsv"
    monkeypatch.setattr(sys.modules["reazonspeech_b200.nemo.asr.transcribe"], "load_model",
                        lambda **kw: asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0))
    cli.main([f"--keywords={kfile}", "--keyword-threshold=-inf", "--max-hits=2", "--to=tsv", "-o", str(out), *paths])
    rows = [line.split("\t") for line in out.read_text(encoding="utf-8").splitlines()[1:] if line.strip()]
    assert len(rows) == 2 * 2 * 2                                # 2 files x 2 keywords x 2 hits
    texts = [r[2] for r in rows]
    assert texts.count(f"{kw[10]}{kw[11]}") == 4 and texts.count(kw[40]) == 4
    starts = [float(r[0]) for r in rows]
    assert starts[:4] == sorted(starts[:4]) and starts[4:] == sorted(starts[4:]) and min(starts[4:]) >= audios[0].seconds - 1e-3


# ---------------------------------------------------------------- production size
# Recovery measured on one H100 with the seeded synthetic 619 M weights: the keyword is 3-5 consecutive greedy tokens from
# the middle of each clip, and a clip counts when one of its 64 best hits (threshold -inf) overlaps those tokens' greedy
# frames.  The synthetic joint is nearly flat, so the cheapest segments pack a keyword into one or two frames wherever the
# emissions happen to be cheapest; the bar holds the measured count, it is not an accuracy claim (DESIGN.md section 4).
PLANTED_HITS_SYNTHETIC_619M = 20


@pytest.fixture(scope="module")
def full():
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    waves = [np.pad(synth_clip(i, 30.0), 8000) for i in range(32)]
    x = torch.from_numpy(np.stack(waves)).float().cuda()
    lens = torch.full((32,), len(waves[0]), dtype=torch.int32).cuda()
    enc, enc_len = eng.encode(*eng.log_mel(x, lens))
    tk, fr, nt = [a.cpu() for a in eng.greedy(enc, enc_len)]
    return cfg, eng, enc, enc_len, [tk[b, : int(nt[b])].tolist() for b in range(32)], [fr[b, : int(nt[b])].tolist() for b in range(32)]


def test_planted_recovery_at_the_bench_geometry(full):
    cfg, eng, enc, enc_len, toks, frs = full
    rng = np.random.default_rng(36)
    kws, spans = [], []
    for b in range(32):
        n = int(rng.integers(3, 6))
        if len(toks[b]) < n:
            kws.append(toks[b][:1] or [5]); spans.append((0, int(enc_len[b]) - 1)); continue
        a = (len(toks[b]) - n) // 2
        kws.append(toks[b][a:a + n]); spans.append((frs[b][a], frs[b][a + n - 1]))
    lab, ll = [x.cuda() for x in _labels(kws)]
    found = {}
    for name, thr in (("default", -1.0), ("-inf", -math.inf)):
        span, score, conf, frames, token_lp, count = [x.cpu() for x in eng.spot(enc, enc_len, lab, ll, thr, 64)]
        hit = 0
        for b, (f0, f1) in enumerate(spans):
            p = b * 32 + b                                        # clip b, its own keyword
            hit += any(int(span[p, h, 0]) <= f1 and int(span[p, h, 1]) >= f0 for h in range(int(count[p])))
        found[name] = hit
        total = int(count.view(32, 32).diagonal().sum())
        print(f"threshold {name}: {hit}/32 clips have a hit overlapping the keyword's greedy frames ({total} hits on the 32 own pairs)")
    assert found["-inf"] >= PLANTED_HITS_SYNTHETIC_619M
