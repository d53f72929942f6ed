"""Caption alignment on the GPU (rnnt_segment_dp_kernel in csrc/align.cu, captions.py): the segment DP against the float64
oracle (tests/segment_oracle.py) on the kernel's own lattice, the whole path against the all-float64 oracle, batch
invariance, the bench geometry at 619 M, argument checks, ``align_captions`` end to end, planted recovery, two devices and
the CLI."""
import math

import numpy as np
import pytest
import torch

import align_oracle as A
import segment_oracle as S
from reazonspeech_b200.synth import synth_clip

pytestmark = pytest.mark.gpu


def _inputs(cfg, T_lens, labels, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(T_lens), max(T_lens), cfg.d_model, generator=g)
    for b, n in enumerate(T_lens):
        enc[b, n:] = 0
    lab = torch.zeros(len(labels), max([len(x) for x in labels] + [1]), dtype=torch.int32)
    for b, x in enumerate(labels):
        lab[b, : len(x)] = torch.tensor(x, dtype=torch.int32)
    return enc, torch.tensor(T_lens, dtype=torch.int32), lab, torch.tensor([len(x) for x in labels], dtype=torch.int32)


def _random_labels(cfg, lens, seed):
    rng = np.random.default_rng(seed)
    return [[int(k) for k in rng.integers(0, cfg.vocab_size, n)] for n in lens]


def _segment(eng, enc, T, lab, ll):
    return [x.cpu() for x in eng.align_segment(enc.cuda().contiguous(), T.cuda(), lab.cuda(), ll.cuda())]


def _check_dp(eng, enc, T, lab, ll, T_lens, U_lens, tag, rows=None):
    """The segment DP on the kernel's own lattice (rs_rnnt_align_lattice) vs the float64 oracle on the same fp32 lattice."""
    lpb, lpe = [x.cpu() for x in eng.align_lattice(enc.cuda().contiguous(), T.cuda(), lab.cuda(), ll.cuda())]
    seg, frames, token_lp, frame_lp, vit, lo = _segment(eng, enc, T, lab, ll)
    differ = 0
    for b in (range(len(T_lens)) if rows is None else rows):
        Tb, Ub = T_lens[b], U_lens[b]
        r = S.segment_align(lpb[b].double().numpy(), lpe[b].double().numpy(), Tb, Ub)
        assert abs(float(vit[b]) - r["score"]) <= 1e-4 * abs(r["score"]) + 1e-5, f"{tag} b={b}"
        assert abs(float(lo[b]) - r["loglik"]) <= 1e-4 * abs(r["loglik"]) + 1e-5, f"{tag} b={b}"
        s, e = int(seg[b, 0]), int(seg[b, 1])
        fr = frames[b, :Ub].numpy()
        if (s, e, fr.tolist()) != (r["s"], r["e"], r["frames"].tolist()):
            assert r["margin"] <= 1e-4, f"{tag} b={b}: segment differs with a decision margin {r['margin']:.2e}"
            differ += 1
        assert 0 <= s <= e < Tb and fr[0] == s and fr[-1] <= e and np.all(np.diff(fr) >= 0), f"{tag} b={b}"
        assert torch.equal(token_lp[b, :Ub], lpe[b, fr, np.arange(Ub)]), f"{tag} b={b}"
        fl = frame_lp[b].double()
        assert torch.isnan(fl[:s]).all() and torch.isnan(fl[e + 1:]).all() and not torch.isnan(fl[s:e + 1]).any()
        assert abs(float(fl[s:e + 1].sum()) - float(vit[b])) <= 1e-4 * abs(float(vit[b])) + 1e-4, f"{tag} b={b}"
        assert float(lo[b]) >= float(vit[b]) - 1e-4 * abs(float(vit[b]))
        assert (frames[b, Ub:] == -1).all() and torch.isnan(token_lp[b, Ub:]).all()
    return differ


# ---------------------------------------------------------------- tiny model
TINY_T = [20, 1, 13, 7, 30, 16, 1]
TINY_U = [6, 1, 3, 12, 9, 1, 4]          # T = 1, U = 1, U > T


def test_dp_on_the_kernels_lattice_tiny(tiny_engine, tiny_cfg):
    labels = _random_labels(tiny_cfg, TINY_U, 21)
    enc, T, lab, ll = _inputs(tiny_cfg, TINY_T, labels, 22)
    _check_dp(tiny_engine, enc, T, lab, ll, TINY_T, TINY_U, "tiny")


def test_dp_wider_than_the_block(tiny_engine, tiny_cfg):
    """U_max + 1 above the DP's 256 threads, with U > T and T > U in one batch."""
    T_lens, U_lens = [120, 300, 40], [300, 90, 5]
    labels = _random_labels(tiny_cfg, U_lens, 23)
    enc, T, lab, ll = _inputs(tiny_cfg, T_lens, labels, 24)
    _check_dp(tiny_engine, enc, T, lab, ll, T_lens, U_lens, "wide")


def test_whole_path_vs_float64_oracle_tiny(tiny_engine, tiny_cfg, tiny_sd):
    """Labels = a middle slice of the greedy transcript; score and log-likelihood against the all-float64 oracle."""
    T_lens = [40, 25, 60, 33]
    enc, T, _, _ = _inputs(tiny_cfg, T_lens, [[]] * len(T_lens), 25)
    tk, _, nt = [x.cpu() for x in tiny_engine.greedy(enc.cuda().contiguous(), T.cuda())]
    labels = []
    for b in range(len(T_lens)):
        toks = tk[b, : int(nt[b])].tolist() or [5, 6]
        labels.append(toks[len(toks) // 3: max(2 * len(toks) // 3, len(toks) // 3 + 1)])
    _, _, lab, ll = _inputs(tiny_cfg, T_lens, labels, 25)
    _, _, _, _, vit, lo = _segment(tiny_engine, enc, T, lab, ll)
    worst = 0.0
    for b, Tb in enumerate(T_lens):
        rb, re = A.lattice(enc[b], labels[b], tiny_sd, tiny_cfg, T=Tb)
        r = S.segment_align(rb, re, Tb, len(labels[b]))
        worst = max(worst, abs(float(vit[b]) - r["score"]), abs(float(lo[b]) - r["loglik"]))
    print(f"tiny whole path: max |error| of score / loglik {worst:.2e}")
    assert worst <= 1e-2


def test_batch_invariance(tiny_engine, tiny_cfg):
    labels = _random_labels(tiny_cfg, TINY_U, 26)
    enc, T, lab, ll = _inputs(tiny_cfg, TINY_T, labels, 27)
    full = _segment(tiny_engine, enc, T, lab, ll)
    perm = [4, 0, 6, 2, 1, 5, 3]
    moved = _segment(tiny_engine, enc[perm], T[perm], lab[perm], ll[perm])
    for i, b in enumerate(perm):
        Tb, Ub = TINY_T[b], TINY_U[b]
        alone = _segment(tiny_engine, enc[b:b + 1, :Tb], T[b:b + 1], lab[b:b + 1, :Ub], ll[b:b + 1])
        for got, row in ((moved, i), (alone, 0)):
            seg, frames, token_lp, frame_lp, vit, lo = got
            assert torch.equal(seg[row], full[0][b]) and torch.equal(frames[row, :Ub], full[1][b, :Ub])
            assert torch.equal(token_lp[row, :Ub], full[2][b, :Ub])
            assert torch.equal(frame_lp[row, :Tb].nan_to_num(7.0), full[3][b, :Tb].nan_to_num(7.0))
            assert torch.equal(vit[row], full[4][b]) and torch.equal(lo[row], full[5][b])


def test_invalid_rows(tiny_engine, tiny_cfg):
    V = tiny_cfg.vocab_size
    labels = [[1, 2, 3], [4, V, 5], [], [7, -1], [8, 9]]
    T_lens = [9, 9, 9, 9, 9]
    enc, T, lab, ll = _inputs(tiny_cfg, T_lens, labels, 28)
    seg, frames, token_lp, frame_lp, vit, lo = _segment(tiny_engine, enc, T, lab, ll)
    for b in (1, 2, 3):
        assert seg[b].tolist() == [-1, -1] and (frames[b] == -1).all() and torch.isnan(token_lp[b]).all()
        assert torch.isnan(frame_lp[b]).all() and math.isnan(float(vit[b])) and math.isnan(float(lo[b]))
    good = [0, 4]
    g = _segment(tiny_engine, enc[good], T[good], lab[good], ll[good])
    for x, y in zip(g, (seg, frames, token_lp, frame_lp, vit, lo)):
        assert torch.equal(x.nan_to_num(7.0), y[good].nan_to_num(7.0))
    T_bad = T.clone(); T_bad[4] = 0                                    # enc_len outside [1, T_max]
    seg2 = _segment(tiny_engine, enc, T_bad, lab, ll)[0]
    assert seg2[4].tolist() == [-1, -1] and torch.equal(seg2[0], seg[0])


def test_bad_host_arguments_are_rejected_before_any_launch(tiny_engine, tiny_cfg):
    eng = tiny_engine
    enc, T, lab, ll = [x.cuda() for x in _inputs(tiny_cfg, [5], [[1, 2]], 29)]
    seg = torch.zeros(1, 2, dtype=torch.int32, device="cuda")
    fr = torch.zeros(1, 2, dtype=torch.int32, device="cuda")
    tl, fl, v, lo = torch.zeros(1, 2, device="cuda"), torch.zeros(1, 5, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    p = [x.data_ptr() for x in (seg, fr, tl, fl, v, lo)]
    f = eng.lib.rs_rnnt_align_segment
    n0 = eng.launch_count
    for B, Tm, U in ((0, 5, 2), (1, 0, 2), (1, 5, 0), (1, 5, 14528)):
        assert f(eng.h, enc.data_ptr(), T.data_ptr(), B, Tm, lab.data_ptr(), ll.data_ptr(), U, *p, None) != 0
    assert f(eng.h, None, T.data_ptr(), 1, 5, lab.data_ptr(), ll.data_ptr(), 2, *p, None) != 0
    for k in range(6):                                                  # each output missing in turn
        q = list(p); q[k] = None
        assert f(eng.h, enc.data_ptr(), T.data_ptr(), 1, 5, lab.data_ptr(), ll.data_ptr(), 2, *q, None) != 0
    assert eng.launch_count == n0
    assert f(eng.h, enc.data_ptr(), T.data_ptr(), 1, 5, lab.data_ptr(), ll.data_ptr(), 2, *p, None) == 0


# ---------------------------------------------------------------- production size
@pytest.fixture(scope="module")
def full():
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    sd = random_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, "cuda:0")
    waves = [np.pad(synth_clip(i, 30.0), 8000) for i in range(32)]
    x = torch.from_numpy(np.stack(waves)).float().cuda()
    lens = torch.full((32,), len(waves[0]), dtype=torch.int32).cuda()
    enc, enc_len = eng.encode(*eng.log_mel(x, lens))
    tk, fr, nt = [a.cpu() for a in eng.greedy(enc, enc_len)]
    return cfg, sd, eng, enc, enc_len, [tk[b, : int(nt[b])].tolist() for b in range(32)], [fr[b, : int(nt[b])].tolist() for b in range(32)]


def _mid_captions(labels, gframes, enc_len):
    """Each clip's caption: the greedy tokens emitted over its middle third of frames [a, b)."""
    caps, spans = [], []
    for b, (toks, frs) in enumerate(zip(labels, gframes)):
        T = int(enc_len[b])
        a, z = T // 3, 2 * T // 3
        keep = [k for k, f in zip(toks, frs) if a <= f < z]
        caps.append(keep or toks[:1])
        spans.append((a, z))
    return caps, spans


def _packed(labels):
    U = max(len(x) for x in labels)
    lab = torch.zeros(len(labels), U, dtype=torch.int32)
    for b, x in enumerate(labels):
        lab[b, : len(x)] = torch.tensor(x, dtype=torch.int32)
    return lab.cuda(), torch.tensor([len(x) for x in labels], dtype=torch.int32, device="cuda")


def test_bench_geometry_inequalities_and_dp(full):
    cfg, sd, eng, enc, enc_len, labels, gframes = full
    caps, _ = _mid_captions(labels, gframes, enc_len)
    lab, ll = _packed(caps)
    seg, frames, token_lp, frame_lp, vit, lo = [x.cpu() for x in eng.align_segment(enc, enc_len, lab, ll)]
    fvit = eng.align(enc, enc_len, lab, ll)[2].cpu()
    for b in range(32):
        tol = 1e-4 * abs(float(fvit[b]))
        assert float(lo[b]) >= float(vit[b]) - tol and float(vit[b]) >= float(fvit[b]) - tol, \
            f"clip {b}: loglik {float(lo[b])}, segment {float(vit[b])}, whole window {float(fvit[b])}"
    n = [len(c) for c in caps]
    picks = sorted({int(np.argmin(n)), int(np.argmax(n)), 5, 17})
    T_lens = [int(t) for t in enc_len.cpu()]
    _check_dp(eng, enc.cpu(), enc_len.cpu(), lab.cpu(), ll.cpu(), T_lens, n, "bench", rows=picks)


# Planted recovery measured on one H100 with the seeded synthetic 619 M weights: 2 of the 32 segments overlap their span.
# The synthetic joint is nearly flat, so a token costs about as much at any frame and the cheapest segment packs the whole
# caption into one or two frames, wherever the emissions happen to be cheapest (scripts/bench_align_captions.py measures
# a median confidence of -109 per frame).  The bar holds that measured rate; it is not an accuracy claim (DESIGN.md section 4).  On lattices where the
# tokens are likely only where they were said, the search finds every planted caption (PLANTED_BAR, checked on the CPU).
PLANTED_HITS_SYNTHETIC_619M = 2


def test_planted_recovery(full):
    """The caption is the window's own greedy tokens over frames [a, b): count the segments that overlap [a, b)."""
    cfg, sd, eng, enc, enc_len, labels, gframes = full
    caps, spans = _mid_captions(labels, gframes, enc_len)
    lab, ll = _packed(caps)
    seg = eng.align_segment(enc, enc_len, lab, ll)[0].cpu()
    hits = [int(seg[b, 0]) < z and int(seg[b, 1]) >= a for b, (a, z) in enumerate(spans)]
    print(f"planted recovery (619 M, synthetic weights): {sum(hits)}/{len(hits)} segments overlap their span")
    assert sum(hits) >= PLANTED_HITS_SYNTHETIC_619M


# ---------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def model(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    return asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=3)


def _program(model, n=6, seconds=6.0):
    """A program of n synthetic clips back to back and one caption per clip: its greedy transcript at its true times plus
    a 2 s delay."""
    from reazonspeech_b200.nemo import asr
    clips = [synth_clip(500 + i, seconds) for i in range(n)]
    heard = asr.transcribe_batch(model, [asr.audio_from_numpy(c, 16000) for c in clips], asr.TranscribeConfig(verbose=False))
    caps = [asr.Caption(i * seconds + 2.0, (i + 1) * seconds + 2.0, r.text or "a") for i, r in enumerate(heard)]
    caps.append(asr.Caption(n * seconds + 100.0, n * seconds + 101.0, "a"))   # outside the audio
    return asr.audio_from_numpy(np.concatenate(clips), 16000), caps


def test_align_captions_end_to_end(model):
    from reazonspeech_b200.nemo import asr
    audio, caps = _program(model)
    res = asr.align_captions(model, audio, caps, before=8.0, transcribe=True)
    assert len(res) == len(caps) and res[-1] is None
    found = [(c, r) for c, r in zip(caps, res) if r is not None]
    assert len(found) == len(caps) - 1
    for c, r in found:
        w0, w1 = max(c.start_seconds - 8.0, 0.0), min(c.end_seconds, audio.seconds)
        assert w0 <= r.start_seconds <= r.end_seconds <= w1 and r.caption is c and r.text == c.text
        secs = [w.seconds for w in r.subwords]
        assert secs == sorted(secs) and all(w0 <= s <= w1 + 0.5 for s in secs)      # a token may sit in the trailing pad
        assert r.log_likelihood >= r.score - 1e-3 and math.isfinite(r.confidence)
        assert isinstance(r.asr, str) and r.cer is not None
    again = asr.align_captions(model, audio, caps, before=8.0)
    for a, b in zip(res, again):
        assert (a is None and b is None) or (a.start_seconds, a.end_seconds, a.score) == (b.start_seconds, b.end_seconds, b.score)


def test_two_devices_equal_one(model, tiny_cfg):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from reazonspeech_b200.nemo import asr
    multi = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, devices=[0, 1])
    audio, caps = _program(model)
    for a, b in zip(asr.align_captions(model, audio, caps), asr.align_captions(multi, audio, caps)):
        assert (a is None and b is None) or (a.start_seconds, a.end_seconds, a.score, a.log_likelihood) == \
            (b.start_seconds, b.end_seconds, b.score, b.log_likelihood)


def test_cli_captions_writes_srt(tmp_path, monkeypatch, model, tiny_cfg):
    import sys
    import scipy.io.wavfile as wavfile
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr import cli
    audio, caps = _program(model, n=3)
    wav = tmp_path / "p.wav"
    wavfile.write(str(wav), 16000, (audio.waveform * 20000).astype(np.int16))
    tsv = tmp_path / "c.tsv"
    tsv.write_text("".join(f"{c.start_seconds:.3f}\t{c.end_seconds:.3f}\t{c.text}\n" for c in caps), encoding="utf-8")
    out = tmp_path / "p.srt"
    monkeypatch.setattr(sys.modules["reazonspeech_b200.nemo.asr.transcribe"], "load_model",
                        lambda **kw: asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0))
    cli.main([f"--captions={tsv}", "--before=8", "--to=srt", "-o", str(out), str(wav)])
    srt = out.read_text(encoding="utf-8")
    assert srt.count("-->") == 3 and all(c.text in srt.replace("\n", "") for c in caps[:3])
