"""Forced alignment on the GPU (csrc/align.cu) against the float64 oracle (tests/align_oracle.py): the lattice seam, the DP on
the kernel's own lattice, the whole path, consistency with the greedy decode, edge cases, the Python / C surfaces, and that
nothing else changes.  The lattice bar (2e-4) is checked on the CPU to lie 3x below the error of listed mis-implementations
(test_align_cpu.py::test_lattice_bar_separates_mis_implementations)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import align_oracle as A
from reazonspeech_b200.synth import synth_clip

pytestmark = pytest.mark.gpu

LATTICE_BAR = 2e-4
NAN_FILL = float("nan")


def _inputs(cfg, T_lens, labels, seed, T_max=None):
    g = torch.Generator().manual_seed(seed)
    T_max = T_max or max(T_lens)
    enc = torch.randn(len(T_lens), T_max, cfg.d_model, generator=g)
    for b, n in enumerate(T_lens):
        enc[b, n:] = 0
    U_max = max([len(x) for x in labels] + [1])
    lab = torch.zeros(len(labels), U_max, dtype=torch.int32)
    for b, x in enumerate(labels):
        lab[b, : len(x)] = torch.tensor(x, dtype=torch.int32)
    return enc, torch.tensor(T_lens, dtype=torch.int32), lab, torch.tensor([len(x) for x in labels], dtype=torch.int32)


def _random_labels(cfg, lens, seed):
    rng = np.random.default_rng(seed)
    return [[int(k) for k in rng.integers(0, cfg.vocab_size, n)] for n in lens]


def _lattice(eng, enc, T, lab, ll):
    return [x.cpu() for x in eng.align_lattice(enc.cuda().contiguous(), T.cuda(), lab.cuda(), ll.cuda())]


def _align(eng, enc, T, lab, ll):
    return [x.cpu() for x in eng.align(enc.cuda().contiguous(), T.cuda(), lab.cuda(), ll.cuda())]


def _ref_lattice_gpu(enc_b, labels, sd, cfg, chunk=32):
    """float64 lattice of one utterance computed with torch on the GPU in frame chunks (the production joint is 3001 x 640
    per cell; the host would take minutes per 30 s clip)."""
    _, pp = A.predictor(labels, sd, cfg)
    ep = A.enc_proj(enc_b, sd)
    W = sd["joint.joint_net.2.weight"].double().cuda(); b = sd["joint.joint_net.2.bias"].double().cuda()
    ppd = pp.double().cuda()
    lpb, lpe = [], []
    lab = torch.tensor(labels, dtype=torch.long, device="cuda")
    U = len(labels)
    for t0 in range(0, ep.shape[0], chunk):
        a = torch.relu(ep[t0:t0 + chunk].double().cuda()[:, None, :] + ppd[None])
        lsm = torch.log_softmax(a @ W.T + b, -1)
        lpb.append(lsm[:, :, cfg.blank].cpu())
        e = torch.full(lsm.shape[:2], -math.inf, dtype=torch.float64, device="cuda")
        if U:
            e[:, :U] = torch.gather(lsm[:, :U, :], 2, lab[None, :, None].expand(lsm.shape[0], U, 1))[..., 0]
        lpe.append(e.cpu())
    return torch.cat(lpb).numpy(), torch.cat(lpe).numpy()


def _check_lattice(lpb, lpe, ref_b, ref_e, T, U, tag):
    db = np.abs(lpb[:T, : U + 1].double().numpy() - ref_b).max()
    de = np.abs(lpe[:T, :U].double().numpy() - ref_e[:, :U]).max() if U else 0.0
    assert np.all(np.isneginf(lpe[:T, U].numpy())), tag
    assert max(db, de) <= LATTICE_BAR, f"{tag}: lattice error blank {db:.2e} emit {de:.2e}"
    return max(db, de)


# ---------------------------------------------------------------- tiny model
TINY_T = [20, 1, 13, 7, 30, 16]
TINY_U = [6, 3, 0, 12, 9, 1]          # U > T (7 frames, 12 labels), a single frame, U = 0


def test_lattice_seam_vs_float64_tiny(tiny_engine, tiny_cfg, tiny_sd):
    labels = _random_labels(tiny_cfg, TINY_U, 1)
    enc, T, lab, ll = _inputs(tiny_cfg, TINY_T, labels, 2)
    lpb, lpe = _lattice(tiny_engine, enc, T, lab, ll)
    worst = 0.0
    for b in range(len(TINY_T)):
        Tb, Ub = TINY_T[b], TINY_U[b]
        rb, re = A.lattice(enc[b], labels[b], tiny_sd, tiny_cfg, T=Tb)
        worst = max(worst, _check_lattice(lpb[b], lpe[b], rb, re, Tb, Ub, f"b={b}"))
        assert torch.isnan(lpb[b, Tb:]).all() and torch.isnan(lpb[b, :, Ub + 1:]).all(), f"b={b}: a cell outside was written"
        assert torch.isnan(lpe[b, Tb:]).all() and torch.isnan(lpe[b, :, Ub + 1:]).all()
    print(f"tiny lattice: max |error| {worst:.2e}")


def test_lattice_batch_invariance(tiny_engine, tiny_cfg):
    labels = _random_labels(tiny_cfg, TINY_U, 3)
    enc, T, lab, ll = _inputs(tiny_cfg, TINY_T, labels, 4)
    lpb, lpe = _lattice(tiny_engine, enc, T, lab, ll)
    perm = [3, 0, 5, 1, 4, 2]
    pb, pe = _lattice(tiny_engine, enc[perm], T[perm], lab[perm], ll[perm])
    for i, b in enumerate(perm):
        Tb, Ub = TINY_T[b], TINY_U[b]
        eb, ee = _lattice(tiny_engine, enc[b:b + 1, :Tb], T[b:b + 1], lab[b:b + 1, :max(Ub, 1)], ll[b:b + 1])
        for x in (pb[i], eb[0]):
            assert torch.equal(x[:Tb, : Ub + 1], lpb[b, :Tb, : Ub + 1])
        for x in (pe[i], ee[0]):
            assert torch.equal(x[:Tb, : Ub + 1], lpe[b, :Tb, : Ub + 1])


def _check_dp(eng, enc, T, lab, ll, T_lens, U_lens, tag):
    """The DP on the kernel's own lattice vs the float64 recursions on the same (fp32) lattice."""
    lpb, lpe = _lattice(eng, enc, T, lab, ll)
    frames, token_lp, vit, ll_out = _align(eng, enc, T, lab, ll)
    for b in range(len(T_lens)):
        Tb, Ub = T_lens[b], U_lens[b]
        r = A.align(lpb[b].double().numpy(), lpe[b].double().numpy(), Tb, Ub)
        assert abs(float(vit[b]) - r["viterbi"]) <= 1e-4 * abs(r["viterbi"]) + 1e-5, f"{tag} b={b}"
        assert abs(float(ll_out[b]) - r["loglik"]) <= 1e-4 * abs(r["loglik"]) + 1e-5, f"{tag} b={b}"
        fr = frames[b, :Ub].numpy()
        if fr.tolist() != r["frames"].tolist():
            assert r["path_margin"] <= 1e-4, f"{tag} b={b}: frames differ with a decision margin {r['path_margin']:.2e}"
        assert np.all(np.diff(fr) >= 0) and (Ub == 0 or (fr[0] >= 0 and fr[-1] < Tb)), f"{tag} b={b}"
        assert torch.equal(token_lp[b, :Ub], lpe[b, fr, np.arange(Ub)]), f"{tag} b={b}"
        assert (frames[b, Ub:] == -1).all() and torch.isnan(token_lp[b, Ub:]).all()


def test_dp_on_the_kernels_lattice_tiny(tiny_engine, tiny_cfg):
    labels = _random_labels(tiny_cfg, TINY_U, 5)
    enc, T, lab, ll = _inputs(tiny_cfg, TINY_T, labels, 6)
    _check_dp(tiny_engine, enc, T, lab, ll, TINY_T, TINY_U, "tiny")


def test_dp_wider_than_the_block(tiny_engine, tiny_cfg):
    """U_max + 1 above the DP's 256 threads, U > T and T > U in one batch."""
    T_lens, U_lens = [120, 300, 40], [300, 90, 0]
    labels = _random_labels(tiny_cfg, U_lens, 7)
    enc, T, lab, ll = _inputs(tiny_cfg, T_lens, labels, 8)
    _check_dp(tiny_engine, enc, T, lab, ll, T_lens, U_lens, "wide")


def test_whole_path_vs_float64_oracle_tiny(tiny_engine, tiny_cfg, tiny_sd):
    """rs_rnnt_align on an encoder output vs the all-float64 oracle (lattice and recursions), labels = the greedy transcript."""
    enc, T, _, _ = _inputs(tiny_cfg, TINY_T, [[]] * len(TINY_T), 9)
    tk, fr, nt = [x.cpu() for x in tiny_engine.greedy(enc.cuda().contiguous(), T.cuda())]
    labels = [tk[b, : int(nt[b])].tolist() for b in range(len(TINY_T))]
    _, _, lab, ll = _inputs(tiny_cfg, TINY_T, labels, 9)
    frames, _, vit, lo = _align(tiny_engine, enc, T, lab, ll)
    worst = 0.0
    for b, Tb in enumerate(TINY_T):
        rb, re = A.lattice(enc[b], labels[b], tiny_sd, tiny_cfg, T=Tb)
        r = A.align(rb, re, Tb, len(labels[b]))
        worst = max(worst, abs(float(vit[b]) - r["viterbi"]), abs(float(lo[b]) - r["loglik"]))
    print(f"tiny whole path: max |error| of viterbi / loglik {worst:.2e}")
    assert worst <= 1e-2


def test_edge_cases_and_bad_labels(tiny_engine, tiny_cfg):
    V = tiny_cfg.vocab_size
    labels = [[1, 2, 3], [4, V, 5], [6], [], [7, -1]]
    T_lens = [9, 9, 9, 5, 9]
    enc, T, lab, ll = _inputs(tiny_cfg, T_lens, labels, 10)
    lpb, _ = _lattice(tiny_engine, enc, T, lab, ll)
    frames, token_lp, vit, lo = _align(tiny_engine, enc, T, lab, ll)
    for b in (1, 4):
        assert math.isnan(float(vit[b])) and math.isnan(float(lo[b])) and (frames[b] == -1).all() and torch.isnan(token_lp[b]).all()
    # U = 0: loglik = viterbi = the sum of lp_blank along the bottom row
    s = float(lpb[3, :5, 0].double().sum())
    assert abs(float(lo[3]) - s) < 1e-4 and abs(float(vit[3]) - s) < 1e-4
    # the other utterances are unaffected by the bad ones
    good = [0, 2, 3]
    f2, t2, v2, l2 = _align(tiny_engine, enc[good], T[good], lab[good], ll[good])
    assert torch.equal(f2, frames[good]) and torch.equal(v2, vit[good]) and torch.equal(l2, lo[good])
    assert torch.equal(t2[~torch.isnan(t2)], token_lp[good][~torch.isnan(token_lp[good])])


def test_bad_host_arguments_are_rejected_before_any_launch(tiny_engine, tiny_cfg):
    eng = tiny_engine
    enc, T, lab, ll = _inputs(tiny_cfg, [5], [[1, 2]], 11)
    enc, T, lab, ll = enc.cuda(), T.cuda(), lab.cuda(), ll.cuda()
    out = [torch.zeros(2, dtype=torch.int32, device="cuda"), torch.zeros(2, device="cuda"), torch.zeros(1, device="cuda"),
           torch.zeros(1, device="cuda")]
    p = [x.data_ptr() for x in out]
    n0 = eng.launch_count
    for args in ((0, 5, 2), (1, 0, 2), (1, 5, 0)):
        B, Tm, U = args
        assert eng.lib.rs_rnnt_align(eng.h, enc.data_ptr(), T.data_ptr(), B, Tm, lab.data_ptr(), ll.data_ptr(), U, *p, None) == -1
    assert eng.lib.rs_rnnt_align(eng.h, None, T.data_ptr(), 1, 5, lab.data_ptr(), ll.data_ptr(), 2, *p, None) == -1
    assert eng.lib.rs_rnnt_align(eng.h, enc.data_ptr(), T.data_ptr(), 1, 5, lab.data_ptr(), ll.data_ptr(), 2, p[0], None, p[2], p[3], None) == -1
    assert eng.lib.rs_rnnt_align_lattice(eng.h, enc.data_ptr(), T.data_ptr(), 1, 5, lab.data_ptr(), ll.data_ptr(), 2, p[1], None, None) == -1
    assert eng.launch_count == n0


def test_off_means_off(tiny_engine, tiny_cfg):
    """Alignment leaves the workspace size and every transcription exactly as they were."""
    eng = tiny_engine
    n = C.c_size_t(0)
    eng.lib.rs_workspace_bytes(eng.h, 8, 48000, C.byref(n))
    wav = torch.from_numpy(np.stack([synth_clip(200 + i, 3.0) for i in range(4)])).float().cuda()
    lens = torch.full((4,), wav.shape[1], dtype=torch.int32, device="cuda")
    before = [x.cpu() for x in eng.transcribe_device(wav, lens)]
    enc, T, lab, ll = _inputs(tiny_cfg, TINY_T, _random_labels(tiny_cfg, TINY_U, 12), 12)
    _align(eng, enc, T, lab, ll)
    after = [x.cpu() for x in eng.transcribe_device(wav, lens)]
    m = C.c_size_t(0)
    eng.lib.rs_workspace_bytes(eng.h, 8, 48000, C.byref(m))
    assert n.value == m.value
    for x, y in zip(before, after):
        assert torch.equal(x, y)


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
    labels = [tk[b, : int(nt[b])].tolist() for b in range(32)]
    gframes = [fr[b, : int(nt[b])].tolist() for b in range(32)]
    return cfg, sd, eng, enc, enc_len, labels, gframes


def _packed(labels, device="cuda"):
    U = max([len(x) for x in labels] + [1])
    lab = torch.zeros(len(labels), U, dtype=torch.int32)
    for b, x in enumerate(labels):
        lab[b, : len(x)] = torch.tensor(x, dtype=torch.int32)
    return lab.to(device), torch.tensor([len(x) for x in labels], dtype=torch.int32, device=device)


def test_bench_geometry_lattice_dp_and_consistency(full):
    cfg, sd, eng, enc, enc_len, labels, gframes = full
    lab, ll = _packed(labels)
    lpb, lpe = [x.cpu() for x in eng.align_lattice(enc, enc_len, lab, ll)]
    frames, token_lp, vit, lo = [x.cpu() for x in eng.align(enc, enc_len, lab, ll)]
    n = [len(x) for x in labels]
    assert min(n) > 0
    picks = sorted({int(np.argmin(n)), int(np.argmax(n)), 5, 17})
    worst = 0.0
    for b in picks:                                                # every cell of 4 clips against float64
        Tb = int(enc_len[b])
        rb, re = _ref_lattice_gpu(enc[b, :Tb].cpu(), labels[b], sd, cfg)
        worst = max(worst, _check_lattice(lpb[b], lpe[b], rb, re, Tb, n[b], f"clip {b}"))
    print(f"bench lattice (clips {picks}): max |error| {worst:.2e}")
    for b in range(32):                                            # invariants on all 32
        Tb, Ub = int(enc_len[b]), n[b]
        r = A.align(lpb[b].double().numpy(), lpe[b].double().numpy(), Tb, Ub)
        assert abs(float(vit[b]) - r["viterbi"]) <= 1e-4 * abs(r["viterbi"]) and abs(float(lo[b]) - r["loglik"]) <= 1e-4 * abs(r["loglik"])
        fr = frames[b, :Ub].numpy()
        assert np.all(np.diff(fr) >= 0) and fr[0] >= 0 and fr[-1] < Tb
        assert float(lo[b]) >= float(vit[b]) - 1e-3
        # the greedy tokens at their greedy frames are a lattice path (the lattice has no max_symbols cap): Viterbi >= its score
        g = 0.0
        t = 0
        for u, f in enumerate(gframes[b]):
            g += float(lpb[b, t:f, u].double().sum()) + float(lpe[b, f, u]); t = f
        g += float(lpb[b, t:Tb, Ub].double().sum())
        assert float(vit[b]) >= g - 1e-3, f"clip {b}: Viterbi {float(vit[b])} below the greedy path's {g}"


def test_long_form_clip(full):
    cfg, sd, eng, *_ = full
    w = torch.from_numpy(np.pad(synth_clip(95, 150.0), 8000)).float()[None].cuda()
    lens = torch.tensor([w.shape[1]], dtype=torch.int32, device="cuda")
    enc, enc_len = eng.encode(*eng.log_mel(w, lens))
    tk, fr, nt = [a.cpu() for a in eng.greedy(enc, enc_len)]
    labels = [tk[0, : int(nt[0])].tolist()]
    lab, ll = _packed(labels)
    lpb, lpe = [x.cpu() for x in eng.align_lattice(enc, enc_len, lab, ll)]
    frames, token_lp, vit, lo = [x.cpu() for x in eng.align(enc, enc_len, lab, ll)]
    Tb, Ub = int(enc_len[0]), len(labels[0])
    r = A.align(lpb[0].double().numpy(), lpe[0].double().numpy(), Tb, Ub)
    assert abs(float(lo[0]) - r["loglik"]) <= 1e-4 * abs(r["loglik"]) and abs(float(vit[0]) - r["viterbi"]) <= 1e-4 * abs(r["viterbi"])
    fr0 = frames[0, :Ub].numpy()
    assert Ub == 0 or (np.all(np.diff(fr0) >= 0) and fr0[-1] < Tb)


# ---------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def model(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    return asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=3)


def _audios():
    from reazonspeech_b200.nemo import asr
    return [asr.audio_from_numpy(synth_clip(300 + i, s), 16000) for i, s in enumerate((2.0, 0.8, 3.3, 1.5, 2.4))]


def test_align_and_align_batch(model, tiny_cfg):
    from reazonspeech_b200.nemo import asr
    audios = _audios()
    cfgv = asr.TranscribeConfig(verbose=False)
    heard = asr.transcribe_batch(model, audios, asr.TranscribeConfig(verbose=False, raw_hypothesis=True))
    texts = [model.tokenizer.ids_to_text([60 + i, 70, 2]) for i in range(len(audios))]
    texts[1] = heard[1].hypothesis.y_sequence.tolist()[1:] or [61]            # token ids, not a str
    batch = asr.align_batch(model, audios, texts, cfgv)
    for i, (a, t, r) in enumerate(zip(audios, texts, batch)):
        ids = model.tokenizer.sentence_to_ids(t) if isinstance(t, str) else t
        kept = [k for k in ids if model.tokenizer.ids_to_text([k])]
        assert [w.token_id for w in r.subwords] == kept, i
        secs = [w.seconds for w in r.subwords]
        # times as a transcription's: the clip plus the 0.5 s of padding behind it
        assert secs == sorted(secs) and all(0 <= s <= a.seconds + 0.5 for s in secs)
        assert all(0 <= g.start_seconds <= g.end_seconds <= a.seconds + 0.6 for g in r.segments)
        h = r.hypothesis
        assert h.log_likelihood >= h.score and len(h.token_logprob) == len(ids) and all(x <= 0 for x in h.token_logprob)
        one = asr.align(model, a, t, cfgv)
        assert one.hypothesis.timestamp == h.timestamp and one.hypothesis.score == h.score and one.text == r.text


def test_two_device_alignment_equals_one(model, tiny_cfg):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from reazonspeech_b200.nemo import asr
    multi = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, devices=[0, 1])
    audios = _audios() * 2
    texts = [[60 + i, 70, 2] for i in range(len(audios))]
    one = asr.align_batch(model, audios, texts)
    two = asr.align_batch(multi, audios, texts)
    for a, b in zip(one, two):
        assert a.hypothesis.timestamp == b.hypothesis.timestamp and a.hypothesis.log_likelihood == b.hypothesis.log_likelihood


def test_cli_text_writes_srt(tmp_path, monkeypatch, tiny_cfg):
    import scipy.io.wavfile as wavfile
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr import cli
    wav = tmp_path / "a.wav"
    wavfile.write(str(wav), 16000, (synth_clip(400, 2.0) * 20000).astype(np.int16))
    tok = asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0).tokenizer
    text = tmp_path / "t.txt"
    text.write_text(tok.ids_to_text([60, 61, 2, 62]) + "\n", encoding="utf-8")
    out = tmp_path / "a.srt"
    import sys
    monkeypatch.setattr(sys.modules["reazonspeech_b200.nemo.asr.transcribe"], "load_model",
                        lambda **kw: asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0))
    cli.main([f"--text={text}", "--to=srt", "-o", str(out), str(wav)])
    srt = out.read_text(encoding="utf-8")
    assert "-->" in srt and tok.ids_to_text([60, 61, 2]) in srt.replace("\n", "")
