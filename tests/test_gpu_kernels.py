"""Kernel-level parity tests (run on an H100 through the C ABI).

GEMM / LayerNorm are floating-point kernels, so their reference is a plain fp32 torch
evaluation of the same op on the same bf16-rounded inputs; every model stage is compared with
the CPU oracle (oracle/nemo_restated.py) on seeded inputs.  Tolerances are stated per test.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from reazonspeech_b200 import engine as E
from reazonspeech_b200.synth import synth_clip


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def pad_batch(waves, dev):
    L = max(len(w) for w in waves)
    x = torch.zeros(len(waves), L, dtype=torch.float32)
    for i, w in enumerate(waves):
        x[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    return x.to(dev), lens.to(dev)


def padded(w):
    """reference transcribe(): 0.5 s of silence both sides (audio.py:80-82)."""
    return np.pad(w, 8000)


# ------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 64, 128), (300, 128, 256), (1000, 1024, 256),
                                   (777, 640, 1024), (2048, 4096, 1024), (1552, 1024, 4096), (4100, 256, 2560)])
def test_gemm_bias_f32(tiny_engine, M, N, K):
    eng = tiny_engine
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    out = eng.gemm(a, w, bias, E.EPI_BIAS_F32, alpha=1.5)
    torch.cuda.synchronize()
    ref = 1.5 * (a.float() @ w.float().T + bias)
    err = (out - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), f"max abs err {err}"   # fp32 accumulate, order differs


@pytest.mark.parametrize("epi", [E.EPI_BIAS_BF16, E.EPI_BIAS_RELU_BF16, E.EPI_BIAS_SWISH_BF16, E.EPI_BIAS_GLU_BF16,
                                 E.EPI_RESID_F32, E.EPI_BIAS_F16])
def test_gemm_epilogues(tiny_engine, epi):
    eng = tiny_engine
    M, N, K = 517, 512, 256
    g = torch.Generator(device="cuda").manual_seed(epi)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    acc = a.float() @ w.float().T + bias
    if epi == E.EPI_RESID_F32:
        resid = torch.randn(M, N, device="cuda", generator=g)
        out = eng.gemm(a, w, bias, epi, resid=resid.clone(), alpha=0.5)
        ref = resid + 0.5 * acc
        tol = 2e-3
    elif epi == E.EPI_BIAS_GLU_BF16:
        d = N // 2
        idx = E.glu_interleave_index(d).cuda()
        out = eng.gemm(a, w[idx].contiguous(), bias[idx].contiguous(), epi).float()
        ref = acc[:, :d] * torch.sigmoid(acc[:, d:])
        tol = 1.2e-2          # bf16 output rounding (2^-8 relative) + fast sigmoid
    else:
        out = eng.gemm(a, w, bias, epi).float()
        ref = {E.EPI_BIAS_BF16: acc, E.EPI_BIAS_RELU_BF16: torch.relu(acc),
               E.EPI_BIAS_SWISH_BF16: torch.nn.functional.silu(acc), E.EPI_BIAS_F16: acc}[epi]
        tol = 2e-3 if epi == E.EPI_BIAS_F16 else 1.2e-2       # half: 2^-11 relative output rounding
    torch.cuda.synchronize()
    err = ((out - ref).abs() / (ref.abs() + 1.0)).max().item()
    assert err < tol, f"epilogue {epi}: max scaled err {err}"


@pytest.mark.parametrize("M,N,K,with_bias,alpha", [(640, 256, 1024, False, 1.0), (1000, 1024, 256, True, 0.5), (12416 // 8 + 3, 1024, 1024, True, 1.0)])
def test_gemm_resid_in_place(tiny_engine, M, N, K, with_bias, alpha):
    """x += alpha * (A W^T + b) in place (out == resid: each element is read and written by one lane) must equal the
    two-buffer result (resid != out) bit for bit: same fp32 operations, each element reduced once."""
    eng = tiny_engine
    g = torch.Generator(device="cuda").manual_seed(5 + M)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g) if with_bias else None
    x = torch.randn(M, N, device="cuda", generator=g)
    ref = x + alpha * (a.float() @ w.float().T + (bias if with_bias else 0.0))
    separate = eng.gemm(a, w, bias, E.EPI_RESID_F32, resid=x.clone(), alpha=alpha)
    guard = torch.full((64, N), 7.0, device="cuda")
    buf = torch.cat([x, guard])                       # rows past M must not be touched by the clipped last tile
    xin = buf[:M]
    eng.gemm(a, w, bias, E.EPI_RESID_F32, resid=xin, alpha=alpha, out=xin)
    torch.cuda.synchronize()
    assert (xin - ref).abs().max().item() < 2e-3
    assert torch.equal(xin, separate)
    assert torch.equal(buf[M:], guard)


@pytest.mark.parametrize("rows", [333, 12419])
def test_layernorm(tiny_engine, rows):
    """rows = 12 419: more rows than resident warps, so every warp walks several rows (the prefetch path of the persistent kernel)."""
    eng = tiny_engine
    for d in (256, 1024):
        g0 = torch.Generator(device="cuda").manual_seed(rows + d)
        x = torch.randn(rows, d, device="cuda", generator=g0) * 3 + 1
        g = torch.randn(d, device="cuda", generator=g0); b = torch.randn(d, device="cuda", generator=g0)
        ref = torch.nn.functional.layer_norm(x, (d,), g, b, eng.cfg.ln_eps)
        out = eng.layernorm(x, g, b, bf16_out=False)
        assert (out - ref).abs().max().item() < 2e-5
        outb = eng.layernorm(x, g, b, bf16_out=True).float()
        assert ((outb - ref).abs() / (ref.abs() + 1)).max().item() < 8e-3


# ------------------------------------------------------------------------------------ frontend
def test_logmel_vs_oracle(tiny_engine, tiny_cfg):
    """fp32 kernel vs torch.stft-based oracle; tolerance 1e-3 max-abs on the normalised features
    (the two FFTs differ in summation order; SURVEY.md A.6 suggests 1e-4, we report the measured value)."""
    from oracle import nemo_restated as O
    eng = tiny_engine
    waves = [padded(synth_clip(0, 1.7)), padded(synth_clip(1, 0.61)), padded(synth_clip(2, 3.003)), np.zeros(400, np.float32) + 0.01]
    x, lens = pad_batch(waves, "cuda")
    mel, mel_len = eng.log_mel(x, lens)
    torch.cuda.synchronize()
    worst = 0.0
    for i, w in enumerate(waves):
        ref = O.log_mel(torch.from_numpy(w), tiny_cfg).T          # [F, 80]
        F = ref.shape[0]
        assert int(mel_len[i]) == F
        got = mel[i, :F].cpu()
        worst = max(worst, (got - ref).abs().max().item())
        assert mel[i, F:].abs().max().item() == 0.0 if F < mel.shape[1] else True
    print("logmel max abs err", worst)
    assert worst < 1e-3


# ------------------------------------------------------------------------------------ encoder stages
def _mel_batch(eng, waves):
    x, lens = pad_batch(waves, "cuda")
    return eng.log_mel(x, lens)


@pytest.mark.parametrize("n_layers", [0, 1, 2])
def test_encoder_vs_oracle(tiny_engine, tiny_cfg, tiny_sd, n_layers):
    """bf16-GEMM engine vs fp32 oracle: relative L2 <= 2e-2 (SURVEY.md A.6) per utterance, and
    padding invariance: the padded batch must reproduce each utterance run alone."""
    from oracle import nemo_restated as O
    eng = tiny_engine
    waves = [padded(synth_clip(3, 2.0)), padded(synth_clip(4, 0.9)), padded(synth_clip(5, 3.2))]
    mel, mel_len = _mel_batch(eng, waves)
    enc, enc_len = eng.encode(mel, mel_len, n_layers=n_layers)
    torch.cuda.synchronize()
    for i, w in enumerate(waves):
        with torch.no_grad():
            ref = O.encoder(O.log_mel(torch.from_numpy(w), tiny_cfg), tiny_sd, tiny_cfg, n_layers=n_layers)
        T = ref.shape[0]
        assert int(enc_len[i]) == T
        got = enc[i, :T].cpu()
        r = _rel(got, ref)
        print(f"layers={n_layers} utt{i} T={T} rel-L2 {r:.4e}")
        assert r < 2e-2
        assert enc[i, T:].abs().max().item() == 0.0 if T < enc.shape[1] else True
        # alone
        m1, l1 = _mel_batch(eng, [w])
        e1, _ = eng.encode(m1, l1, n_layers=n_layers)
        assert _rel(e1[0, :T].cpu(), got) < 1e-5, "padding changed the result"


# ------------------------------------------------------------------------------------ decode
def test_greedy_teacher_forced(tiny_engine, tiny_cfg, tiny_sd):
    """The decode kernel alone (windowed, weights stationary, joint on wgmma): fed the ORACLE's encoder output, tokens and
    frames must be identical."""
    from oracle import nemo_restated as O
    eng = tiny_engine
    waves = [padded(synth_clip(6, 4.0)), padded(synth_clip(7, 2.5)), padded(synth_clip(8, 6.0))]
    refs, encs = [], []
    with torch.no_grad():
        for w in waves:
            e = O.encoder(O.log_mel(torch.from_numpy(w), tiny_cfg), tiny_sd, tiny_cfg)
            encs.append(e)
            refs.append(O.rnnt_greedy(e, tiny_sd, tiny_cfg, emulate=True))    # enc rounded to bf16 like the engine's joint.enc GEMM input
    T = max(e.shape[0] for e in encs)
    enc = torch.zeros(len(encs), T, tiny_cfg.d_model)
    for i, e in enumerate(encs):
        enc[i, : e.shape[0]] = e
    enc_len = torch.tensor([e.shape[0] for e in encs], dtype=torch.int32)
    tokens, frames, ntok = eng.greedy(enc.cuda(), enc_len.cuda())
    torch.cuda.synchronize()
    for i, r in enumerate(refs):
        n = int(ntok[i])
        print(f"utt{i}: {n} tokens (oracle {len(r.tokens)}), min margin {min(r.margins):.3e}")
        assert n == len(r.tokens)
        assert tokens[i, :n].cpu().tolist() == r.tokens
        assert frames[i, :n].cpu().tolist() == r.frames


from parity import check_decisions, decisions_from     # noqa: E402  (tests/ is on sys.path under pytest)


def test_end_to_end_tokens(tiny_engine, tiny_cfg, tiny_sd):
    """Whole path vs the oracle with the engine's bf16 storage points emulated: the engine's decision sequence is walked
    through the oracle teacher-forced to the LAST frame (tests/parity.py, noise-aware bar: every difference within 4 sigma of
    the storage noise the oracle measures on itself for the clip, no more of them than that noise predicts)."""
    from oracle import nemo_restated as O
    from parity import check_decisions_noise_aware
    eng = tiny_engine
    waves = [padded(synth_clip(10 + i, s)) for i, s in enumerate((3.0, 5.0, 1.2, 4.4))]
    x, lens = pad_batch(waves, "cuda")
    tokens, frames, ntok = eng.transcribe_device(x, lens)
    torch.cuda.synchronize()
    diffs, n_tok = [], 0
    for i, w in enumerate(waves):
        with torch.no_grad():
            mel = O.log_mel(torch.from_numpy(w), tiny_cfg)
            emu = O.encoder(mel, tiny_sd, tiny_cfg, emulate=True)
            ref = O.encoder(mel, tiny_sd, tiny_cfg)
        n = int(ntok[i])
        n_tok += n
        r = check_decisions_noise_aware(tokens[i, :n].cpu().tolist(), frames[i, :n].cpu().tolist(), emu, ref, tiny_sd, tiny_cfg, f"utt{i}")
        diffs.append((r["differences"], round(r["expected"], 1)))
    print(f"differing decisions per clip (observed, predicted by the storage noise): {diffs}")
    assert n_tok > 0


@pytest.mark.parametrize("B", [16, 19])
def test_host_entry_chunked_copies_equal_device_entry(tiny_engine, B):
    """rs_transcribe_batch overlaps its host->device copies with the frontend in utterance chunks (B >= 16):
    the result must be bit-identical to rs_transcribe_device on the same batch (ragged lengths, a batch size
    that does not divide into the chunk count)."""
    eng = tiny_engine
    waves = [padded(synth_clip(60 + i, 0.6 + 0.37 * (i % 7))) for i in range(B)]
    x, lens = pad_batch(waves, "cpu")
    th, fh, nh = eng.transcribe_host(x.pin_memory(), lens)
    td, fd, nd = eng.transcribe_device(x.cuda(), lens.cuda())
    torch.cuda.synchronize()
    assert torch.equal(nh, nd.cpu())
    for b in range(B):
        n = int(nh[b])
        assert torch.equal(th[b, :n], td[b, :n].cpu()) and torch.equal(fh[b, :n], fd[b, :n].cpu())
    assert int(nh.sum()) > 0


def test_long_form_clip_in_one_call(tiny_engine, tiny_cfg, tiny_sd):
    """SURVEY.md section 8(f).2: the reference feeds audio of any length to the model in one shot (transcribe.py:44-53,
    relying on local attention).  A 150 s clip (1 882 encoder frames = 15 query tiles of the tensor-core attention,
    ~470 decode windows) goes through the engine in one call, next to a short one: encoder within 2e-2 relative L2 of the
    fp32 oracle, decision sequence walked through the oracle to the last frame (tests/parity.py)."""
    from oracle import nemo_restated as O
    eng = tiny_engine
    waves = [padded(synth_clip(90, 150.0)), padded(synth_clip(91, 2.0))]
    x, lens = pad_batch(waves, "cuda")
    mel, mel_len = eng.log_mel(x, lens)
    enc, enc_len = eng.encode(mel, mel_len)
    tokens, frames, ntok = eng.transcribe_device(x, lens)
    torch.cuda.synchronize()
    for i, w in enumerate(waves):
        with torch.no_grad():
            ref = O.encoder(O.log_mel(torch.from_numpy(w), tiny_cfg), tiny_sd, tiny_cfg)
            emu = O.encoder(O.log_mel(torch.from_numpy(w), tiny_cfg), tiny_sd, tiny_cfg, emulate=True)
        T = ref.shape[0]
        assert int(enc_len[i]) == T == tiny_cfg.enc_frames(len(w))
        r = _rel(enc[i, :T].cpu(), ref)
        n = int(ntok[i])
        assert r < 2e-2
        from parity import check_decisions_noise_aware             # whole path: storage noise measured in the oracle itself
        res = check_decisions_noise_aware(tokens[i, :n].cpu().tolist(), frames[i, :n].cpu().tolist(), emu, ref, tiny_sd, tiny_cfg, f"utt{i}")
        print(f"utt{i}: T={T}, encoder rel-L2 {r:.3e}, {n} tokens, {res['differences']} of {res['decisions']} decisions differ "
              f"(storage noise sigma {res['sigma']:.2e} -> {res['expected']:.1f} expected)")


@pytest.mark.parametrize("L_pad", [0, 3])
def test_pcm16_ingest_equals_float_path(tiny_engine, L_pad):
    """rs_transcribe_device_pcm16 / rs_transcribe_batch_pcm16 (int16 samples scaled by 2^-15 inside the log-mel kernel's staging
    load) against the float entry points on the converted samples: the same values in, so tokens and frames must be
    bit-identical -- with rows that allow the 8-byte vector load (L % 4 == 0) and rows that force the scalar path."""
    eng = tiny_engine
    waves = [np.round(padded(synth_clip(150 + i, 0.9 + 0.8 * i)) * 32767.0).astype(np.int16) for i in range(5)]
    L = max(len(w) for w in waves)
    L = ((L + 3) & ~3) + L_pad
    x16 = torch.zeros(len(waves), L, dtype=torch.int16)
    for i, w in enumerate(waves):
        x16[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    xf = x16.to(torch.float32) / 32768.0
    tf, ff, nf = [a.cpu() for a in eng.transcribe_device(xf.cuda(), lens.cuda())]
    ti, fi, ni = [a.cpu() for a in eng.transcribe_device(x16.cuda(), lens.cuda())]
    th, fh, nh = eng.transcribe_host(x16.pin_memory(), lens)
    assert int(nf.sum()) > 0 and torch.equal(nf, ni) and torch.equal(nf, nh)
    for b in range(len(waves)):
        n = int(nf[b])
        assert torch.equal(tf[b, :n], ti[b, :n]) and torch.equal(ff[b, :n], fi[b, :n])
        assert torch.equal(tf[b, :n], th[b, :n]) and torch.equal(ff[b, :n], fh[b, :n])
