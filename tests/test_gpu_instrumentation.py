"""The engine's measurement aids on one step of the tiny model: the launch counter, the per-kernel and GEMM event logs, and
the stage events of the host-buffer path; the launch count of an ALSD beam search."""
import pytest
import torch

pytestmark = pytest.mark.gpu

B, L = 2, 48000


def _conv_len(n):
    return (n - 1) // 2 + 1 if n > 0 else 0


def _batch(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    wav = 0.1 * torch.randn(n, L, generator=g)
    lens = torch.full((n,), L, dtype=torch.int32)
    lens[0] = L // 2
    return wav, lens


@pytest.fixture
def engine(tiny_cfg, tiny_sd):
    """A fresh engine with its workspace sized and every kernel loaded by one step."""
    from reazonspeech_b200.engine import Engine
    eng = Engine(tiny_cfg, tiny_sd, "cuda:0")
    wav, lens = _batch(B)
    eng.transcribe_device(wav.cuda(), lens.cuda())
    torch.cuda.synchronize()
    return eng


def test_launch_count_per_step(engine, tiny_cfg):
    wav, lens = _batch(B)
    wav, lens = wav.cuda(), lens.cuda()
    n0 = engine.launch_count
    engine.transcribe_device(wav, lens)
    a = 2 if tiny_cfg.global_tokens > 0 else 1          # the global-token row kernel follows the local attention
    assert engine.launch_count - n0 == 13 + tiny_cfg.n_layers * (13 + a)


def test_launch_count_of_alsd(tiny_cfg, tiny_sd):
    """Eight launches per anti-diagonal step (rows, GEMM, reduce, select, lstm_in, GEMM, cell, GEMM) and eight around them
    (f32 -> bf16, joint.enc GEMM, init, the first predictor pass, output)."""
    from reazonspeech_b200.engine import Engine
    eng = Engine(tiny_cfg, tiny_sd, "cuda:0", alsd=True)
    wav, lens = _batch(B)
    mel, mel_len = eng.log_mel(wav.cuda(), lens.cuda())
    enc, enc_len = eng.encode(mel, mel_len)
    eng.alsd(enc, enc_len, beam=4)                      # loads every kernel
    torch.cuda.synchronize()
    eng.kernel_timing(True)
    n0 = eng.launch_count
    eng.alsd(enc, enc_len, beam=4)
    kt = eng.kernel_timing()
    eng.kernel_timing(False)
    steps = kt["alsd_launch_rows"][0]
    assert steps > 0
    assert eng.launch_count - n0 == 8 + 8 * steps


def test_kernel_timing_of_one_step(engine, tiny_cfg):
    wav, lens = _batch(B)
    wav, lens = wav.cuda(), lens.cuda()
    engine.kernel_timing(True)
    engine.transcribe_device(wav, lens)
    kt = engine.kernel_timing()
    engine.kernel_timing(False)
    for name in ("launch_logmel_fused", "launch_layernorm", "launch_conv_dw", "launch_attention_tc", "launch_rnnt_greedy_spec"):
        assert name in kt, sorted(kt)
    assert kt["launch_layernorm"][0] == 4 * tiny_cfg.n_layers + 1
    assert all(ms > 0 for _, ms in kt.values()), kt


def test_gemm_timing_of_one_step(engine, tiny_cfg):
    c = tiny_cfg
    wav, lens = _batch(B)
    wav, lens = wav.cuda(), lens.cuda()
    engine.enable_gemm_timing(True)
    engine.transcribe_device(wav, lens)
    ms, flops, n = engine.gemm_timing()
    engine.enable_gemm_timing(False)
    T2 = _conv_len(_conv_len(L // c.n_window_stride + 1))
    F2 = _conv_len(_conv_len(c.n_mels))
    F3 = _conv_len(F2)
    T3 = engine.enc_frames(L)
    M, C, d = B * T3, c.sub_channels, c.d_model
    layer = [(M, c.d_ff, d), (M, d, c.d_ff), (M, 3 * d, d), (M, d, d), (M, 2 * d, d), (M, d, d), (M, c.d_ff, d), (M, d, c.d_ff)]
    shapes = [(B * T2 * F2, C, C), (B * T3 * F3, C, C), (M, d, F3 * C)] + layer * c.n_layers + [(M, c.joint_hidden, d)]
    assert n == len(shapes) == 8 * c.n_layers + 4
    assert flops == sum(2.0 * m * nn * k for m, nn, k in shapes)
    assert ms > 0


def test_stage_times_on_the_chunked_host_path(tiny_cfg, tiny_sd):
    """16 utterances take the chunked host-to-device copy; on a fresh engine every stage event comes from this call."""
    from reazonspeech_b200.engine import Engine
    eng = Engine(tiny_cfg, tiny_sd, "cuda:0")
    wav, lens = _batch(16, seed=1)
    eng.enable_stage_timing(True)
    eng.transcribe_host(wav.pin_memory(), lens)
    st = eng.stage_times_ms()
    eng.enable_stage_timing(False)
    assert len(st) == 5 and all(v > 0 for v in st.values()), st
