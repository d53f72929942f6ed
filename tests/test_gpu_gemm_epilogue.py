"""The wgmma GEMM's epilogue (gemm_wgmma.cu): every output is written through shared memory by TMA stores, the residual
one by a TMA f32 add into out.  Each epilogue is checked bit for bit against torch's rounding of the same launch's
RS_EPI_BIAS_F32 result, so the only arithmetic under test is the epilogue's own.

Shapes marked 256 take the 128 x 256 instance on a 132-SM H100, the others the 128 x 64 one.  The K = 64 launches run a
one-k-block main loop over many tiles per CTA: the epilogue buffers are rewritten as fast as the stores can drain, so a
reuse race shows up as wrong values.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from reazonspeech_b200 import engine as E

SHAPES = [(12672, 1024, 256),    # 256: 99 M-tiles
          (296, 640, 128),       # 64: partial last M tile
          (40000, 1024, 64),     # 256: ~9 tiles per CTA, one k-block each
          (40000, 96, 64)]       # 64: ~5 tiles per CTA, partial last W tile


def _operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    return a, w, bias, g


def _bits_equal(x, y):
    return torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32))


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_two_byte_outputs_round_the_f32_result(tiny_engine, M, N, K):
    a, w, bias, _ = _operands(M, N, K, M + N)
    f = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_F32, alpha=1.0)
    bf = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_BF16)
    relu = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_RELU_BF16)
    half = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_F16)
    torch.cuda.synchronize()
    assert torch.equal(bf.view(torch.int16), f.to(torch.bfloat16).view(torch.int16))
    assert torch.equal(relu, torch.relu(f).to(torch.bfloat16))          # values: relu may give either zero
    assert torch.equal(half.view(torch.int16), f.to(torch.float16).view(torch.int16))


@pytest.mark.parametrize("in_place", [True, False])
@pytest.mark.parametrize("alpha", [0.5, 1.0])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_residual_add_is_x_plus_bias_f32(tiny_engine, M, N, K, alpha, in_place):
    """out = x + RS_EPI_BIAS_F32(alpha), rounded once after the rounded product (exact for a power-of-two alpha).  Every
    seventh row of x is subnormal, and eight W rows and their biases are zero, so those columns add +0 to x: the TMA f32
    add keeps subnormal residuals and subnormal sums, it does not flush them to zero."""
    a, w, bias, g = _operands(M, N, K, 3 * M + N)
    w[5:13] = 0
    bias[5:13] = 0
    x = torch.randn(M, N, device="cuda", generator=g)
    x[::7] *= 1e-39
    assert (x[::7].abs() < torch.finfo(torch.float32).tiny).all()
    f = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_F32, alpha=alpha)
    if in_place:
        out = x.clone()
        tiny_engine.gemm(a, w, bias, E.EPI_RESID_F32, resid=out, alpha=alpha, out=out)
    else:
        out = torch.full_like(x, 7.0)
        tiny_engine.gemm(a, w, bias, E.EPI_RESID_F32, resid=x, alpha=alpha, out=out)
    torch.cuda.synchronize()
    assert _bits_equal(out[:, 5:13], x[:, 5:13])
    assert _bits_equal(out, x + f)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_glu_and_qkv_vt_round_the_f32_result(tiny_engine, M, N, K):
    """GLU: the f32 values and gates give the same products as the fused epilogue only up to the fast sigmoid, so the
    check is against torch within bf16 rounding; V^T is the transposed bf16 rounding of the f32 result, bit for bit."""
    a, w, bias, _ = _operands(M, N, K, 5 * M + N)
    d = N // 2
    idx = E.glu_interleave_index(d).cuda()
    glu = tiny_engine.gemm(a, w[idx].contiguous(), bias[idx].contiguous(), E.EPI_BIAS_GLU_BF16).float()
    split = N - 32 * max(1, N // 96)
    out = torch.full((M, N), 3.0, dtype=torch.bfloat16, device="cuda")
    out2 = torch.full((N - split, M + 40), 5.0, dtype=torch.bfloat16, device="cuda")
    tiny_engine.gemm(a, w, bias, E.EPI_QKV_VT, out=out, out2=out2, split=split)
    f = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_F32, alpha=1.0)
    torch.cuda.synchronize()
    ref = f[:, :d] * torch.sigmoid(f[:, d:])
    assert ((glu - ref).abs() / (ref.abs() + 1.0)).max().item() < 1.2e-2
    assert torch.equal(out[:, :split].view(torch.int16), f[:, :split].to(torch.bfloat16).view(torch.int16))
    assert torch.equal(out2[:, :M].view(torch.int16), f[:, split:].T.to(torch.bfloat16).view(torch.int16))
    assert torch.all(out[:, split:] == 3.0) and torch.all(out2[:, M:] == 5.0)
