"""Geometry of the two instances of the wgmma GEMM (gemm_wgmma.cu): odd M-tile counts, partial last W tiles, the QKV
split inside a 256-wide tile, guard rows past M, and the row invariance between the 128 x 256 instance and the
128 x 64 one that small launches use.

launch_gemm takes the 256-wide instance when N % 256 == 0 and ceil(M / 128) * N / 256 tiles give every SM one; the
shapes marked 256 do so on a 132-SM H100 (the row-invariance case runs one launch of each instance).
References: fp32 torch on the same bf16 inputs, with the tolerances of test_gpu_kernels.py.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from reazonspeech_b200 import engine as E


def _operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    return a, w, bias


def _check_f32(out, ref):
    err = (out - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), f"max abs err {err}"


@pytest.mark.parametrize("M,N,K", [(100, 33792, 64), (300, 11264, 128), (12672, 1024, 256),   # 256: 1, 3, 99 M-tiles
                                   (40000, 64, 256), (40000, 96, 256), (12544, 640, 1024), (12544, 3008, 256)])  # 64
def test_gemm_geometry(tiny_engine, M, N, K):
    a, w, bias = _operands(M, N, K, M + N + K)
    out = tiny_engine.gemm(a, w, bias, E.EPI_BIAS_F32, alpha=1.5)
    torch.cuda.synchronize()
    _check_f32(out, 1.5 * (a.float() @ w.float().T + bias))


def test_qkv_split_inside_tile(tiny_engine):
    M, N, K, split = 5640, 768, 256, 320                       # 256: the split at column 320 lies inside the second W tile
    d = N - split
    a, w, bias = _operands(M, N, K, 11)
    out = torch.full((M, N), 3.0, dtype=torch.bfloat16, device="cuda")
    ld2 = M + 24
    out2 = torch.full((d, ld2), 5.0, dtype=torch.bfloat16, device="cuda")
    tiny_engine.gemm(a, w, bias, E.EPI_QKV_VT, out=out, out2=out2, split=split)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().T + bias
    err_qk = ((out[:, :split].float() - ref[:, :split]).abs() / (ref[:, :split].abs() + 1.0)).max().item()
    err_v = ((out2[:, :M].float() - ref[:, split:].T).abs() / (ref[:, split:].T.abs() + 1.0)).max().item()
    assert err_qk < 1.2e-2 and err_v < 1.2e-2, (err_qk, err_v)
    assert torch.all(out[:, split:] == 3.0)                    # V columns of out are not written
    assert torch.all(out2[:, M:] == 5.0)                       # nor frames past M


def test_glu_guard_rows(tiny_engine):
    M, N, K = 12600, 2048, 256                                 # 256: 99 M-tiles
    a, w, bias = _operands(M, N, K, 12)
    d = N // 2
    idx = E.glu_interleave_index(d).cuda()
    guard = torch.full((64, d), 7.0, dtype=torch.bfloat16, device="cuda")
    buf = torch.cat([torch.zeros(M, d, dtype=torch.bfloat16, device="cuda"), guard])
    tiny_engine.gemm(a, w[idx].contiguous(), bias[idx].contiguous(), E.EPI_BIAS_GLU_BF16, out=buf[:M])
    torch.cuda.synchronize()
    acc = a.float() @ w.float().T + bias
    ref = acc[:, :d] * torch.sigmoid(acc[:, d:])
    err = ((buf[:M].float() - ref).abs() / (ref.abs() + 1.0)).max().item()
    assert err < 1.2e-2, err
    assert torch.equal(buf[M:], guard)


def test_resid_in_place_guard_rows(tiny_engine):
    M, N, K = 12600, 1024, 512
    a, w, bias = _operands(M, N, K, 13)
    x = torch.randn(M, N, device="cuda")
    ref = x + 0.5 * (a.float() @ w.float().T + bias)
    guard = torch.full((64, N), 7.0, device="cuda")
    buf = torch.cat([x, guard])
    xin = buf[:M]
    tiny_engine.gemm(a, w, bias, E.EPI_RESID_F32, resid=xin, alpha=0.5, out=xin)
    torch.cuda.synchronize()
    assert (xin - ref).abs().max().item() < 2e-3
    assert torch.equal(buf[M:], guard)


@pytest.mark.parametrize("N,K,epi", [(1024, 1024, E.EPI_BIAS_F32), (4096, 1024, E.EPI_BIAS_SWISH_BF16), (3072, 1024, E.EPI_BIAS_BF16)])
@pytest.mark.parametrize("M_small", [392, 128])
def test_row_invariance_between_instances(tiny_engine, N, K, epi, M_small):
    """Rows computed inside an M = 12 544 launch (128 x 256 tiles) equal, bit for bit, the same rows computed in a
    launch of M_small rows (128 x 64 tiles): an utterance decodes the same alone and in a batch."""
    M = 12544
    a, w, bias = _operands(M, N, K, N + K)
    big = tiny_engine.gemm(a, w, bias, epi)
    r0 = 5 * 392
    small = tiny_engine.gemm(a[r0:r0 + M_small].contiguous(), w, bias, epi)
    torch.cuda.synchronize()
    assert torch.equal(big[r0:r0 + M_small], small)
