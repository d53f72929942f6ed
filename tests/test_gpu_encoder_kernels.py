"""Direct parity tests of the encoder's attention, depthwise-conv, subsampling and chained-LayerNorm kernels and of the
V^T-writing QKV epilogue, each against a float64 CPU reference of the same operation.

Every reference is computed from exactly the bf16 / f32 values the kernel reads, so a bar only has to cover the kernel's own
rounding points (named in each test).  Inputs come from a seeded CPU ``torch.Generator`` and are copied to the device, so the
CPU tests at the end of each section see the same data: they compute a list of plausible mis-implementations of every kernel
on those inputs and require each to sit at least ``SEPARATION`` times the bar away from the reference on valid rows, i.e.
the bar is tight enough to catch them.

Errors are scaled as in the GEMM tests: max |got - ref| / (|ref| + 1) over valid rows.
"""
from __future__ import annotations

import functools
import math
import re
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import pytest
import torch
import torch.nn.functional as F

from oracle import nemo_restated as O
from reazonspeech_b200 import engine as E
from reazonspeech_b200.config import ModelConfig

gpu = pytest.mark.gpu
SEPARATION = 3.0
DK = 128


def _scaled_err(got: torch.Tensor, ref: torch.Tensor) -> float:
    return ((got.double() - ref.double()).abs() / (ref.double().abs() + 1.0)).max().item()


def _round8(n: int) -> int:
    return (n + 7) // 8 * 8


def _conv_len(n: int) -> int:
    return (n - 1) // 2 + 1 if n > 0 else 0


def _bf(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16)


def _dev(d: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {k: v.cuda() for k, v in d.items()}


# ==================================================================================================== attention
# Bar: the kernel rounds the positional term (q + pos_bias_v) . p[c] / sqrt(dk) * log2(e) to IEEE half, the probabilities
# exp2(t - m) to bf16 before the P.V product (the row sums use the same rounded values), and the output to bf16; the
# global row's kernel rounds only its output.  Everything else is fp32 accumulation of bf16 products.
ATTN_BAR = 2e-2

ATTN_LENS = (1, 7, 8, 127, 128, 129, 255, 257, 388)
ATTN_WINDOWS = ((16, 16, 1), (128, 128, 1), (128, 128, 0), (8, 24, 1), (0, 128, 1), (128, 0, 1), (8, 13, 1), (0, 0, 1))


@dataclass(frozen=True)
class AttnCase:
    wl: int
    wr: int
    G: int
    H: int
    lens: Tuple[int, ...] = ATTN_LENS
    edge: bool = False       # the band-edge columns 0 and wl + wr of the positional table carry a large score

    @property
    def id(self) -> str:
        return f"w{self.wl}-{self.wr}-g{self.G}-h{self.H}" + ("-edge" if self.edge else "") + ("-long" if max(self.lens) > 1024 else "")


ATTN_CASES = [AttnCase(wl, wr, G, H) for (wl, wr, G) in ATTN_WINDOWS for H in (2, 8)] + [
    AttnCase(128, 128, 1, 8, edge=True),
    AttnCase(16, 16, 1, 2, edge=True),
    AttnCase(128, 128, 1, 2, lens=(1500, 1030)),      # T_max > 1024: the global row's score buffer beyond its 1024 floor
]


@functools.lru_cache(maxsize=None)
def attn_inputs(case: AttnCase) -> Dict[str, torch.Tensor]:
    """Kernel inputs on the CPU.  q' = q + pos_bias_u (what the QKV projection writes), k and v ~ N(0, 2) and N(0, 1) per
    element, so that the content score q'.k / sqrt(dk) has a standard deviation of about 2 (a peaked softmax); the positional
    table is scaled so the positional score is comparable.  bd_bias = (pos_bias_v - pos_bias_u) . p[c] as pack_weights makes
    it.  Rows >= len hold random data as well (the kernel must not read them as valid)."""
    g = torch.Generator().manual_seed(1000 + 7 * case.wl + 3 * case.wr + case.G + 11 * case.H + 13 * case.edge + len(case.lens))
    H, d = case.H, case.H * DK
    B, T = len(case.lens), _round8(max(case.lens))
    M = B * T
    n_rel = case.wl + case.wr + 1
    n_rel_pad = (n_rel + 31) // 32 * 32
    qp = _bf(torch.randn(M, d, generator=g) * math.sqrt(2.0))
    k = _bf(torch.randn(M, d, generator=g) * math.sqrt(2.0))
    v = _bf(torch.randn(M, d, generator=g))
    u = _bf(torch.randn(H, DK, generator=g) * 0.5).float()
    vb = _bf(torch.randn(H, DK, generator=g) * 0.5).float()
    pos = torch.zeros(H, n_rel_pad, DK)
    pos[:, :n_rel] = torch.randn(H, n_rel, DK, generator=g) * 1.2
    if case.edge:
        # (vb - u) . p[c] grows by ~9 * sqrt(dk) at the two edge columns: a positional score ~9 above the others
        e = (vb - u) / (vb - u).norm(dim=1, keepdim=True) ** 2
        for c in {0, n_rel - 1}:
            pos[:, c] += e * 9.0 * math.sqrt(DK)
    pos = _bf(pos)
    bd_bias = ((pos.double() * (vb - u).double()[:, None, :]).sum(-1)).float()
    ld_vt = (M + 255) // 256 * 256 + 64                     # the engine's pitch
    vt = torch.zeros(d, ld_vt, dtype=torch.bfloat16)
    vt[:, :M] = v.T
    qkv = torch.cat([qp, k, v], 1).contiguous()
    return dict(qkv=qkv, vt=vt, pos=pos, bd_bias=bd_bias, u=u, vb=vb, enc_len=torch.tensor(case.lens, dtype=torch.int32))


def _heads(x: torch.Tensor, H: int) -> torch.Tensor:
    return x.double().view(x.shape[0], H, DK).transpose(0, 1)              # [H, L, dk]


def attn_oracle(case: AttnCase, inp, b: int) -> torch.Tensor:
    """oracle.nemo_restated.local_attention_core in float64 on utterance b -> [L, H*dk]."""
    H, d, T, L = case.H, case.H * DK, _round8(max(case.lens)), case.lens[b]
    rows = inp["qkv"][b * T: b * T + L]
    qp, k, v = _heads(rows[:, :d], H), _heads(rows[:, d:2 * d], H), _heads(rows[:, 2 * d:], H)
    u = inp["u"].double()
    cfg = ModelConfig.tiny().replace(att_left=case.wl, att_right=case.wr, global_tokens=case.G)
    p = inp["pos"][:, : cfg.n_rel].double()
    out = O.local_attention_core(qp - u[:, None], k, v, p, u, inp["vb"].double(), cfg)
    return out.transpose(0, 1).reshape(L, d)


ATTN_MUTANTS = ("band_wide", "band_narrow", "bd_col+1", "bd_col-1", "last_key_masked",
                "no_global_col", "global_not_in_band", "global_with_qprime")


def attn_dense(case: AttnCase, inp, b: int, mutant: Optional[str] = None) -> torch.Tensor:
    """The same operation restated from the kernel's inputs (positional term = q'.p[c] + bd_bias[c]), float64, with an
    optional mis-implementation: the band one key wider / narrower on each side, the positional table read one column off
    (rel_shift off by one; columns outside the table read as 0, like the table's zero padding), the last valid key masked,
    the global column dropped, the global key removed from the local band, or the global score taken with q' = q + u."""
    H, d, T, L = case.H, case.H * DK, _round8(max(case.lens)), case.lens[b]
    wl, wr, G = case.wl, case.wr, case.G
    rows = inp["qkv"][b * T: b * T + L]
    qp, k, v = _heads(rows[:, :d], H), _heads(rows[:, d:2 * d], H), _heads(rows[:, 2 * d:], H)
    q = qp - inp["u"].double()[:, None]
    scale = 1.0 / math.sqrt(DK)
    table = qp @ inp["pos"].double().transpose(1, 2) + inp["bd_bias"].double()[:, None, :]    # [H, L, n_rel_pad]
    n_pad = table.shape[2]
    i, j = torch.arange(L)[:, None], torch.arange(L)[None, :]
    rel = j - i
    lo, hi = -wl, wr
    if mutant == "band_wide":
        lo, hi = lo - 1, hi + 1
    elif mutant == "band_narrow":
        lo, hi = lo + 1, hi - 1
    band = (rel >= lo) & (rel <= hi)
    if mutant == "last_key_masked":
        band = band & (j < L - 1)
    if mutant == "global_not_in_band" and G:
        band = band & (j > 0)
    col = rel + wl + {"bd_col+1": 1, "bd_col-1": -1}.get(mutant, 0)
    inside = (col >= 0) & (col < n_pad)
    bd = torch.gather(table, 2, col.clamp(0, n_pad - 1).unsqueeze(0).expand(H, L, L)) * inside
    s = ((qp @ k.transpose(1, 2) + bd) * scale).masked_fill(~band, float("-inf"))
    vv = v
    if G and mutant != "no_global_col":
        qg = qp if mutant == "global_with_qprime" else q
        s = torch.cat([(qg @ k[:, :1].transpose(1, 2)) * scale, s], -1)
        vv = torch.cat([v[:, :1], v], 1)
    out = torch.nan_to_num(torch.softmax(s, -1)) @ vv         # a row without a key (a mutant's empty band) gives zeros
    if G:
        out[:, 0] = (torch.softmax((q[:, 0:1] @ k.transpose(1, 2)) * scale, -1) @ v)[:, 0]
    return out.transpose(0, 1).reshape(L, d)


def _attn_call(eng, case: AttnCase, inp, T: Optional[int] = None):
    B = len(case.lens)
    T = T or _round8(max(case.lens))
    out = eng.attention(inp["qkv"], inp["vt"], inp["pos"], inp["bd_bias"], inp["u"], inp["enc_len"], B, T, case.wl, case.wr, case.G)
    torch.cuda.synchronize()
    return out.cpu()


@gpu
@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: c.id)
def test_attention_matches_oracle(tiny_engine, case):
    """Valid rows within ATTN_BAR of the float64 oracle; rows at or beyond an utterance's length are exact zeros."""
    inp = attn_inputs(case)
    out = _attn_call(tiny_engine, case, _dev(inp))
    T = _round8(max(case.lens))
    worst = 0.0
    for b, L in enumerate(case.lens):
        worst = max(worst, _scaled_err(out[b * T: b * T + L], attn_oracle(case, inp, b)))
        assert torch.count_nonzero(out[b * T + L: (b + 1) * T]).item() == 0, f"utterance {b}: rows >= len not zero"
    print(f"attention {case.id}: worst scaled error {worst:.3e} (bar {ATTN_BAR:.0e})")
    assert worst < ATTN_BAR


@gpu
@pytest.mark.parametrize("case", [AttnCase(16, 16, 1, 2), AttnCase(128, 128, 1, 8), AttnCase(8, 24, 0, 2), AttnCase(0, 128, 1, 2)], ids=lambda c: c.id)
def test_attention_padding_and_batch_position_invariance(tiny_engine, case):
    """(1) Large finite garbage in the q', k and V^T rows at or beyond every utterance's length leaves every valid row
    bit-identical (the TMA tiles of the local kernel cover those rows; they must be masked, and their probabilities are
    exactly 0).  NaN or inf in padded V is outside the contract: 0 * NaN in the P.V product.
    (2) An utterance gives the same bits alone at b = 0 as at b = 2 behind two utterances of other lengths: a tile's keys
    at negative offsets are the previous utterance's rows."""
    inp = attn_inputs(case)
    T, B, d = _round8(max(case.lens)), len(case.lens), case.H * DK
    clean = _attn_call(tiny_engine, case, _dev(inp))
    g = torch.Generator().manual_seed(77)
    dirty = dict(inp)
    qkv, vt = inp["qkv"].clone(), inp["vt"].clone()
    for b, L in enumerate(case.lens):
        n = T - L
        qkv[b * T + L: (b + 1) * T] = _bf(torch.randn(n, 3 * d, generator=g) * 3e4)
        vt[:, b * T + L: (b + 1) * T] = _bf(torch.randn(d, n, generator=g) * 3e4)
    dirty["qkv"], dirty["vt"] = qkv, vt
    got = _attn_call(tiny_engine, case, _dev(dirty))
    for b, L in enumerate(case.lens):
        assert torch.equal(got[b * T: b * T + L], clean[b * T: b * T + L]), f"utterance {b}: padding garbage changed a valid row"
    # utterance 8 (len 388) alone, and at b = 2 behind utterances 5 (129) and 1 (7)
    order = [5, 1, 8]
    sub = AttnCase(case.wl, case.wr, case.G, case.H, lens=tuple(case.lens[i] for i in order))
    rows = lambda t, i: t[i * T: (i + 1) * T]
    trio = dict(inp, qkv=torch.cat([rows(inp["qkv"], i) for i in order]), enc_len=torch.tensor(sub.lens, dtype=torch.int32))
    vt3 = torch.zeros(d, 3 * T + 64, dtype=torch.bfloat16)
    vt3[:, : 3 * T] = torch.cat([inp["vt"][:, i * T: (i + 1) * T] for i in order], 1)
    trio["vt"] = vt3
    alone_case = AttnCase(case.wl, case.wr, case.G, case.H, lens=(case.lens[8],))
    alone = dict(inp, qkv=rows(inp["qkv"], 8).contiguous(), enc_len=torch.tensor(alone_case.lens, dtype=torch.int32),
                 vt=inp["vt"][:, 8 * T: 9 * T].contiguous())
    out3 = _attn_call(tiny_engine, sub, _dev(trio), T)
    out1 = _attn_call(tiny_engine, alone_case, _dev(alone), T)
    assert torch.equal(out3[2 * T: 3 * T], out1)
    assert torch.equal(out3[2 * T: 3 * T], clean[8 * T: 9 * T])


@gpu
def test_attention_rejects_unsupported_geometry_before_launch(tiny_engine):
    case = AttnCase(16, 16, 1, 2)
    inp = _dev(attn_inputs(case))
    T = _round8(max(case.lens))
    for wl, wr, G, t_max, msg in ((4, 16, 1, T, "(-5)"), (16, 200, 1, T, "(-5)"), (16, 16, 2, T, "(-5)"), (16, 16, 1, T - 4, "(-5)")):
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            tiny_engine.attention(inp["qkv"], inp["vt"], inp["pos"], inp["bd_bias"], inp["u"], inp["enc_len"], len(case.lens), t_max, wl, wr, G)
    with pytest.raises(RuntimeError, match=re.escape("(-1)")):        # V^T pitch below B * T_max
        tiny_engine.attention(inp["qkv"], inp["vt"][:, :64].contiguous(), inp["pos"], inp["bd_bias"], inp["u"], inp["enc_len"], len(case.lens), T, 16, 16, 1)


@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: c.id)
def test_attention_bar_separates_mutants(case):
    """CPU: the float64 restatement equals the oracle, and every mis-implementation of ATTN_MUTANTS that applies to the case
    is at least SEPARATION x ATTN_BAR away from it on the valid rows of the batch."""
    inp = attn_inputs(case)
    ref = [attn_dense(case, inp, b) for b in range(len(case.lens))]
    for b in range(len(case.lens)):
        # they differ only by bd_bias being stored in f32 (~1e-7)
        assert (ref[b] - attn_oracle(case, inp, b)).abs().max().item() < 1e-5
    dist = {}
    for m in ATTN_MUTANTS:
        if m in ("no_global_col", "global_not_in_band", "global_with_qprime") and case.G == 0:
            continue
        if m == "global_not_in_band" and case.wl == 0:      # then key 0 is in the band of the global row alone: no difference
            continue
        dist[m] = max(_scaled_err(attn_dense(case, inp, b, m), ref[b]) for b in range(len(case.lens)))
    print(f"attention {case.id}: smallest mutant distance {min(dist.values()):.3e} ({min(dist, key=dist.get)})")
    for m, x in dist.items():
        assert x >= SEPARATION * ATTN_BAR, f"{m}: {x:.3e}"




# ==================================================================================================== QKV projection, V^T
@gpu
@pytest.mark.parametrize("M", [8, 136, 392, 3104])
@pytest.mark.parametrize("pitch", ["M", "engine"])
def test_gemm_qkv_vt_epilogue(tiny_engine, M, pitch):
    """RS_EPI_QKV_VT against an RS_EPI_BIAS_BF16 run of the same GEMM: the q | k block is bit-identical, and V^T is bit-identical
    to the transposed V columns (the same main loop, the same fp32 tile and the same bf16 rounding; only the store differs).
    The V^T columns [M, ld2) and the V columns of the row-major output are never written, with ld2 = M as well as with the
    engine's pitch (M rounded up to 256, + 64).  The BIAS_BF16 run itself is within bf16 rounding of a float64 matmul."""
    eng = tiny_engine
    d = 256
    N, K = 3 * d, d
    g = torch.Generator().manual_seed(M)
    a = _bf(torch.randn(M, K, generator=g)).cuda()
    w = _bf(torch.randn(N, K, generator=g) / math.sqrt(K)).cuda()
    bias = torch.randn(N, generator=g).cuda()
    plain = eng.gemm(a, w, bias, E.EPI_BIAS_BF16)
    ld2 = M if pitch == "M" else (M + 255) // 256 * 256 + 64
    guard = torch.tensor(-7.0, dtype=torch.bfloat16)
    out = torch.full((M, N), -7.0, dtype=torch.bfloat16, device="cuda")
    vt = torch.full((d + 1, ld2), -7.0, dtype=torch.bfloat16, device="cuda")       # + one guard row
    eng.gemm(a, w, bias, E.EPI_QKV_VT, out=out, out2=vt[:d], split=2 * d)
    torch.cuda.synchronize()
    plain, out, vt = plain.cpu(), out.cpu(), vt.cpu()
    ref = a.cpu().double() @ w.cpu().double().T + bias.cpu().double()
    assert _scaled_err(plain, ref) < 8e-3
    assert torch.equal(out[:, : 2 * d], plain[:, : 2 * d])
    assert torch.equal(vt[:d, :M], plain[:, 2 * d:].T)
    assert bool((out[:, 2 * d:] == guard).all()) and bool((vt[:d, M:] == guard).all()) and bool((vt[d] == guard).all())


@gpu
def test_gemm_qkv_vt_rejects_bad_shapes_before_launch(tiny_engine):
    eng = tiny_engine
    a = torch.zeros(13, 256, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(768, 256, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(13, 768, dtype=torch.bfloat16, device="cuda")
    for m, ld2, split in ((13, 16, 512), (8, 16, 500), (8, 4, 512)):        # M % 8, split % 32, ld2 < M
        vt = torch.zeros(256, ld2, dtype=torch.bfloat16, device="cuda")
        with pytest.raises(RuntimeError, match=re.escape("(-1)")):
            eng.gemm(a[:m], w, None, E.EPI_QKV_VT, out=out, out2=vt, split=split)


# ==================================================================================================== depthwise conv + Swish
# Bar: fp32 accumulation of the nine taps, the fast Swish (ex2.approx / rcp.approx) and the bf16 output rounding.
CONV_BAR = 8e-3
CONV_LENS = (1, 4, 8, 9, 17, 388)


@functools.lru_cache(maxsize=None)
def conv_inputs(d: int) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(2000 + d)
    B, T = len(CONV_LENS), _round8(max(CONV_LENS))
    return dict(u=_bf(torch.randn(B * T, d, generator=g)), w=torch.randn(9, d, generator=g) / 3.0,
                shift=torch.randn(d, generator=g) * 0.5, enc_len=torch.tensor(CONV_LENS, dtype=torch.int32))


def conv_ref(inp, b: int, mutant: Optional[str] = None) -> torch.Tensor:
    """float64 depthwise conv1d (taps w[j, c] at offsets j - 4, BatchNorm folded into w and shift), input frames >= len read
    as zero, then Swish -> [len, d].  Mutants: the taps reversed; the frame at len read as valid."""
    d = inp["w"].shape[1]
    T, L = _round8(max(CONV_LENS)), CONV_LENS[b]
    n = L + 1 if mutant == "row_len_valid" else L
    x = torch.zeros(T + 8, d, dtype=torch.float64)
    x[4: 4 + n] = inp["u"][b * T: b * T + n].double()
    w = inp["w"].double()
    if mutant == "taps_reversed":
        w = w.flip(0)
    y = F.conv1d(x.T.unsqueeze(0), w.T.unsqueeze(1), inp["shift"].double(), groups=d)[0].T[:L]
    return y * torch.sigmoid(y)


@gpu
@pytest.mark.parametrize("d", [256, 1024])
def test_conv_dw_matches_reference(tiny_engine, d):
    """Valid rows within CONV_BAR.  Rows >= len are not zero: they hold the convolution of the masked input (swish(shift) once
    the window is past the utterance) and are never read as valid, so they are not asserted.  Garbage in the input rows >= len
    leaves every valid output bit-identical."""
    inp = conv_inputs(d)
    T = _round8(max(CONV_LENS))
    out = tiny_engine.conv_dw(inp["u"].cuda(), inp["w"].cuda(), inp["shift"].cuda(), inp["enc_len"].cuda(), T).cpu()
    worst = max(_scaled_err(out[b * T: b * T + L], conv_ref(inp, b)) for b, L in enumerate(CONV_LENS))
    print(f"conv_dw d={d}: worst scaled error {worst:.3e} (bar {CONV_BAR:.0e})")
    assert worst < CONV_BAR
    u = inp["u"].clone()
    g = torch.Generator().manual_seed(5)
    for b, L in enumerate(CONV_LENS):
        u[b * T + L: (b + 1) * T] = _bf(torch.randn(T - L, d, generator=g) * 3e4)
    dirty = tiny_engine.conv_dw(u.cuda(), inp["w"].cuda(), inp["shift"].cuda(), inp["enc_len"].cuda(), T).cpu()
    for b, L in enumerate(CONV_LENS):
        assert torch.equal(dirty[b * T: b * T + L], out[b * T: b * T + L])


@pytest.mark.parametrize("d", [256, 1024])
def test_conv_dw_bar_separates_mutants(d):
    inp = conv_inputs(d)
    for m in ("taps_reversed", "row_len_valid"):
        x = max(_scaled_err(conv_ref(inp, b, m), conv_ref(inp, b)) for b in range(len(CONV_LENS)))
        print(f"conv_dw d={d} {m}: {x:.3e}")
        assert x >= SEPARATION * CONV_BAR, m


# ==================================================================================================== subsampling
# Bar: fp32 accumulation (conv.0: 9 taps, conv.2: 9 taps of the ReLU'd conv.0 values, held in fp32) and the bf16 output
# rounding; with statistics, the normalisation (x - mean) * inv_std in fp32 on load.
SUB_BAR = 8e-3
SUB_F_MAX = 37


@functools.lru_cache(maxsize=None)
def sub_inputs(n_mels: int, C: int) -> Dict[str, torch.Tensor]:
    """Lengths 1, 2, 3, 4, 5, 8, 9, 13 and F_max cover every parity combination of len1 / len2 at the utterance's end; the mel
    rows >= len0 hold large finite garbage."""
    g = torch.Generator().manual_seed(3000 + n_mels + C)
    lens = (1, 2, 3, 4, 5, 8, 9, 13, SUB_F_MAX)
    mel = torch.randn(len(lens), SUB_F_MAX, n_mels, generator=g) * 2.0 + 0.5
    for b, L in enumerate(lens):
        mel[b, L:] = torch.randn(SUB_F_MAX - L, n_mels, generator=g) * 3e4
    stats = torch.stack([torch.randn(len(lens), n_mels, generator=g) * 0.5, torch.rand(len(lens), n_mels, generator=g) + 0.5], -1)
    return dict(mel=mel, mel_len=torch.tensor(lens, dtype=torch.int32), stats=stats.contiguous(),
                w0=torch.randn(C, 9, generator=g) / 3.0, b0=torch.randn(C, generator=g) * 0.3,
                wd=torch.randn(C, 9, generator=g) / 3.0, bd=torch.randn(C, generator=g) * 0.3)


def sub_conv0_dw1_ref(inp, b: int, with_stats: bool, mutant: Optional[str] = None) -> torch.Tensor:
    """float64 conv.0 (1 -> C, 3x3, s2, p1) + ReLU, conv.0 rows t1 >= len1 zeroed, conv.2 (depthwise 3x3, s2, p1) -> [len2, F2, C].
    Mel frames >= len0 read as zero (NeMo's zero tail).  Mutants: the conv.0 row t1 = len1 left unmasked; conv.0's stride-2
    input columns (mel bins) shifted by one."""
    L0 = int(inp["mel_len"][b])
    L1, L2 = _conv_len(L0), _conv_len(_conv_len(L0))
    C = inp["w0"].shape[0]
    x = inp["mel"][b].double().clone()
    if with_stats:
        x = (x - inp["stats"][b, :, 0].double()) * inp["stats"][b, :, 1].double()
    x[L0:] = 0.0
    if mutant == "column_shift":
        x = torch.cat([x[:, 1:], torch.zeros(x.shape[0], 1, dtype=torch.float64)], 1)
    y1 = F.relu(F.conv2d(x[None, None], inp["w0"].double().view(C, 1, 3, 3), inp["b0"].double(), stride=2, padding=1))
    y1[:, :, L1 + (1 if mutant == "t1_len1_unmasked" else 0):] = 0.0
    y2 = F.conv2d(y1, inp["wd"].double().view(C, 1, 3, 3), inp["bd"].double(), stride=2, padding=1, groups=C)
    return y2[0, :, :L2].permute(1, 2, 0)


SUB_CASES = [(n_mels, C, st) for n_mels in (80, 128) for C in (64, 256) for st in (False, True)]


@gpu
@pytest.mark.parametrize("n_mels,C,with_stats", SUB_CASES)
def test_sub_conv0_dw1_matches_reference(tiny_engine, n_mels, C, with_stats):
    """n_mels = 80 runs the compile-time-pitch instance, 128 the run-time-pitch one.  Valid rows within SUB_BAR; rows
    t2 >= len2 are exact zeros; the garbage in mel rows >= len0 never reaches a valid row (it is in the inputs)."""
    inp = sub_inputs(n_mels, C)
    dv = _dev(inp)
    out = tiny_engine.sub_conv0_dw1(dv["mel"], dv["mel_len"], dv["stats"] if with_stats else None, dv["w0"], dv["b0"], dv["wd"], dv["bd"]).cpu()
    worst = 0.0
    for b in range(out.shape[0]):
        L2 = _conv_len(_conv_len(int(inp["mel_len"][b])))
        worst = max(worst, _scaled_err(out[b, :L2], sub_conv0_dw1_ref(inp, b, with_stats)))
        assert torch.count_nonzero(out[b, L2:]).item() == 0
    print(f"sub_conv0_dw1 n_mels={n_mels} C={C} stats={with_stats}: worst scaled error {worst:.3e} (bar {SUB_BAR:.0e})")
    assert worst < SUB_BAR


@pytest.mark.parametrize("n_mels,C,with_stats", SUB_CASES)
def test_sub_conv0_dw1_bar_separates_mutants(n_mels, C, with_stats):
    inp = sub_inputs(n_mels, C)
    B = inp["mel"].shape[0]
    for m in ("t1_len1_unmasked", "column_shift"):
        x = max(_scaled_err(sub_conv0_dw1_ref(inp, b, with_stats, m), sub_conv0_dw1_ref(inp, b, with_stats)) for b in range(B))
        print(f"sub_conv0_dw1 n_mels={n_mels} C={C} stats={with_stats} {m}: {x:.3e}")
        assert x >= SEPARATION * SUB_BAR, m


def sub_dw_inputs(C: int):
    """Channels-last bf16 input of the second depthwise conv: [B, T2, F2, C] for mel lengths as in sub_inputs (80 bins), rows
    t >= len2 holding large finite garbage."""
    base = sub_inputs(80, C)
    g = torch.Generator().manual_seed(4000 + C)
    T2, F2 = _conv_len(_conv_len(SUB_F_MAX)), _conv_len(_conv_len(80))
    x = torch.randn(base["mel"].shape[0], T2, F2, C, generator=g)
    for b in range(x.shape[0]):
        x[b, _conv_len(_conv_len(int(base["mel_len"][b]))):] *= 3e4
    return dict(x=_bf(x), mel_len=base["mel_len"], w=base["wd"], b=base["bd"])


def sub_dw_ref(inp, b: int, mutant: Optional[str] = None) -> torch.Tensor:
    """float64 depthwise 3x3 s2 p1, input rows t >= len2 zeroed -> [len3, F3, C].  Mutants: the input row t = len2 read as
    valid; the stride-2 input columns shifted by one."""
    L2 = _conv_len(_conv_len(int(inp["mel_len"][b])))
    L3 = _conv_len(L2)
    C = inp["x"].shape[3]
    x = inp["x"][b].double().permute(2, 0, 1).clone()                      # [C, T2, F2]
    x[:, L2 + (1 if mutant == "row_len_valid" else 0):] = 0.0
    if mutant == "column_shift":
        x = torch.cat([x[:, :, 1:], torch.zeros(C, x.shape[1], 1, dtype=torch.float64)], 2)
    y = F.conv2d(x[None], inp["w"].double().view(C, 1, 3, 3), inp["b"].double(), stride=2, padding=1, groups=C)
    return y[0, :, :L3].permute(1, 2, 0)


@gpu
@pytest.mark.parametrize("C", [64, 256])
def test_sub_dw_matches_reference(tiny_engine, C):
    """len_shift = 2 as in the encoder.  Valid rows within SUB_BAR (fp32 accumulation, bf16 output), rows >= len3 exact zeros."""
    inp = sub_dw_inputs(C)
    dv = _dev(inp)
    out = tiny_engine.sub_dw(dv["x"], dv["w"], dv["b"], dv["mel_len"], 2).cpu()
    worst = 0.0
    for b in range(out.shape[0]):
        L3 = _conv_len(_conv_len(_conv_len(int(inp["mel_len"][b]))))
        worst = max(worst, _scaled_err(out[b, :L3], sub_dw_ref(inp, b)))
        assert torch.count_nonzero(out[b, L3:]).item() == 0
    print(f"sub_dw C={C}: worst scaled error {worst:.3e} (bar {SUB_BAR:.0e})")
    assert worst < SUB_BAR


@pytest.mark.parametrize("C", [64, 256])
def test_sub_dw_bar_separates_mutants(C):
    inp = sub_dw_inputs(C)
    for m in ("row_len_valid", "column_shift"):
        x = max(_scaled_err(sub_dw_ref(inp, b, m), sub_dw_ref(inp, b)) for b in range(inp["x"].shape[0]))
        print(f"sub_dw C={C} {m}: {x:.3e}")
        assert x >= SEPARATION * SUB_BAR, m


# ==================================================================================================== chained LayerNorm
@gpu
@pytest.mark.parametrize("rows", [333, 12419])
@pytest.mark.parametrize("d", [256, 1024])
def test_layernorm_chained_in_place(tiny_engine, rows, d):
    """norm_out of one layer chained with the next layer's first pre-norm, as the encoder runs it: x <- LN1(x) in place (f32)
    and LN2(LN1(x)) as bf16.  The kernel declares x and out_f32 __restrict__ while the encoder passes one buffer for both;
    with 12 419 rows every warp prefetches its next row while it writes the current one.  The in-place result must equal
    the two-buffer result bit for bit; f32 within 2e-5 of float64 LN1, bf16 within 8e-3 (scaled) of LN2(LN1)."""
    eng = tiny_engine
    g0 = torch.Generator().manual_seed(rows + d)
    x = torch.randn(rows, d, generator=g0) * 3 + 1
    g1, b1, g2, b2 = (torch.randn(d, generator=g0) for _ in range(4))
    eps = eng.cfg.ln_eps
    ln1 = F.layer_norm(x.double(), (d,), g1.double(), b1.double(), eps)
    ln2 = F.layer_norm(ln1, (d,), g2.double(), b2.double(), eps)
    xd, g1d, b1d, g2d, b2d = (t.cuda() for t in (x, g1, b1, g2, b2))
    sep_f32 = torch.empty_like(xd)
    sep_bf = torch.empty(rows, d, dtype=torch.bfloat16, device="cuda")
    eng.layernorm_chained(xd, g1d, b1d, g2d, b2d, sep_f32, sep_bf)
    inp_bf = torch.empty(rows, d, dtype=torch.bfloat16, device="cuda")
    xin = xd.clone()
    eng.layernorm_chained(xin, g1d, b1d, g2d, b2d, xin, inp_bf)
    torch.cuda.synchronize()
    assert torch.equal(xin, sep_f32) and torch.equal(inp_bf, sep_bf)
    assert (xin.cpu().double() - ln1).abs().max().item() < 2e-5
    assert _scaled_err(inp_bf.cpu(), ln2) < 8e-3
