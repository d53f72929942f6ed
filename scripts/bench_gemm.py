"""Per-shape timing of the wgmma GEMM (gemm_wgmma.cu) through Engine.gemm, the rs_gemm_bf16 seam.

    python scripts/bench_gemm.py [--lib path/to/librs_engine.so] [--launches 50] [--tiling current|n-only]
                                 [--dump-outputs DIR]

Shapes: the six GEMMs of a Conformer layer at configs[1] (M = 32 x 392 rows) with their own epilogues, the two
subsampling 1x1 convs, the joint's encoder projection and the three products of an ALSD step (M = 32 clips x beam 4).
Per shape: 5 warm-up launches, then --launches launches between one pair of CUDA events.  Reported per shape: ms per
launch, algorithmic TFLOP/s (2 M N K), algorithmic HBM bytes (operands read once, output written once, the residual read
once) and GB/s, and the operand bytes a CTA pulls from L2 per FLOP for the tile the launch uses.  --lib loads another
build of the library (the Python binding is the same), so two builds can be timed alternately on one machine; --tiling
names the tile-selection rule of that build (n-only: 128 x 128 tiles when N % 128 == 0, else 128 x 64).
--dump-outputs writes each shape's outputs of one launch on fresh buffers (raw bytes, <shape>.out / <shape>.out2) into
DIR before it is timed, so that two builds can be compared byte for byte.
Prints one JSON line, with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from reazonspeech_b200 import engine as E  # noqa: E402

M_ENC = 32 * 392
M_ALSD = 32 * 4
# name, M, N, K, epilogue
SHAPES = [
    ("ffn_w1", M_ENC, 4096, 1024, E.EPI_BIAS_SWISH_BF16),
    ("ffn_w2", M_ENC, 1024, 4096, E.EPI_RESID_F32),
    ("qkv", M_ENC, 3072, 1024, E.EPI_QKV_VT),
    ("attn_out", M_ENC, 1024, 1024, E.EPI_RESID_F32),
    ("conv_pw1", M_ENC, 2048, 1024, E.EPI_BIAS_GLU_BF16),
    ("conv_pw2", M_ENC, 1024, 1024, E.EPI_RESID_F32),
    ("sub_pw1", 32 * 776 * 20, 256, 256, E.EPI_BIAS_RELU_BF16),
    ("sub_pw2", 32 * 392 * 10, 256, 256, E.EPI_BIAS_RELU_BF16),
    ("joint_enc", M_ENC, 640, 1024, E.EPI_BIAS_F32),
    ("alsd_lstm", M_ALSD, 2560, 3840, E.EPI_BIAS_F32),
    ("alsd_pred", M_ALSD, 640, 1920, E.EPI_BIAS_F32),
    ("alsd_out", M_ALSD, 3008, 1920, E.EPI_BIAS_F32),
]
OUT_BYTES = {E.EPI_BIAS_SWISH_BF16: 2, E.EPI_RESID_F32: 4, E.EPI_BIAS_GLU_BF16: 1, E.EPI_BIAS_RELU_BF16: 2,
             E.EPI_BIAS_F32: 4, E.EPI_QKV_VT: 2}     # per output column of N (GLU writes N / 2 bf16 columns)


def tile(M: int, N: int, num_sms: int, tiling: str):
    """(BM, BN) as launch_gemm of that build picks them."""
    if tiling == "n-only":
        return (128, 128) if N % 128 == 0 else (128, 64)
    return (128, 256) if N % 256 == 0 and math.ceil(M / 128) * (N // 256) >= num_sms else (128, 64)


def l2_bytes_per_flop(bm: int, bn: int) -> float:
    """Operand bytes one CTA loads per k-block (its A and W blocks) over the k-block's FLOPs."""
    return (bm + bn) * 64 * 2 / (2.0 * bm * bn * 64)


def card() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, limit, mx = [f.strip() for f in r.stdout.strip().split(",")][:3]
        return {"gpu": name, "power_limit_w": float(limit), "sm_max_mhz": float(mx)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "sm_max_mhz": None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="librs_engine.so to load (default: the one in this tree)")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--tiling", default="current", choices=["current", "n-only"])
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="write each shape's outputs (raw bytes) into DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a CUDA device")
    if args.lib:
        E._LIB_PATH = os.path.abspath(args.lib)
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig.tiny()
    eng = E.Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for name, M, N, K, epi in SHAPES:
        a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
        bias = torch.randn(N, device="cuda", generator=g)
        kw = {}
        if epi == E.EPI_RESID_F32:
            x = torch.randn(M, N, device="cuda", generator=g)
            kw = dict(resid=x, out=x)
        elif epi == E.EPI_QKV_VT:
            kw = dict(out=torch.empty(M, N, dtype=torch.bfloat16, device="cuda"),
                      out2=torch.empty(N // 3, M, dtype=torch.bfloat16, device="cuda"), split=2 * N // 3)
        elif epi == E.EPI_BIAS_GLU_BF16:
            kw = dict(out=torch.empty(M, N // 2, dtype=torch.bfloat16, device="cuda"))
        elif epi == E.EPI_BIAS_F32:
            kw = dict(out=torch.empty(M, N, dtype=torch.float32, device="cuda"))
        else:
            kw = dict(out=torch.empty(M, N, dtype=torch.bfloat16, device="cuda"))
        if args.dump_outputs:
            os.makedirs(args.dump_outputs, exist_ok=True)
            fresh = {k: v.clone() for k, v in kw.items() if k != "split"}
            if epi == E.EPI_RESID_F32:
                fresh["resid"] = fresh["out"]
            eng.gemm(a, w, bias, epi, **fresh, **({"split": kw["split"]} if "split" in kw else {}))
            torch.cuda.synchronize()
            for k in ("out", "out2"):
                if k in fresh:
                    fresh[k].view(torch.uint8).cpu().numpy().tofile(os.path.join(args.dump_outputs, f"{name}.{k}"))
        for _ in range(5):
            eng.gemm(a, w, bias, epi, **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            eng.gemm(a, w, bias, epi, **kw)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.launches
        flop = 2.0 * M * N * K
        hbm = M * K * 2 + N * K * 2 + M * N * OUT_BYTES[epi] + (M * N * 4 if epi == E.EPI_RESID_F32 else 0)
        bm, bn = tile(M, N, num_sms, args.tiling)
        rows.append({"shape": name, "M": M, "N": N, "K": K, "ms": round(ms, 5), "tflops": round(flop / ms / 1e9, 1),
                     "hbm_bytes": hbm, "hbm_gbs": round(hbm / ms / 1e6, 1), "tile": f"{bm}x{bn}",
                     "l2_bytes_per_flop": round(l2_bytes_per_flop(bm, bn), 5)})
        del a, w, bias, kw
    print(json.dumps({"lib": E._LIB_PATH, "tiling": args.tiling, "launches": args.launches, **card(), "shapes": rows}))


if __name__ == "__main__":
    main()
