"""Cost of forced alignment on the benchmark batch (BASELINE.json configs[1]: 32 x 30 s synthetic clips, full 619 M model,
seeded weights), each clip aligned to its own greedy transcript.  ``B200RnntModel.align_tokens`` (staging, log-mel, encoder,
joint.enc projection, predictor, lattice, DP, copies back) is timed end to end with a host clock around the synchronised call,
ROUNDS rounds of STEPS calls after WARMUP; then one more call runs with ``rs_enable_kernel_timing`` on and its per-kernel device
times are grouped into encoder (log-mel, subsampling and the conformer layers), projection (joint.enc), predictor, lattice and
DP.  The lattice's algorithmic FLOPs are 2 * cells * (V + 1) * Hj over the valid cells (sum of T_b * (U_b + 1)); the kernel
executes twice that (two half terms per activation).  Its share of the 989 TFLOP/s dense FP16 figure of the H100 SXM data sheet
is given for the algorithmic and the executed work.  One JSON line, with the GPU name and power limit read in the same run.

    python scripts/bench_align.py [--steps 5] [--rounds 3] [--warmup 2]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_confidence import PAD, gpu_info  # noqa: E402  (scripts/ is on sys.path when this file runs)

DENSE_FP16_TFLOPS = 989.0


def group(tag: str, cfg) -> str:
    if "lattice" in tag:
        return "lattice"
    if "align_dp" in tag:
        return "dp"
    if "lstm_step" in tag or "pred_proj" in tag:
        return "predictor"
    if tag == f"gemm N={cfg.joint_hidden} K={cfg.d_model} epi=5" or "f32_to_bf16" in tag:
        return "projection"
    return "encoder"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    args = ap.parse_args()
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    model = B200RnntModel(eng, PieceTableTokenizer(synthetic_pieces(cfg.vocab_size)), max_batch=args.clips)
    waves = [synth_clip(i, args.seconds).astype(np.float32) for i in range(args.clips)]
    heard = model.transcribe_tokens(waves, pad=PAD)
    labels = [tokens for tokens, _ in heard]
    T_b = [eng.cfg.enc_frames(len(w) + 2 * PAD) for w in waves]
    for _ in range(args.warmup):
        out = model.align_tokens(waves, labels, pad=PAD)
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            model.align_tokens(waves, labels, pad=PAD)
            torch.cuda.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
        rounds.append(float(np.median(ms)))
    eng.kernel_timing(True)                                 # the next call's launches are logged
    model.align_tokens(waves, labels, pad=PAD)
    kernels = eng.kernel_timing()
    eng.kernel_timing(False)
    groups = {}
    for tag, (n, ms) in kernels.items():
        g = groups.setdefault(group(tag, cfg), {"launches": 0, "ms": 0.0})
        g["launches"] += n; g["ms"] += ms
    cells = sum(t * (len(y) + 1) for t, y in zip(T_b, labels))
    flops = 2.0 * cells * (cfg.vocab_size + 1) * cfg.joint_hidden
    lat_ms = groups.get("lattice", {}).get("ms", float("nan"))
    tflops = flops / (lat_ms * 1e-3) / 1e12
    res = dict(round_median_ms=rounds, median_ms=float(np.median(rounds)), spread_ms=max(rounds) - min(rounds), kernels=groups,
               cells=cells, cells_per_s=cells / (lat_ms * 1e-3), lattice_tflops_algorithmic=tflops,
               lattice_tflops_executed=2 * tflops, share_of_989_algorithmic=tflops / DENSE_FP16_TFLOPS,
               share_of_989_executed=2 * tflops / DENSE_FP16_TFLOPS, tokens_per_clip=float(np.mean([len(y) for y in labels])),
               loglik_mean=float(np.mean([o[3] for o in out])), viterbi_mean=float(np.mean([o[2] for o in out])))
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
