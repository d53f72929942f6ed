"""Cost of the confidence statistics on the benchmark batch (BASELINE.json configs[1]: 32 x 30 s clips, one batch, full model,
seeded weights): rs_transcribe_device against rs_transcribe_device_confidence (alpha = 0.33), alternating variants, STEPS timed
steps per variant per round, ROUNDS rounds.  Prints one JSON line: per variant the median step time of every round, the
overall median and the spread (max - min of the round medians), with the GPU name and power limit read in the same run.

    python scripts/bench_confidence.py [--steps 20] [--rounds 3] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PAD = 8000          # pad_audio: 0.5 s of silence on both sides


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    args = ap.parse_args()
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    L = int(args.seconds * 16000) + 2 * PAD
    wav = torch.zeros(args.clips, L)
    for i in range(args.clips):
        wav[i, PAD:L - PAD] = torch.from_numpy(synth_clip(i, args.seconds))
    wav, lens = wav.cuda(), torch.full((args.clips,), L, dtype=torch.int32).cuda()
    variants = {"off": None, "on": 0.33}
    outs = {k: None for k in variants}

    def step(alpha):
        return eng.transcribe_device(wav, lens, out=outs_for(alpha), alpha=alpha)

    bufs = {}

    def outs_for(alpha):
        if alpha not in bufs:
            U = eng.u_max(L)
            B = args.clips
            o = (torch.zeros(B, U, dtype=torch.int32, device="cuda"), torch.zeros(B, U, dtype=torch.int32, device="cuda"),
                 torch.zeros(B, dtype=torch.int32, device="cuda"))
            bufs[alpha] = o if alpha is None else o + (torch.zeros(B, U, 4, device="cuda"),)
        return bufs[alpha]

    for name, alpha in variants.items():
        for _ in range(args.warmup):
            outs[name] = step(alpha)
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(outs["off"][:3], outs["on"][:3]))
    rounds = {k: [] for k in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.steps)]
    for _ in range(args.rounds):
        for name, alpha in variants.items():
            for i in range(args.steps):
                ev[2 * i].record()
                step(alpha)
                ev[2 * i + 1].record()
            torch.cuda.synchronize()
            rounds[name].append(float(np.median([ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(args.steps)])))
    res = {k: {"round_median_ms": v, "median_ms": float(np.median(v)), "spread_ms": max(v) - min(v)} for k, v in rounds.items()}
    res["overhead_ms"] = res["on"]["median_ms"] - res["off"]["median_ms"]
    res["within_spread"] = abs(res["overhead_ms"]) <= max(res["on"]["spread_ms"], res["off"]["spread_ms"])
    res["tokens_identical"] = same
    res["tokens_per_clip"] = float(outs["off"][2].float().mean())
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
