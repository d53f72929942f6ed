"""Produce reazonspeech_b200/data/synth_calib_<config>_seed<seed>.json for the seeded synthetic
checkpoint (see weights.random_state_dict): (1) the time-average of the encoder output on a
calibration clip set -> joint.enc bias that cancels it, (2) a power-of-two joint.enc gain bringing
the time-varying part of enc_proj to about unit standard deviation, (3) the blank-bias shift giving
a greedy emission rate of about one token per three encoder frames.  A deterministic function of the
seeded weights; it shapes the decode load of the benchmark only and is not part of the engine.

    python scripts/calibrate_synthetic.py --config tiny     # on an H100, through the engine (a few short clips)
    python scripts/calibrate_synthetic.py --config full     # on an H100, through the engine (the benchmark's clip set)

Both go through the product path (the engine); the oracle is test infrastructure and is not used here.
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from reazonspeech_b200.config import ModelConfig
from reazonspeech_b200.synth import synth_clip
from reazonspeech_b200.weights import _bf16_round, apply_calibration, calibration_path, random_state_dict

TARGET = 1.0 / 3.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="tiny", choices=["tiny", "full"])
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    ap.add_argument("--ac-target", type=float, default=1.0, help="std of the time-varying part of enc_proj after the gain")
    a = ap.parse_args()
    cfg = ModelConfig.tiny() if a.config == "tiny" else ModelConfig()
    sd = random_state_dict(cfg, a.seed, calibrate=False)
    # tiny: a few short clips; full: the benchmark's own clip set (bench.py make_batch)
    secs = (6.0, 9.0, 12.0, 7.0) if a.config == "tiny" else (30.0,) * 32
    first = 100 if a.config == "tiny" else 0
    waves = [np.pad(synth_clip(first + i, s), 8000) for i, s in enumerate(secs)]
    n_frames = [cfg.enc_frames(len(w)) for w in waves]
    W, b0 = sd["joint.enc.weight"].clone(), sd["joint.enc.bias"].clone()
    bout0 = sd["joint.joint_net.2.bias"].clone()

    from reazonspeech_b200.engine import Engine
    eng = Engine(cfg, sd, "cuda:0")
    L = max(len(w) for w in waves)
    x = torch.zeros(len(waves), L)
    for i, w in enumerate(waves):
        x[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32).cuda()
    x = x.cuda()
    mel, mel_len = eng.log_mel(x, lens)
    enc, enc_len = eng.encode(mel, mel_len)
    torch.cuda.synchronize()
    enc = enc.cpu()
    valid = torch.cat([enc[i, : n_frames[i]] for i in range(len(waves))])

    dc = valid.mean(0)
    ac = valid - dc
    ep_ac = ac @ W.T
    print(f"enc: |dc| rms {dc.pow(2).mean().sqrt():.3f}, ac rms {ac.pow(2).mean().sqrt():.3f}; enc_proj ac std {ep_ac.std():.4f}")
    k = int(round(math.log2(a.ac_target / float(ep_ac.std()))))
    gain = 2.0 ** k
    bias = _bf16_round(b0 - gain * (W @ dc))
    calib = {"joint_enc_gain_log2": k, "joint_enc_bias": bias.tolist(), "blank_shift": 0.0}

    def install(shift):
        calib["blank_shift"] = shift
        s2 = dict(sd)
        s2["joint.enc.weight"], s2["joint.enc.bias"], s2["joint.joint_net.2.bias"] = W.clone(), b0.clone(), bout0.clone()
        apply_calibration(s2, cfg, calib)
        return s2

    worst = [0.0]

    def rate(shift):
        s2 = install(shift)
        eng.weights["joint.enc.w"].copy_(s2["joint.enc.weight"].to(torch.bfloat16))
        eng.weights["joint.enc.b"].copy_(s2["joint.enc.bias"])
        eng.weights["joint.out.b"].copy_(s2["joint.joint_net.2.bias"])
        _, _, ntok = eng.transcribe_device(x, lens)
        torch.cuda.synchronize()
        worst[0] = float((ntok.cpu().float() / torch.tensor(n_frames, dtype=torch.float32)).max())
        return float(ntok.sum()) / sum(n_frames)

    curve = {s: rate(s) for s in np.arange(-2.0, 8.01, 0.5)}
    print("rate curve:", {float(k2): round(v, 3) for k2, v in curve.items()})
    # the blank bias is stored in bf16: scan every representable value between the coarse bracket
    xs = sorted(curve)
    lo = max([s for s in xs if curve[s] > TARGET], default=xs[0])
    hi = min([s for s in xs if s > lo and curve[s] <= 0.3 * TARGET], default=xs[-1])   # wide enough to satisfy the worst-clip bound
    base = float(bout0[cfg.blank])
    vals = sorted({float(_bf16_round(torch.tensor(base + v))) - base for v in np.arange(lo, hi + 1e-6, 1.0 / 128)})
    fine, fine_worst = {}, {}
    for v in vals:
        fine[v] = rate(v); fine_worst[v] = worst[0]
    print("fine scan (mean rate, worst clip):", {round(k2, 4): (round(v, 3), round(fine_worst[k2], 2)) for k2, v in fine.items()})
    ok = {k2: v for k2, v in fine.items() if v > 0 and fine_worst[k2] <= 0.6} or {k2: v for k2, v in fine.items() if v > 0}
    best = min(ok, key=lambda k2: abs(math.log(ok[k2] / TARGET)))
    calib["blank_shift"] = best
    calib["rate"] = rate(best)
    calib["worst_clip_rate"] = worst[0]
    calib["note"] = f"config={a.config} seed={a.seed}; clips={list(secs)} s; produced by scripts/calibrate_synthetic.py"
    out = a.out or calibration_path(cfg, a.seed)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(calib, open(out, "w"))
    print(json.dumps({k2: v for k2, v in calib.items() if k2 != "joint_enc_bias"}), "->", out)


if __name__ == "__main__":
    main()
