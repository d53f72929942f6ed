"""Streaming capacity at the 619 M geometry (synthetic weights): N concurrent streams of the bench's synthetic 30 s clips, each fed
one chunk (0.08 s-aligned) per step at the default StreamingConfig (1.6 s chunk, 1.2 s left and right).

Per N it reports, over the steps in which every stream steps (the steady state; the first steps only fill the right context):
  step_wall_ms      host wall time of StreamingTranscriber.step(), staging and copies included (rs_stream_step synchronises)
  step_device_ms    summed device time of the step's launches (per-launch CUDA events, a separate pass)
  decode_share      the greedy decode kernel's part of step_device_ms
  streams_realtime  N * chunk seconds / step_wall_ms: streams one GPU keeps in real time at this N
  latency_s         added latency = right context + step_wall_ms
plus the card's name and power limit, read in the same run.

    python scripts/bench_streaming.py [--streams 32,128,512] [--out bench_out/bench_streaming.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:                      # the numbers still stand; say the card could not be read
        return f"unknown ({exc})"


def run(model, N, config, clips, timed, lists=None):
    """``lists``: stream k is opened with its own phrase list ``lists[k % len(lists)]`` (None: the model's global list)."""
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    C = config.frames()[0]
    piece = C * 1280
    st = StreamingTranscriber(model, config, max_streams=N)
    ids = [st.open(boosting=None if lists is None else lists[k % len(lists)]) for k in range(N)]
    pos = [0] * N
    eng = model.engine
    wall, dev, dec = [], [], []
    while not all(st.done(s) for s in ids):
        for k, sid in enumerate(ids):
            w = clips[k % len(clips)]
            if sid in st.open_streams and pos[k] < len(w):
                st.feed(sid, w[pos[k]:pos[k] + piece])
                pos[k] += piece
                if pos[k] >= len(w):
                    st.close(sid)
        full = len(st.plan()) == N
        if timed:
            eng.kernel_timing(True)
        t0 = time.perf_counter()
        st.step()
        t1 = time.perf_counter()
        if timed:
            kt = eng.kernel_timing()
            eng.kernel_timing(False)
            if full:
                dev.append(sum(ms for _, ms in kt.values()))
                dec.append(sum(ms for name, (_, ms) in kt.items() if "greedy" in name))
        elif full:
            wall.append((t1 - t0) * 1e3)
    return wall, dev, dec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="32,128,512")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_streaming needs a CUDA device")
    from reazonspeech_b200.nemo.asr import load_model
    from reazonspeech_b200.streaming import StreamingConfig
    from reazonspeech_b200.synth import synth_clip
    model = load_model("cuda:0", synthetic=True, max_batch=64)
    config = StreamingConfig()
    C, Lc, R = config.frames()
    clips = [synth_clip(i, 30.0).astype(np.float32) for i in range(32)]
    run(model, 32, config, clips, timed=False)                       # warm-up of every shape the steps use
    out = {"card": card(), "config": {"chunk_s": config.chunk_seconds, "left_s": config.left_seconds, "right_s": config.right_seconds},
           "results": []}
    for N in [int(x) for x in args.streams.split(",")]:
        wall, _, _ = run(model, N, config, clips, timed=False)
        _, dev, dec = run(model, N, config, clips, timed=True)
        w, d, k = float(np.median(wall)), float(np.median(dev)), float(np.median(dec))
        r = {"streams": N, "steps": len(wall), "step_wall_ms": round(w, 2), "step_wall_spread_ms": round(float(np.max(wall) - np.min(wall)), 2),
             "step_device_ms": round(d, 2), "decode_share": round(k / d, 3), "streams_realtime": int(N * config.chunk_seconds * 1e3 / w),
             "latency_s": round(R * 0.08 + w / 1e3, 3)}
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
