"""Streaming keyword spotting at the 619 M geometry (synthetic weights): N live streams of the bench's synthetic 30 s clips,
each fed one chunk per step at the default StreamingConfig (1.6 s chunk, 1.2 s left and right), searched for 100 seeded
keywords drawn as scripts/bench_keywords.py draws them, at the default threshold and alert delay (10 s).

Per N it reports, over the steps in which every stream steps:
  step_wall_ms      host wall time of StreamingTranscriber.step() (rs_stream_step_spot synchronises)
  kernels_ms        device time per step of each part: encoder (log-mel, subsampling, conformer layers, joint.enc), decode,
                    gather, lattice, DP and pick (per-launch CUDA events, a separate pass)
  pairs_realtime    stream-keyword pairs one GPU keeps in real time at this N: N x keywords x chunk seconds / step_wall_ms
  record_bytes      one (stream, keyword) record, and the records of all N streams
  delay_p50_s / delay_p95_s / forced_share
                    the decision delay (decoded frame at the decision minus the hit's end frame) and the share of forced hits:
                    properties of the synthetic weights only, not of the released checkpoint on real audio
plus the card's name and power limit, read in the same run.  Then the lattice's tile waste: the lattice time of one
rs_rnnt_spot_resume call over 32 rows x the keywords at C = 16 frames (one 16-frame tile per row) and at C = 20 (two tiles,
12 of 32 frame rows unused).

    python scripts/bench_stream_keywords.py [--streams 32,128] [--keywords 100] [--threshold=-inf]

With the default threshold the synthetic weights give no hits on these clips; ``--threshold=-inf`` makes every end frame a
candidate, which exercises the cuts and measures the delays of the policy itself.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_keywords import keywords_from_pieces  # noqa: E402  (scripts/ is on sys.path when this file runs)
from bench_streaming import card  # noqa: E402


def group(tag: str) -> str:
    for key, name in (("spot_gather", "gather"), ("lattice", "lattice"), ("resume_dp", "dp"), ("resume_pick", "pick"), ("greedy", "decode")):
        if key in tag:
            return name
    return "encoder"


def run(model, N, config, clips, kw, timed):
    from reazonspeech_b200.nemo.asr import StreamingTranscriber
    C = config.frames()[0]
    piece = C * 1280
    st = StreamingTranscriber(model, config, max_streams=N, keywords=kw)
    ids = [st.open() for _ in range(N)]
    pos = [0] * N
    eng = model.engine
    wall, kern, delays, n_hits, n_forced = [], [], [], 0, 0
    while not all(st.done(s) for s in ids):
        for k, sid in enumerate(ids):
            w = clips[k % len(clips)]
            if sid in st.open_streams and pos[k] < len(w):
                st.feed(sid, w[pos[k]:pos[k] + piece])
                pos[k] += piece
                if pos[k] >= len(w):
                    st.close(sid)
        plan = dict(st.plan())
        full = len(plan) == N
        if timed:
            eng.kernel_timing(True)
        t0 = time.perf_counter()
        st.step()
        t1 = time.perf_counter()
        if timed:
            kt = eng.kernel_timing()
            eng.kernel_timing(False)
            if full:
                g = {}
                for tag, (_, ms) in kt.items():
                    g[group(tag)] = g.get(group(tag), 0.0) + ms
                kern.append(g)
        elif full:
            wall.append((t1 - t0) * 1e3)
        for sid, hits in st.take_hits().items():
            for h in hits:
                n_hits += 1; n_forced += h.forced
                if sid in plan:                          # decided at the end of this step's frames
                    row = plan[sid]
                    delays.append(max(0.08 * (row.dec_end + row.offset) - 0.5 - h.end_seconds, 0.0))
    return wall, kern, delays, n_hits, n_forced


def tile_waste(model, ids, reps=5):
    """Median lattice device time of one resumed-spot call over 32 rows x len(ids) keywords at 16 and at 20 frames per row."""
    eng = model.engine
    g = torch.Generator().manual_seed(0)
    enc = torch.randn(32, 40, model.cfg.d_model, generator=g).cuda()
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    out = {}
    for C in (16, 20):
        eng.set_spot_keywords(ids, -1.0, 125, C)
        rec = torch.zeros(32, len(ids), eng.spot_state_bytes, dtype=torch.uint8, device="cuda")
        ms = []
        for _ in range(reps):
            rec.zero_()
            eng.kernel_timing(True)
            eng.spot_resume(enc, i32([0] * 32), i32([C] * 32), i32(list(range(32))), i32([0] * 32), rec)
            kt = eng.kernel_timing()
            eng.kernel_timing(False)
            ms.append(sum(t for tag, (_, t) in kt.items() if "lattice" in tag))
        out[f"lattice_ms_c{C}"] = round(float(np.median(ms)), 3)
    out["c20_over_c16"] = round(out["lattice_ms_c20"] / out["lattice_ms_c16"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="32,128")
    ap.add_argument("--keywords", type=int, default=100)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--threshold", type=float, default=None, help="default: keywords.THRESHOLD")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_keywords needs a CUDA device")
    from reazonspeech_b200.keywords import StreamKeywordsConfig
    from reazonspeech_b200.nemo.asr import load_model
    from reazonspeech_b200.streaming import StreamingConfig
    from reazonspeech_b200.synth import synth_clip
    model = load_model("cuda:0", synthetic=True, max_batch=64)
    config = StreamingConfig()
    clips = [synth_clip(i, args.seconds).astype(np.float32) for i in range(32)]
    from reazonspeech_b200.keywords import THRESHOLD
    kw = StreamKeywordsConfig(keywords_from_pieces(model.tokenizer.pieces, args.keywords, args.seed),
                              threshold=THRESHOLD if args.threshold is None else args.threshold)
    run(model, 8, config, clips[:8], kw, timed=False)              # warm-up
    out = {"card": card(), "keywords": args.keywords, "delay_s": kw.max_delay_seconds, "threshold": kw.threshold, "results": []}
    for N in [int(x) for x in args.streams.split(",")]:
        wall, _, delays, n_hits, n_forced = run(model, N, config, clips, kw, timed=False)
        _, kern, _, _, _ = run(model, N, config, clips, kw, timed=True)
        w = float(np.median(wall))
        rec = model.engine.spot_state_bytes
        r = {"streams": N, "steps": len(wall), "step_wall_ms": round(w, 2), "step_wall_spread_ms": round(float(np.max(wall) - np.min(wall)), 2),
             "kernels_ms": {k: round(float(np.median([g.get(k, 0.0) for g in kern])), 3) for k in ("encoder", "decode", "gather", "lattice", "dp", "pick")},
             "pairs_realtime": int(N * args.keywords * config.chunk_seconds * 1e3 / w),
             "record_bytes": rec, "records_mb": round(N * args.keywords * rec / 2 ** 20, 1),
             "hits": n_hits, "forced_share": round(n_forced / max(n_hits, 1), 3),
             "delay_p50_s": round(float(np.percentile(delays, 50)), 2) if delays else None,
             "delay_p95_s": round(float(np.percentile(delays, 95)), 2) if delays else None}
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    from reazonspeech_b200.keywords import keyword_ids
    out["tile_waste"] = tile_waste(model, keyword_ids(kw.keywords, model.cfg.vocab_size, model.tokenizer))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
