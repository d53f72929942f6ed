"""Cost of long-form alignment (``nemo.asr.align_long``) of a whole transcript without timestamps: the benchmark's 30 s
synthetic clips (BASELINE.json configs[1], full 619 M model, seeded weights) played back to back as one 960 s program (32
clips, the caption and keyword benches' program) and one 64-minute program (128 clips).  The text is the program's own greedy
transcript with seeded edits (5 % substitutions, 5 % deletions, 5 % insertions, ``synth.edit_tokens``): the shape of a script
that mostly, but not exactly, matches the audio.

Reported per program: the wall time of one ``align_long`` call (host clock around the synchronised call, the median of STEPS
calls after WARMUP); the device time of one more call with ``rs_enable_kernel_timing`` on, grouped into encoder (log-mel,
subsampling, the conformer layers and joint.enc), anchor decode (the greedy decode), predictor (the teacher-forced LSTM steps,
one launch per label position, and joint.pred), lattice and DP (recursions and backtrace); the host clock of the anchor
matching (difflib); the alignments run (widening), the band's cells against the full lattice's T x (U + 1), and the GPU name
and power limit read in the same run.  One JSON line.

    python scripts/bench_align_long.py [--steps 3] [--warmup 1] [--programs 32,128]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_confidence import gpu_info  # noqa: E402  (scripts/ is on sys.path when this file runs)


def group(tag: str) -> str:
    if "lattice" in tag:
        return "lattice"
    if "band_dp" in tag:
        return "dp"
    if "lstm_step" in tag or "pred_proj" in tag:
        return "predictor"
    if "greedy" in tag or "spec" in tag:
        return "anchor_decode"
    return "encoder"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--programs", default="32,128", help="clips per program, comma separated")
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.nemo.asr import TranscribeConfig, audio_from_numpy, align_long, transcribe
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.synth import edit_tokens, synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    T = sys.modules["reazonspeech_b200.nemo.asr.transcribe"]    # the module (the package exports a function of that name)
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    model = B200RnntModel(eng, PieceTableTokenizer(synthetic_pieces(cfg.vocab_size)))
    seen = {"match_ms": 0.0, "bands": []}
    anchors, build_band = T.anchors, T.build_band

    def timed_anchors(*a):
        t0 = time.perf_counter()
        out = anchors(*a)
        seen["match_ms"] += 1e3 * (time.perf_counter() - t0)
        return out

    def recorded_band(anchor, n_frames, W):
        lo, hi = build_band(anchor, n_frames, W)
        seen["bands"].append((int((hi.astype(np.int64) - lo).sum()), n_frames * len(lo)))
        return lo, hi

    T.anchors, T.build_band = timed_anchors, recorded_band
    programs = []
    for clips in (int(x) for x in args.programs.split(",")):
        program = audio_from_numpy(np.concatenate([synth_clip(i, args.seconds).astype(np.float32) for i in range(clips)]), 16000)
        heard = transcribe(model, program, TranscribeConfig(verbose=False, raw_hypothesis=True))
        greedy = heard.hypothesis.y_sequence.tolist()[1:]
        text = edit_tokens(greedy, cfg.vocab_size, seed=args.seed)
        for _ in range(args.warmup):
            align_long(model, program, text)
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            align_long(model, program, text)
            torch.cuda.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
        seen["match_ms"], seen["bands"] = 0.0, []
        eng.kernel_timing(True)
        r = align_long(model, program, text)
        kernels = eng.kernel_timing()
        eng.kernel_timing(False)
        groups = {}
        for tag, (n, k_ms) in kernels.items():
            g = groups.setdefault(group(tag), {"launches": 0, "ms": 0.0})
            g["launches"] += n; g["ms"] += k_ms
        band_cells, full_cells = seen["bands"][-1]
        programs.append(dict(clips=clips, program_seconds=program.seconds, tokens=len(text), greedy_tokens=len(greedy),
                             call_ms=ms, median_ms=float(np.median(ms)), spread_ms=max(ms) - min(ms), kernels=groups,
                             host_match_ms=seen["match_ms"], alignments=len(seen["bands"]), band_frames=r.hypothesis.band_frames,
                             edge=r.hypothesis.edge, band_cells=band_cells, full_cells=full_cells,
                             audio_hours_per_s=program.seconds / 3600.0 / (float(np.median(ms)) * 1e-3)))
    res = dict(programs=programs)
    res.update(gpu_info())
    res.update({"seconds": args.seconds, "steps": args.steps, "warmup": args.warmup, "seed": args.seed})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
