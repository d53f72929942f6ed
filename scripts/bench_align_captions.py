"""Cost and recovery of caption alignment (``nemo.asr.align_captions``) on a 16-minute program: the benchmark's 32 x 30 s
synthetic clips (BASELINE.json configs[1], full 619 M model, seeded weights) played back to back.  The captions are each
clip's greedy transcript cut into pieces of about 15 tokens, stamped with the piece's true program times plus a seeded
5-20 s delay, as live captions trail the speech; each is searched in [start - 25 s, end).

Reported: the wall time of one ``align_captions`` call per program (host clock around the synchronised call, ROUNDS rounds of
STEPS calls after WARMUP) and captions per second; the device time of one more call with ``rs_enable_kernel_timing`` on,
grouped into encoder (log-mel, subsampling and the conformer layers), projection (joint.enc), predictor, lattice and DP; and
the share of captions whose located segment overlaps its true span.  The weights are synthetic, so that share says that the
search finds planted text in this engine, not how well it locates real broadcast captions.  One JSON line, with the GPU name
and power limit read in the same run.

    python scripts/bench_align_captions.py [--steps 3] [--rounds 3] [--warmup 1]
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

from bench_align import group as align_group  # noqa: E402  (scripts/ is on sys.path when this file runs)
from bench_confidence import PAD, gpu_info  # noqa: E402

PIECE_TOKENS = 15


def group(tag: str, cfg) -> str:
    return "dp" if "segment_dp" in tag else align_group(tag, cfg)


def clocks():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None


def make_captions(model, waves, seconds, seed):
    """-> (captions, true spans in program seconds) from each clip's greedy tokens and frames."""
    from reazonspeech_b200.nemo.asr import Caption
    rng = np.random.default_rng(seed)
    caps, spans = [], []
    for i, (tokens, frames) in enumerate(model.transcribe_tokens(waves, pad=PAD)):
        for lo in range(0, len(tokens), PIECE_TOKENS):
            ids, frs = tokens[lo:lo + PIECE_TOKENS], frames[lo:lo + PIECE_TOKENS]
            t0 = i * seconds + max(0.08 * frs[0] - 0.5, 0.0)
            t1 = i * seconds + max(0.08 * (frs[-1] + 1) - 0.5, 0.0)
            text = model.tokenizer.ids_to_text(ids)
            if not text:
                continue
            delay = float(rng.uniform(5.0, 20.0))
            caps.append(Caption(t0 + delay, t1 + delay, text))
            spans.append((t0, t1))
    return caps, spans


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.nemo.asr import align_captions, audio_from_numpy
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    model = B200RnntModel(eng, PieceTableTokenizer(synthetic_pieces(cfg.vocab_size)))
    waves = [synth_clip(i, args.seconds).astype(np.float32) for i in range(args.clips)]
    program = audio_from_numpy(np.concatenate(waves), 16000)
    caps, spans = make_captions(model, waves, args.seconds, args.seed)
    for _ in range(args.warmup):
        out = align_captions(model, program, caps)
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            align_captions(model, program, caps)
            torch.cuda.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
        rounds.append(float(np.median(ms)))
    eng.kernel_timing(True)
    align_captions(model, program, caps)
    kernels = eng.kernel_timing()
    eng.kernel_timing(False)
    groups = {}
    for tag, (n, ms) in kernels.items():
        g = groups.setdefault(group(tag, cfg), {"launches": 0, "ms": 0.0})
        g["launches"] += n; g["ms"] += ms
    located = [(r, sp) for r, sp in zip(out, spans) if r is not None]
    overlap = sum(r.start_seconds < t1 and r.end_seconds > t0 for r, (t0, t1) in located)
    med = float(np.median(rounds))
    res = dict(program_seconds=program.seconds, captions=len(caps), located=len(located), overlap=overlap,
               overlap_share=overlap / max(len(caps), 1), round_median_ms=rounds, median_ms=med,
               spread_ms=max(rounds) - min(rounds), captions_per_s=len(caps) / (med * 1e-3), kernels=groups,
               window_seconds_mean=float(np.mean([min(c.end_seconds, program.seconds) - max(c.start_seconds - 25.0, 0.0) for c in caps])),
               tokens_per_caption=float(np.mean([len(model.tokenizer.sentence_to_ids(c.text)) for c in caps])),
               confidence_median=float(np.median([r.confidence for r, _ in located])) if located else None,
               clocks_sm_maxsm_mem=clocks())
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds, "seed": args.seed})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
