"""Cost of keyword spotting (``nemo.asr.find_keywords``) on a 16-minute program: the benchmark's 32 x 30 s synthetic clips
(BASELINE.json configs[1], full 619 M model, seeded weights) played back to back, searched for 100 seeded keywords of 2-6
tokens drawn from the piece table as scripts/bench_boosting.py draws its phrases (index 7 on: no boundary, no punctuation).
A 16-minute program and 100 keywords is the shape of the archive search this feature is for: hours of audio are searched a
program at a time, and a keyword list is tens to hundreds of names.

Reported: the wall time of one ``find_keywords`` call (host clock around the synchronised call, ROUNDS rounds of STEPS calls
after WARMUP; the median of the round medians and their spread); the device time of one more call with
``rs_enable_kernel_timing`` on, grouped into encoder (log-mel, subsampling, the conformer layers and joint.enc), predictor,
lattice, spot DP and pick (the hit policy and the backtraces); keyword-hours per second (keywords x program hours / median
time) and lattice cells per second (pairs x frames x (U_max + 1) of the calls, over the median time).  One JSON line, with the
GPU name and power limit read in the same run.

    python scripts/bench_keywords.py [--steps 3] [--rounds 3] [--warmup 1]
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
    if "spot_dp" in tag:
        return "spot_dp"
    if "spot_pick" in tag:
        return "pick"
    if "lstm_step" in tag or "pred_proj" in tag:
        return "predictor"
    return "encoder"


def keywords_from_pieces(pieces, n, seed):
    """n keywords of 2-6 pieces each, drawn from the table's kana / ideographs."""
    rng = np.random.default_rng(seed)
    return ["".join(pieces[int(i)] for i in rng.integers(7, len(pieces), int(rng.integers(2, 7)))) for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--keywords", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.keywords import keyword_groups, keyword_ids
    from reazonspeech_b200.nemo.asr import audio_from_numpy, find_keywords
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    tok = PieceTableTokenizer(synthetic_pieces(cfg.vocab_size))
    model = B200RnntModel(eng, tok)
    program = audio_from_numpy(np.concatenate([synth_clip(i, args.seconds).astype(np.float32) for i in range(args.clips)]), 16000)
    keywords = keywords_from_pieces(tok.pieces, args.keywords, args.seed)
    ids = keyword_ids(keywords, cfg.vocab_size, tok)
    for _ in range(args.warmup):
        out = find_keywords(model, program, keywords)
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            find_keywords(model, program, keywords)
            torch.cuda.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
        rounds.append(float(np.median(ms)))
    eng.kernel_timing(True)
    find_keywords(model, program, keywords)
    kernels = eng.kernel_timing()
    eng.kernel_timing(False)
    groups = {}
    for tag, (n, ms) in kernels.items():
        g = groups.setdefault(group(tag), {"launches": 0, "ms": 0.0})
        g["launches"] += n; g["ms"] += ms
    T = eng.enc_frames((len(program.waveform) + 16000 + 3) & ~3)   # encoder frames of the padded, staged program
    lengths = [len(k) for k in ids]
    cells = sum(len(g) * T * (max(lengths[k] for k in g) + 1) for g in keyword_groups(lengths, 1, T))
    med = float(np.median(rounds))
    hours = program.seconds / 3600.0
    res = dict(program_seconds=program.seconds, keywords=len(keywords), tokens_per_keyword=float(np.mean(lengths)),
               hits=sum(len(h) for h in out), keywords_with_hits=sum(bool(h) for h in out),
               round_median_ms=rounds, median_ms=med, spread_ms=max(rounds) - min(rounds), kernels=groups,
               keyword_hours_per_s=len(keywords) * hours / (med * 1e-3), lattice_cells=cells, lattice_cells_per_s=cells / (med * 1e-3))
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds, "seed": args.seed})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
