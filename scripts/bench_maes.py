"""Cost of the MAES beam search on the benchmark batch (32 x 30 s synthetic clips, full 619 M model, seeded weights).  On the
batch's encoder output (log-mel and encoder run once, outside the timing): ``Engine.maes`` at beam 4 with NeMo's defaults
(num_steps 2, prefix_alpha 1, expansion_beta 2, expansion_gamma 2.3) without and with a seeded 4-gram LM
(tests/ngram_oracle.write_arpa, alpha 0.1), and ``Engine.alsd`` at beam 4 for comparison.  Each is timed with a host clock
around the synchronised call, ROUNDS rounds of STEPS calls after WARMUP; the result is the median over rounds of each round's
median.  ``live_rows_per_frame``: the mean number of expansion rows per frame (the rows that went through the predictor, all
rounds and clips together; the host reads each round's count, one pinned read per round), next to the worst case
B x beam x (beam + beta)^num_steps the GEMMs would otherwise run.  One JSON line, with the GPU name and power limit read in the
same run.

    python scripts/bench_maes.py [--steps 3] [--rounds 3] [--warmup 1]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_confidence import PAD, gpu_info  # noqa: E402  (scripts/ is on sys.path when this file runs)


def timed(fn, steps, rounds, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    meds = []
    for _ in range(rounds):
        ms = []
        for _ in range(steps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
        meds.append(float(np.median(ms)))
    return {"median_ms": float(np.median(meds)), "round_median_ms": meds, "spread_ms": max(meds) - min(meds)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--beam", type=int, default=4)
    args = ap.parse_args()
    from ngram_oracle import write_arpa
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0", alsd=True)
    waves = [np.pad(synth_clip(i, args.seconds).astype(np.float32), PAD) for i in range(args.clips)]
    L = max(len(w) for w in waves)
    x = torch.zeros(len(waves), L)
    for i, w in enumerate(waves):
        x[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    enc, enc_len = eng.encode(*eng.log_mel(x.cuda(), lens.cuda()))
    res = {}

    def maes():
        return eng.maes(enc, enc_len, beam=args.beam)

    def rows_per_frame():
        maes()
        rows, frames = eng.maes_last_rows()
        return rows / frames

    res["maes"] = timed(maes, args.steps, args.rounds, args.warmup)
    res["maes_live_rows_per_frame"] = rows_per_frame()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "lm4.arpa")
        n_grams = write_arpa(path, cfg.vocab_size, 4, 3000, seed=3)
        eng.set_ngram_lm(build_lm_tables(NgramLMConfig(path, 0.1), cfg.vocab_size))
        res["maes_lm"] = timed(maes, args.steps, args.rounds, args.warmup)
        res["maes_lm_live_rows_per_frame"] = rows_per_frame()
        eng.set_ngram_lm(None)
    res["alsd"] = timed(lambda: eng.alsd(enc, enc_len, beam=args.beam), args.steps, args.rounds, args.warmup)
    res["worst_case_rows_per_frame"] = args.clips * args.beam * (args.beam + 2) ** 2
    res["lm_ngrams"] = n_grams
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "beam": args.beam, "steps": args.steps, "rounds": args.rounds})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
