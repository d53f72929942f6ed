"""Cost of ALSD N-best lists on the benchmark batch (32 x 30 s synthetic clips, full 619 M model, seeded weights, beam 4).
On the batch's encoder output (log-mel and encoder run once, outside the timing): ``Engine.alsd`` (the winner only) and
``Engine.alsd_nbest`` at N = 4 and 64.  End to end: ``B200RnntModel.transcribe_alsd_nbest(n_best=4, log_likelihood=True)``
(staging, log-mel, encoder, the search, and forced alignment of every candidate).  Each is timed with a host clock around the
synchronised call, ROUNDS rounds of STEPS calls after WARMUP; the result is the median over rounds of each round's median.
The mean size of NeMo's whole list per clip (``pool``) shows how much of it N = 64 covers.  One JSON line, with the GPU name
and power limit read in the same run.

    python scripts/bench_alsd_nbest.py [--steps 3] [--rounds 3] [--warmup 1]
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
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0", alsd=True)
    model = B200RnntModel(eng, PieceTableTokenizer(synthetic_pieces(cfg.vocab_size)), max_batch=args.clips, decoding="alsd",
                          beam_size=args.beam)
    waves = [np.pad(synth_clip(i, args.seconds).astype(np.float32), PAD) for i in range(args.clips)]
    L = max(len(w) for w in waves)
    x = torch.zeros(len(waves), L)
    for i, w in enumerate(waves):
        x[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    mel, mel_len = eng.log_mel(x.cuda(), lens.cuda())
    enc, enc_len = eng.encode(mel, mel_len)
    res = {"alsd": timed(lambda: eng.alsd(enc, enc_len, beam=args.beam), args.steps, args.rounds, args.warmup)}
    for N in (4, 64):
        res[f"alsd_nbest_{N}"] = timed(lambda: eng.alsd_nbest(enc, enc_len, N, beam=args.beam), args.steps, args.rounds, args.warmup)
    out = [a.cpu() for a in eng.alsd_nbest(enc, enc_len, 64, beam=args.beam)]
    count, pool, from_final = out[4], out[5], out[6]
    res["transcribe_alsd_nbest_4_log_likelihood"] = timed(lambda: model.transcribe_alsd_nbest(waves, 4, log_likelihood=True),
                                                          args.steps, args.rounds, args.warmup)
    res.update(pool_mean=float(pool.float().mean()), pool_max=int(pool.max()), count64_mean=float(count.float().mean()),
               from_final_clips=int(from_final.sum()), tokens_per_clip=float(out[2][:, 0].float().mean()))
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "beam": args.beam, "steps": args.steps, "rounds": args.rounds})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
