"""Cost of n-gram LM shallow fusion in the greedy decode on the benchmark batch (BASELINE.json configs[1]: 32 x 30 s clips, one
batch, full 619 M model, seeded weights).  A seeded 4-gram ARPA over the model's vocabulary (tests/ngram_oracle.write_arpa;
about 1 M n-grams by default) is written to a temporary directory and compiled once (the host build time is reported).  The
clips are encoded once; ``Engine.greedy`` alone (joint.enc projection + the decode kernel) is timed with device events under
three settings, alternated in one process, ROUNDS rounds of STEPS decodes each: no LM, the LM at a vanishing alpha (2^-30:
every lookup is done, yet the decisions must equal those without the LM, which the script asserts) and the LM at a realistic
alpha.  Per setting: the median decode time of every round, the overall median and the spread, the decode kernel's iterations
and phase cycle counters of CTA 0 (``rs_debug_decode_cycles``, from one whole-path call) and tokens per clip.  One JSON line,
with the n-gram / state counts, the table size, the GPU name and power limit read in the same run.

    python scripts/bench_ngram_lm.py [--steps 20] [--rounds 3] [--warmup 3] [--sentences 40000]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--order", type=int, default=4)
    ap.add_argument("--sentences", type=int, default=40000)
    ap.add_argument("--alpha", type=float, default=0.02)
    args = ap.parse_args()
    from ngram_oracle import write_arpa
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "lm.arpa")
        t0 = time.perf_counter()
        n_ngrams = write_arpa(path, cfg.vocab_size, args.order, args.sentences, seed=0)
        write_s = time.perf_counter() - t0
        tables = {"vanishing": build_lm_tables(NgramLMConfig(path, 2.0 ** -30), cfg.vocab_size),
                  "realistic": build_lm_tables(NgramLMConfig(path, args.alpha), cfg.vocab_size)}
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    L = int(args.seconds * 16000) + 2 * PAD
    wav = torch.zeros(args.clips, L)
    for i in range(args.clips):
        wav[i, PAD:L - PAD] = torch.from_numpy(synth_clip(i, args.seconds))
    wav, lens = wav.cuda(), torch.full((args.clips,), L, dtype=torch.int32).cuda()
    enc, enc_len = eng.encode(*eng.log_mel(wav, lens))
    settings = ("off", "vanishing", "realistic")

    def use(name):
        eng.set_ngram_lm(tables.get(name))

    outs, extra = {}, {}
    for name in settings:
        use(name)
        for _ in range(args.warmup):
            outs[name] = eng.greedy(enc, enc_len)
        eng.transcribe_device(wav, lens)                    # one whole-path call: its decode leaves the phase counters
        cyc = eng.decode_cycles(args.clips, L, eng.u_max(L))
        extra[name] = {"iterations": cyc["iterations"], "cycles_cta0": {k: v for k, v in cyc.items() if k not in ("iterations", "_")},
                       "tokens_per_clip": float(outs[name][2].float().mean())}
    same = all(torch.equal(a, b) for a, b in zip(outs["off"], outs["vanishing"]))
    assert same, "the LM at alpha 2^-30 changed the decisions"
    torch.cuda.synchronize()
    rounds = {k: [] for k in settings}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.steps)]
    for _ in range(args.rounds):
        for name in settings:
            use(name)
            for i in range(args.steps):
                ev[2 * i].record()
                eng.greedy(enc, enc_len)
                ev[2 * i + 1].record()
            torch.cuda.synchronize()
            rounds[name].append(float(np.median([ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(args.steps)])))
    use("off")
    res = {k: dict(round_median_ms=v, median_ms=float(np.median(v)), spread_ms=max(v) - min(v), **extra[k]) for k, v in rounds.items()}
    base = res["off"]["median_ms"]
    for k in settings:
        res[k]["overhead_pct"] = 100.0 * (res[k]["median_ms"] - base) / base
    t = tables["realistic"]
    res.update({"vanishing_decisions_identical": same, "n_ngrams": n_ngrams, "n_states": t.n_states, "n_arcs": t.n_arcs,
                "table_mb": t.nbytes / 2 ** 20, "arpa_write_s": write_s, "host_build_s": t.build_seconds})
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds, "order": args.order,
                "alpha": args.alpha})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
