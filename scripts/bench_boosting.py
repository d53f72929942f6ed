"""Cost of phrase boosting in the greedy decode on the benchmark batch (BASELINE.json configs[1]: 32 x 30 s clips, one batch,
full 619 M model, seeded weights).  The clips are encoded once; ``Engine.greedy`` alone (joint.enc projection + the decode
kernel) is timed with device events under four settings, alternated in one process, ROUNDS rounds of STEPS decodes each:
no table, an empty phrase list, 100 and 1000 phrases (drawn deterministically from the piece table: 1-4 pieces each, as
text through ``text_to_ids``), lambda = 2.0.  Per setting: the median decode time of every round, the overall median and the
spread, the decode kernel's iterations and phase cycle counters of CTA 0 (``rs_debug_decode_cycles``, from one whole-path
call), tokens per clip, and the number of automaton states.  One JSON line, with the GPU name and power limit read in the
same run.

    python scripts/bench_boosting.py [--steps 20] [--rounds 3] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_confidence import PAD, gpu_info  # noqa: E402  (scripts/ is on sys.path when this file runs)


def phrases_from_pieces(pieces, n, seed):
    """n phrases of 1-4 pieces each, pieces drawn from the table's kana / ideographs (index 7 on: no boundary, no punctuation)."""
    rng = np.random.default_rng(seed)
    return ["".join(pieces[int(i)] for i in rng.integers(7, len(pieces), int(rng.integers(1, 5)))) for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--score", type=float, default=2.0)
    args = ap.parse_args()
    from reazonspeech_b200.boosting import PhraseBoostingConfig, build_tables
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    eng = Engine(cfg, random_state_dict(cfg, seed=0), "cuda:0")
    tok = PieceTableTokenizer(synthetic_pieces(cfg.vocab_size))
    L = int(args.seconds * 16000) + 2 * PAD
    wav = torch.zeros(args.clips, L)
    for i in range(args.clips):
        wav[i, PAD:L - PAD] = torch.from_numpy(synth_clip(i, args.seconds))
    wav, lens = wav.cuda(), torch.full((args.clips,), L, dtype=torch.int32).cuda()
    enc, enc_len = eng.encode(*eng.log_mel(wav, lens))
    settings = {"unset": None, "empty": [], "100": phrases_from_pieces(tok.pieces, 100, 1), "1000": phrases_from_pieces(tok.pieces, 1000, 2)}
    tables = {k: None if v is None else build_tables(PhraseBoostingConfig(v, args.score), cfg.vocab_size, tok) for k, v in settings.items()}
    dev_tables = {k: None if t is None else (torch.from_numpy(t.bonus).cuda(), torch.from_numpy(t.next).cuda()) for k, t in tables.items()}

    def use(name):
        t = dev_tables[name]
        eng.set_phrase_boosting(None if t is None else t[0], None if t is None else t[1])

    outs, extra = {}, {}
    for name in settings:
        use(name)
        for _ in range(args.warmup):
            outs[name] = eng.greedy(enc, enc_len)
        eng.transcribe_device(wav, lens)                    # one whole-path call: its decode leaves the phase counters
        cyc = eng.decode_cycles(args.clips, L, eng.u_max(L))
        extra[name] = {"iterations": cyc["iterations"], "cycles_cta0": {k: v for k, v in cyc.items() if k not in ("iterations", "_")},
                       "tokens_per_clip": float(outs[name][2].float().mean()),
                       "n_states": None if tables[name] is None else tables[name].n_states}
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
    use("unset")
    res = {k: dict(round_median_ms=v, median_ms=float(np.median(v)), spread_ms=max(v) - min(v), **extra[k]) for k, v in rounds.items()}
    base = res["unset"]["median_ms"]
    for k in settings:
        res[k]["overhead_pct"] = 100.0 * (res[k]["median_ms"] - base) / base
    res["empty_tokens_identical"] = all(torch.equal(a, b) for a, b in zip(outs["unset"], outs["empty"]))
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds, "score": args.score})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
