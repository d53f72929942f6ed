"""Cost of phrase boosting per row (rs_set_boost_roots) on the benchmark batch (BASELINE.json configs[1]: 32 x 30 s clips, one
batch, full 619 M model, seeded weights).  The clips are encoded once; ``Engine.greedy`` alone (joint.enc projection + the decode
kernel) is timed with device events under three settings, alternated in one process, ROUNDS rounds of STEPS decodes each:

- ``global_empty``: the empty phrase list set globally (the kBoost instance, no roots);
- ``rows_empty``: 32 per-row copies of the empty list in one combined table with per-row roots -- the same decisions, so the
  difference to ``global_empty`` is the cost of the root lookup alone;
- ``rows_real``: 32 different lists of 50 phrases each (drawn from the piece table as scripts/bench_boosting.py draws them).

Also the host side of a ``phrases=`` call: building the combined table of 64 lists of 50 phrases (``combine_tables``) and
uploading it, and restacking the same 64 lists already built (what ``StreamingTranscriber`` does when the set of open lists
changes: ``stack_tables``) and uploading that, medians of a few repeats.  Then streaming (``bench_streaming.run``): 32 streams
of the bench's 30 s clips at the default configuration, each with its own (empty, distinct) list against none, alternated twice;
the median wall time of the steps in which every stream steps (per-step root staging and table swaps included; the first
step's restack is not in the median).  One JSON line, with the GPU name and power limit read in the same run.

    python scripts/bench_boosting_rows.py [--steps 20] [--rounds 3] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_boosting import phrases_from_pieces  # noqa: E402  (scripts/ is on sys.path when this file runs)
from bench_confidence import PAD, gpu_info  # noqa: E402
from bench_streaming import run as run_streams  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--score", type=float, default=2.0)
    args = ap.parse_args()
    from reazonspeech_b200.boosting import PhraseBoostingConfig, build_tables, combine_tables, stack_tables
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
    V, B = cfg.vocab_size, args.clips
    # per-row copies of the empty list are distinct lists (a different score each), so each gets its own 1-state region
    empties = [PhraseBoostingConfig([], args.score + 0.01 * i) for i in range(B)]
    reals = [PhraseBoostingConfig(phrases_from_pieces(tok.pieces, 50, 100 + i), args.score) for i in range(B)]
    settings = {"global_empty": combine_tables([], V, tok), "rows_empty": combine_tables(empties, V, tok),
                "rows_real": combine_tables(reals, V, tok)}
    dev = {k: (torch.from_numpy(t.bonus).cuda(), torch.from_numpy(t.next).cuda()) for k, (t, _) in settings.items()}

    def use(name):
        eng.set_phrase_boosting(*dev[name])
        if name != "global_empty":
            eng.set_boost_roots(settings[name][1])

    outs = {}
    for name in settings:
        use(name)
        for _ in range(args.warmup):
            outs[name] = eng.greedy(enc, enc_len)
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
    eng.set_phrase_boosting(None)
    res = {k: dict(round_median_ms=v, median_ms=float(np.median(v)), spread_ms=max(v) - min(v),
                   n_states=settings[k][0].n_states, tokens_per_clip=float(outs[k][2].float().mean())) for k, v in rounds.items()}
    base = res["global_empty"]["median_ms"]
    for k in settings:
        res[k]["overhead_pct"] = 100.0 * (res[k]["median_ms"] - base) / base
    res["rows_empty_tokens_identical"] = all(torch.equal(a, b) for a, b in zip(outs["global_empty"], outs["rows_empty"]))
    # host build + upload of 64 lists of 50 phrases
    lists64 = [PhraseBoostingConfig(phrases_from_pieces(tok.pieces, 50, 1000 + i), args.score) for i in range(64)]
    built = [build_tables(PhraseBoostingConfig(), V)] + [build_tables(c, V, tok) for c in lists64]
    build_ms, upload_ms, restack_ms = [], [], []
    for _ in range(5):
        t0 = time.perf_counter()
        t, _ = combine_tables(lists64, V, tok)
        t1 = time.perf_counter()
        d = (torch.from_numpy(t.bonus).cuda(), torch.from_numpy(t.next).cuda())
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        r, _ = stack_tables(built, V)
        d = (torch.from_numpy(r.bonus).cuda(), torch.from_numpy(r.next).cuda())
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        build_ms.append(1e3 * (t1 - t0)); upload_ms.append(1e3 * (t2 - t1)); restack_ms.append(1e3 * (t3 - t2))
        del d
    res["host_64x50"] = {"build_ms": float(np.median(build_ms)), "upload_ms": float(np.median(upload_ms)),
                         "restack_and_upload_ms": float(np.median(restack_ms)), "n_states": t.n_states,
                         "table_mb": 8 * t.n_states * t.pitch / 1e6}
    del eng, dev, enc, wav
    torch.cuda.empty_cache()
    from reazonspeech_b200.nemo.asr import load_model
    from reazonspeech_b200.streaming import StreamingConfig
    model = load_model("cuda:0", synthetic=True, max_batch=64)
    config = StreamingConfig()
    clips = [synth_clip(i, 30.0).astype(np.float32) for i in range(32)]
    # distinct empty lists: the same decisions as no lists, so the difference is the per-step cost of per-stream lists (the
    # kBoost instance, the roots, the table swaps around each engine call)
    stream_lists = [PhraseBoostingConfig([], args.score + 0.01 * i) for i in range(32)]
    run_streams(model, 32, config, clips, timed=False, lists=stream_lists)          # warm-up
    steps = {"no_lists": [], "own_lists": []}
    for _ in range(2):
        steps["no_lists"] += run_streams(model, 32, config, clips, timed=False)[0]
        steps["own_lists"] += run_streams(model, 32, config, clips, timed=False, lists=stream_lists)[0]
    res["streaming_32"] = {k: {"step_wall_ms": float(np.median(v)), "steps": len(v), "spread_ms": float(np.max(v) - np.min(v))}
                           for k, v in steps.items()}
    res.update(gpu_info())
    res.update({"clips": args.clips, "seconds": args.seconds, "steps": args.steps, "rounds": args.rounds, "score": args.score})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
