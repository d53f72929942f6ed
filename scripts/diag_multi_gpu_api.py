"""Where the one-process multi-GPU API (load_model(devices=[...]) + transcribe_batch) spends its wall time.

    python scripts/diag_multi_gpu_api.py [n_devices]        # on a box with that many H100s

Wraps the staging call, the engine call and decode_hypothesis with timers (per thread), runs the same clip list three times,
prints one JSON line per run.
"""
import json
import sys
import threading
import time

import torch

sys.path.insert(0, ".")
import importlib                                                                    # noqa: E402

mg = importlib.import_module("reazonspeech_b200.nemo.asr.multi_gpu")                # (asr.transcribe the attribute is the function)
tr = importlib.import_module("reazonspeech_b200.nemo.asr.transcribe")
from reazonspeech_b200.config import ModelConfig                                    # noqa: E402
from reazonspeech_b200.engine import Engine                                         # noqa: E402
from reazonspeech_b200.nemo.asr import TranscribeConfig, audio_from_numpy, load_model, transcribe_batch   # noqa: E402
from reazonspeech_b200.synth import synth_clip                                      # noqa: E402

acc = {}
lock = threading.Lock()


def timed(name, fn):
    def wrapper(*a, **k):
        t0 = time.perf_counter()
        try:
            return fn(*a, **k)
        finally:
            dt = time.perf_counter() - t0
            with lock:
                acc[name] = acc.get(name, 0.0) + dt
    return wrapper


def main():
    n_dev = int(sys.argv[1]) if len(sys.argv) > 1 else torch.cuda.device_count()
    cfg = ModelConfig()
    model = load_model(synthetic=True, config=cfg, seed=0, max_batch=32, devices=list(range(n_dev)))
    audios = [audio_from_numpy(synth_clip(i, 30.0), 16000) for i in range(n_dev * 32)]
    conf = TranscribeConfig(verbose=False)
    transcribe_batch(model, audios, conf)
    tr.HostStaging.stage = timed("stage (sum over threads)", tr.HostStaging.stage)
    Engine.transcribe_host = timed("engine call (sum over threads)", Engine.transcribe_host)
    tr.decode_hypothesis = timed("decode_hypothesis (caller thread)", tr.decode_hypothesis)
    for variant in ("first call of this shape (allocates the second pinned staging set)", "steady state", "steady state"):
        acc.clear()
        t0 = time.perf_counter()
        res = transcribe_batch(model, audios * 4, conf)
        dt = time.perf_counter() - t0
        print(json.dumps({"variant": variant, "devices": n_dev, "clips": len(res), "seconds": round(dt, 4), "rtfx": round(len(res) * 30.0 / dt),
                          "ms_per_clip": round(dt / len(res) * 1e3, 3), **{k: round(v, 4) for k, v in acc.items()}}))


if __name__ == "__main__":
    main()
