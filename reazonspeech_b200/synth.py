"""Seeded synthetic 16 kHz test audio (SURVEY.md section 8d): speech-like AM/FM tone mixtures.

Clip ``i`` is a pure function of (seed + i, seconds): a few slowly frequency-modulated
sinusoids between 100 and 3500 Hz under a syllabic (3-6 Hz) amplitude envelope plus white
noise at -30 dBFS, peak-normalised to 0.3.  No dataset is reachable offline, so these clips
are the fixed clip set of the parity tests and the workload of bench.py."""
from __future__ import annotations

import numpy as np

SAMPLE_RATE = 16000


def synth_clip(index: int, seconds: float, seed: int = 1234) -> np.ndarray:
    rng = np.random.default_rng(seed + index)
    n = int(round(seconds * SAMPLE_RATE))
    t = np.arange(n, dtype=np.float64) / SAMPLE_RATE
    x = np.zeros(n, dtype=np.float64)
    for _ in range(int(rng.integers(3, 6))):
        f0 = rng.uniform(100.0, 3500.0)
        fm_rate, fm_depth = rng.uniform(0.5, 3.0), rng.uniform(0.02, 0.15) * f0
        phase = 2 * np.pi * (f0 * t - fm_depth / (2 * np.pi * fm_rate) * np.cos(2 * np.pi * fm_rate * t + rng.uniform(0, 6.28)))
        am = 0.5 * (1 + np.sin(2 * np.pi * rng.uniform(3.0, 6.0) * t + rng.uniform(0, 6.28)))
        x += rng.uniform(0.3, 1.0) * am * np.sin(phase + rng.uniform(0, 6.28))
    x += 10 ** (-30 / 20) * rng.standard_normal(n)
    x *= 0.3 / max(np.abs(x).max(), 1e-9)
    return x.astype(np.float32)


def synth_batch(count: int, seconds: float, seed: int = 1234):
    return [synth_clip(i, seconds, seed) for i in range(count)]


def edit_tokens(tokens, vocab_size: int, seed: int, sub: float = 0.05, dele: float = 0.05, ins: float = 0.05):
    """A transcript that differs from ``tokens`` by seeded edits: each token is substituted by a random id with probability
    ``sub`` or deleted with probability ``dele``, and a random id is inserted after it with probability ``ins``."""
    rng = np.random.default_rng(seed)
    out = []
    for k in tokens:
        r = rng.random()
        if r < sub:
            out.append(int(rng.integers(0, vocab_size)))
        elif r >= sub + dele:
            out.append(int(k))
        if rng.random() < ins:
            out.append(int(rng.integers(0, vocab_size)))
    return out
