"""Token and word confidence of the greedy decode, NeMo's confidence measures computed from four softmax statistics.

The decode kernel (csrc/decode_spec.cu, kConf) reduces, for every emitted token, the softmax p over all V classes of the
joint evaluation that emitted it (blank included, as NeMo's softmax is) to

    lp = log p[emitted]  (the emitted token is the argmax),  H1 = sum p log p,  A = sum p^alpha,  G = sum p^alpha log p.

EVERY measure below depends on the distribution only through (lp, H1, A, G) and V: max_prob uses the largest log-probability,
the Gibbs entropy sum p log p (alpha = 1) or sum p^alpha log p, the Tsallis and Renyi entropies sum p^alpha.  So the
logits never leave the kernel.

(R) The measure formulas, their names and defaults are NeMo's ``get_confidence_measure_bank`` /
``ConfidenceMethodConfig`` / ``ConfidenceConfig`` (nemo.collections.asr.parts.utils.asr_confidence_utils) as recalled,
not verified against an installed NeMo: the image carries none.  They are restated here with x = log p, v = V, t = alpha,
in terms of the four statistics:

    max_prob            t = 1: (v e^lp - 1) / (v - 1)             else (e^(t lp) v^t - 1) / (v^t - 1)
    entropy gibbs  lin  t = 1: 1 + H1 / ln v                      else 1 + G / ln v / v^(1 - t)
    entropy gibbs  exp  t = 1: (e^H1 v - 1) / (v - 1)             else (e^(t G) - c) / (1 - c),  c = v^(-t v^(1 - t))
    entropy tsallis lin t = 1: as gibbs lin                       else 1 + (1 - A) / (v^(1 - t) - 1)
    entropy tsallis exp t = 1: as gibbs exp                       else (e^((1 - A) / (1 - t)) - c) / (1 - c),  c = e^((1 - v^(1 - t)) / (1 - t))
    entropy renyi  lin  t = 1: as gibbs lin                       else 1 + log2(A) / (t - 1) / log2(v)
    entropy renyi  exp  t = 1: as gibbs exp                       else (A^(1 / (t - 1)) v - 1) / (v - 1)

(R) Aggregations (``mean`` / ``min`` / ``max`` / ``prod``) and the SentencePiece word grouping (a word starts at a piece that
begins with the word-boundary mark; a bare mark piece belongs to no word) are NeMo's as recalled.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

WORD_BOUNDARY = "▁"
METHODS = ("max_prob", "entropy")
ENTROPY_TYPES = ("gibbs", "tsallis", "renyi")
ENTROPY_NORMS = ("lin", "exp")
AGGREGATIONS = ("mean", "min", "max", "prod")


@dataclass
class ConfidenceMethodConfig:
    """NeMo's ConfidenceMethodConfig (R): ``name`` max_prob / entropy, ``entropy_type`` gibbs / tsallis / renyi, ``alpha`` > 0
    (the entropy parameter, and the max_prob exponent), ``entropy_norm`` lin / exp."""
    name: str = "entropy"
    entropy_type: str = "tsallis"
    alpha: float = 0.33
    entropy_norm: str = "exp"


@dataclass
class ConfidenceConfig:
    """NeMo's ConfidenceConfig (R) as far as greedy token / word confidence goes.  Only ``exclude_blank=True`` exists here: the
    decode records the emitted tokens, not the blank frames."""
    exclude_blank: bool = True
    aggregation: str = "min"
    method_cfg: ConfidenceMethodConfig = field(default_factory=ConfidenceMethodConfig)

    def validate(self) -> "ConfidenceConfig":
        m = self.method_cfg
        if not self.exclude_blank:
            raise ValueError("ConfidenceConfig(exclude_blank=False) is not supported: blank frames carry no recorded statistics")
        if self.aggregation not in AGGREGATIONS:
            raise ValueError(f"aggregation must be one of {AGGREGATIONS}, got {self.aggregation!r}")
        if m.name not in METHODS:
            raise ValueError(f"method name must be one of {METHODS}, got {m.name!r}")
        if m.entropy_type not in ENTROPY_TYPES:
            raise ValueError(f"entropy_type must be one of {ENTROPY_TYPES}, got {m.entropy_type!r}")
        if m.entropy_norm not in ENTROPY_NORMS:
            raise ValueError(f"entropy_norm must be one of {ENTROPY_NORMS}, got {m.entropy_norm!r}")
        if not (math.isfinite(m.alpha) and m.alpha > 0):
            raise ValueError(f"alpha must be positive and finite, got {m.alpha!r}")
        return self

    @property
    def alpha(self) -> float:
        return float(self.method_cfg.alpha)


def measure(stats, num_classes: int, method: ConfidenceMethodConfig) -> np.ndarray:
    """stats [..., 4] = (lp, H1, A_alpha, G_alpha) at alpha = ``method.alpha`` -> confidence [...] (float64)."""
    s = np.asarray(stats, dtype=np.float64)
    lp, h1, a, g = s[..., 0], s[..., 1], s[..., 2], s[..., 3]
    v, t = float(num_classes), float(method.alpha)
    if method.name == "max_prob":
        if t == 1.0:
            return (np.exp(lp) * v - 1) / (v - 1)
        return (np.exp(lp * t) * v ** t - 1) / (v ** t - 1)
    kind = method.entropy_type if t != 1.0 else "gibbs"         # every entropy is the Gibbs one at alpha = 1
    if method.entropy_norm == "lin":
        if kind == "gibbs":
            return 1 + (h1 if t == 1.0 else g / v ** (1 - t)) / math.log(v)
        if kind == "tsallis":
            return 1 + (1 - a) / (v ** (1 - t) - 1)
        return 1 + np.log2(a) / (t - 1) / math.log2(v)
    if kind == "gibbs":
        if t == 1.0:
            return (np.exp(h1) * v - 1) / (v - 1)
        c = v ** (-t * v ** (1 - t))
        return (np.exp(g * t) - c) / (1 - c)
    if kind == "tsallis":
        c = math.exp((1 - v ** (1 - t)) / (1 - t))
        return (np.exp((1 - a) / (1 - t)) - c) / (1 - c)
    return (a ** (1 / (t - 1)) * v - 1) / (v - 1)


def aggregate(values: Sequence[float], how: str) -> float:
    x = np.asarray(values, dtype=np.float64)
    if how == "mean":
        return float(x.mean())
    if how == "min":
        return float(x.min())
    if how == "max":
        return float(x.max())
    if how == "prod":
        return float(x.prod())
    raise ValueError(f"aggregation must be one of {AGGREGATIONS}, got {how!r}")


def word_spans(pieces: Sequence[str]) -> List[tuple]:
    """[start, end) token ranges of the words of a SentencePiece sequence: a word starts at a piece beginning with the
    word-boundary mark (or at the first piece); a bare mark piece is dropped, as ids_to_text drops it (R)."""
    spans, start = [], 0
    for i in range(1, len(pieces) + 1):
        if i == len(pieces) or pieces[i].startswith(WORD_BOUNDARY):
            if i > start and not (i - start == 1 and pieces[start] == WORD_BOUNDARY):
                spans.append((start, i))
            start = i
    return spans


def word_confidence(token_confidence: Sequence[float], pieces: Sequence[str], how: str) -> List[float]:
    return [aggregate(token_confidence[a:b], how) for a, b in word_spans(pieces)]
