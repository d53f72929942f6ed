"""n-gram language-model shallow fusion of the greedy decode: ARPA file -> the decode kernel's lookup tables.

Users adapting the model to a domain train an n-gram LM on domain text, tokenised into the model's BPE ids, and fuse it into
the decode.  This is NeMo's convention for transducer shallow fusion with a KenLM ARPA trained by ``train_kenlm.py`` (recalled,
not checked against NeMo's code: marked (R)).

ARPA input.  A standard ARPA file with orders 1..N, 2 <= N <= 6; every n-gram line is ``log10p<TAB>w1 ... wn[<TAB>log10bow]``
(words separated by single spaces; a missing back-off weight is 0).  The ``\\data\\`` counts must match the sections and
``\\end\\`` must be present.

Token mapping (R).  A word is a token id in NeMo's BPE convention, ``word == chr(token_id + token_offset)`` (token_offset
defaults to 100).  ``<s>``, ``</s>`` and ``<unk>`` are the only other words accepted; any other word, including one that maps
outside [0, vocab_size), is a ValueError naming it.  A token without a unigram gets ``<unk>``'s probability; an LM without
``<unk>`` is rejected.  ``</s>`` is never used: greedy decoding has no end-of-sentence step.

State.  An utterance's state is a context h: the longest suffix of ``<s> y_1 ... y_t`` that occurs in the ARPA as an n-gram of
order <= N - 1 (only contexts the decode can reach count: token ids, with ``<s>`` only in front).  Every call starts each
utterance at ``<s>``, or at the empty context when the LM has no ``<s>``.  The state moves only on emissions: emitting token k
leads to the longest suffix of h.k that is such a context.

Fused decision.  For every (utterance, frame) with context h the decision is the argmax over all V + 1 classes of

    z_c = logit_c + [c != blank] * (bonus_boost(s, c) + alpha * ln(10) * log10 P(c | h))

with the standard back-off rule: P(c | h) is the explicit n-gram (h, c) when the ARPA has it, otherwise bow(h) * P(c | h'),
h' = h without its first token (log10: bow(h) + log10 P(c | h')).  Blank gets no LM term (R).  Adding the terms to the logits
or to the log-softmax gives the same argmax, since the normaliser is shared by all classes of a frame.  Everything else is
unchanged: ``max_symbols`` still applies; with confidence on, the statistics are those of the UNFUSED softmax at the fused
decisions; ``Hypothesis.score`` stays the sum of the acoustic log-probabilities of the emitted tokens.  Fusion and phrase
boosting can both be on: their terms add, and each keeps its own state.

Tables (``build_lm_tables``; computed in float64, stored float32, with the decode kernel adding ``cb[s] + w`` in fp32):
  states    every context of order <= N - 1, plus the empty context (state 0).  Per state: ``backoff`` (the longest proper
            suffix that is a state), ``level`` (its order), ``cb`` = alpha * ln10 * the sum of bow over its back-off chain (the
            state, its back-off state, ... ; the root excluded), and ``chain`` [n_states, N - 1] = the state, its back-off
            state, ... padded with 0 (the kernel reads the whole chain with one load instead of walking ``backoff``).
  arcs      CSR ``arc_begin[s] .. arc_begin[s+1]``, sorted by token: ``arc_tok``, ``arc_to`` (the state reached, already the
            longest suffix of s.k that is a state) and ``arc_w = alpha * ln10 * log10p - cb[s]``.  An arc exists for every
            explicit n-gram whose context is a state.  In an ARPA that is not suffix-closed, a suffix u of a state s can lie
            between s and its back-off state without being a state itself; the back-off rule still uses the n-grams u.k, so
            they become "gap" arcs on the lowest chain state ending in u, with ``arc_w = alpha * ln10 * log10p - cb[backoff]``
            (see ``build_lm_tables``).
  root row  the unigram level as two dense rows ``uni_w`` / ``uni_to`` of pitch = vocab_size rounded up to 4.
Then term(k | s) = cb[s] + arc_w of the highest-level arc for k on s's chain, or cb[s] + uni_w[k] when there is none.
"""
from __future__ import annotations

import math
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

MAX_ORDER = 6
LN10 = math.log(10.0)


@dataclass
class NgramLMConfig:
    """An ARPA LM over BPE token ids and its fusion weight ``alpha`` (no default: it depends on the LM and the domain)."""
    path: str
    alpha: float
    token_offset: int = 100

    def validate(self) -> "NgramLMConfig":
        a = float(self.alpha)
        if not (math.isfinite(a) and a > 0.0):
            raise ValueError(f"the LM weight alpha must be finite and > 0, got {self.alpha!r}")
        if int(self.token_offset) < 0:
            raise ValueError(f"token_offset must be >= 0, got {self.token_offset!r}")
        return self


@dataclass
class NgramLMTables:
    """Host tables of an n-gram LM (see the module docstring); ``contexts[s]`` is state s's context as token ids, ``<s>`` as
    ``vocab_size``."""
    order: int
    vocab_size: int
    pitch: int
    start_state: int
    n_ngrams: int
    contexts: List[Tuple[int, ...]]
    backoff: np.ndarray      # i32 [n_states]
    level: np.ndarray        # i32 [n_states]
    cb: np.ndarray           # f32 [n_states]
    chain: np.ndarray        # i32 [n_states, order - 1]
    arc_begin: np.ndarray    # i32 [n_states + 1]
    arc_tok: np.ndarray      # i32 [max(n_arcs, 1)]
    arc_to: np.ndarray       # i32 [max(n_arcs, 1)]
    arc_w: np.ndarray        # f32 [max(n_arcs, 1)]
    uni_w: np.ndarray        # f32 [pitch]
    uni_to: np.ndarray       # i32 [pitch]
    build_seconds: float = 0.0
    _keys: Optional[np.ndarray] = field(default=None, repr=False)

    @property
    def n_states(self) -> int:
        return len(self.cb)

    @property
    def n_arcs(self) -> int:
        return int(self.arc_begin[-1])

    def device_arrays(self) -> Dict[str, np.ndarray]:
        """The arrays the decode kernel reads (rs_ngram_lm's fields)."""
        return {k: getattr(self, k) for k in ("cb", "chain", "arc_begin", "arc_tok", "arc_to", "arc_w", "uni_w", "uni_to")}

    @property
    def nbytes(self) -> int:
        return sum(a.nbytes for a in self.device_arrays().values())


# ---------------------------------------------------------------------------------------------------------------- ARPA parsing
def read_arpa(path: str, vocab_size: int, token_offset: int = 100):
    """-> (N, grams): grams[n] = {word-id tuple: (log10p, log10bow)} for n = 1..N.  Word ids: tokens 0..V-1, ``<s>`` = V,
    ``</s>`` = V + 1, ``<unk>`` = V + 2.  Raises ValueError on a malformed file or an unknown word."""
    V = int(vocab_size)
    special = {"<s>": V, "</s>": V + 1, "<unk>": V + 2}
    ids: Dict[str, int] = {}

    def word_id(w: str) -> int:
        k = ids.get(w)
        if k is None:
            k = special.get(w)
            if k is None:
                k = ord(w) - token_offset if len(w) == 1 else -1
                if not 0 <= k < V:
                    raise ValueError(f"{path}: ARPA word {w!r} is not <s>, </s>, <unk> nor a token: token ids are "
                                     f"ord(word) - {token_offset} in [0, {V})")
            ids[w] = k
        return k

    with open(path, encoding="utf-8") as f:
        lines = f.read().split("\n")          # not splitlines(): token characters may be Unicode line separators
    i, n_lines = 0, len(lines)
    while i < n_lines and lines[i].strip(" \t\r") != "\\data\\":
        i += 1
    if i == n_lines:
        raise ValueError(f"{path}: no \\data\\ section")
    i += 1
    counts: Dict[int, int] = {}
    while i < n_lines:
        ln = lines[i].strip(" \t\r")
        if ln.startswith("ngram "):
            try:
                n, c = ln[6:].split("=")
                counts[int(n)] = int(c)
            except ValueError:
                raise ValueError(f"{path}:{i + 1}: bad count line {ln!r}") from None
        elif ln:
            break
        i += 1
    N = max(counts) if counts else 0
    if sorted(counts) != list(range(1, N + 1)) or N < 2:
        raise ValueError(f"{path}: the \\data\\ counts must list orders 1..N with N >= 2, got {sorted(counts)}")
    if N > MAX_ORDER:
        raise ValueError(f"{path}: LM order {N} exceeds the supported maximum {MAX_ORDER}")
    grams: Dict[int, Dict[Tuple[int, ...], Tuple[float, float]]] = {}
    ended = False
    while i < n_lines:
        ln = lines[i].strip(" \t\r")
        i += 1
        if not ln:
            continue
        if ln == "\\end\\":
            ended = True
            break
        if not (ln.startswith("\\") and ln.endswith("-grams:")):
            raise ValueError(f"{path}:{i}: expected a \\N-grams: section or \\end\\, got {ln!r}")
        try:
            n = int(ln[1:-7])
        except ValueError:
            raise ValueError(f"{path}:{i}: bad section header {ln!r}") from None
        if n not in counts or n in grams:
            raise ValueError(f"{path}:{i}: unexpected section {ln!r}")
        d: Dict[Tuple[int, ...], Tuple[float, float]] = {}
        while i < n_lines:
            raw = lines[i].rstrip("\r")
            if not raw.strip(" \t") or raw.startswith("\\"):
                break
            i += 1
            parts = raw.split("\t")
            if len(parts) not in (2, 3):
                raise ValueError(f"{path}:{i}: expected 'log10p<TAB>words[<TAB>log10bow]', got {raw!r}")
            words = parts[1].strip(" ").split(" ")
            if len(words) != n:
                raise ValueError(f"{path}:{i}: {len(words)} words in the {n}-gram section")
            try:
                lp = float(parts[0])
                bow = float(parts[2]) if len(parts) == 3 and parts[2].strip(" ") else 0.0
            except ValueError:
                raise ValueError(f"{path}:{i}: bad number in {raw!r}") from None
            d[tuple(word_id(w) for w in words)] = (lp, bow)
        if len(d) != counts[n]:
            raise ValueError(f"{path}: \\data\\ declares {counts[n]} {n}-grams, the section has {len(d)}")
        grams[n] = d
    if not ended:
        raise ValueError(f"{path}: no \\end\\ marker")
    missing = [n for n in counts if n not in grams]
    if missing:
        raise ValueError(f"{path}: no section for the {missing[0]}-grams")
    if (V + 2,) not in grams[1]:
        raise ValueError(f"{path}: the LM has no <unk> unigram (tokens without a unigram get <unk>'s probability)")
    return N, grams


# -------------------------------------------------------------------------------------------------------------------- tables
def _is_context(g: Tuple[int, ...], V: int) -> bool:
    """A context the decode can reach: token ids, with <s> allowed only in front."""
    return all(w < V for w in g[1:]) and (g[0] < V or g[0] == V)


def build_lm_tables(cfg: NgramLMConfig, vocab_size: int) -> NgramLMTables:
    """Validated decode tables of ``cfg``'s ARPA for a vocabulary of ``vocab_size`` tokens (see the module docstring)."""
    cfg.validate()
    t0 = time.perf_counter()
    V = int(vocab_size)
    N, grams = read_arpa(cfg.path, V, int(cfg.token_offset))
    scale = float(cfg.alpha) * LN10
    # states: the empty context, then every reachable context of order <= N - 1 by (order, ids)
    contexts: List[Tuple[int, ...]] = [()]
    for n in range(1, N):
        contexts += sorted(g for g in grams[n] if _is_context(g, V))
    sid = {c: s for s, c in enumerate(contexts)}
    S = len(contexts)
    backoff = np.zeros(S, np.int32)
    level = np.array([len(c) for c in contexts], np.int32)
    cb = np.zeros(S, np.float64)
    for s in range(1, S):
        c = contexts[s]
        b = 0
        for i in range(1, len(c)):
            b = sid.get(c[i:], -1)
            if b >= 0:
                break
        backoff[s] = max(b, 0)
        cb[s] = scale * grams[len(c)][c][1] + cb[backoff[s]]
    chain = np.zeros((S, N - 1), np.int32)
    cur = np.arange(S, dtype=np.int32)
    for d in range(N - 1):
        chain[:, d] = cur
        cur = backoff[cur]
    chain[0, :] = 0

    def longest_state(g: Tuple[int, ...]) -> int:
        for i in range(len(g)):
            s = sid.get(g[i:])
            if s is not None:
                return s
        return 0

    # explicit arcs: an n-gram (n >= 2) predicting a token from a context that is a state
    own: List[int] = []
    tok: List[int] = []
    to: List[int] = []
    lp: List[float] = []
    explicit: Dict[Tuple[int, int], float] = {}
    for n in range(2, N + 1):
        for g, (p, _) in grams[n].items():
            k = g[-1]
            o = sid.get(g[:-1])
            if k >= V or o is None:
                continue
            explicit[(o, k)] = p
            own.append(o); tok.append(k); lp.append(p)
            to.append(longest_state(g))
    unk = grams[1][(V + 2,)][0]
    w64 = [scale * p - cb[o] for o, p in zip(own, lp)]
    # gap arcs: a suffix u of a state s that lies strictly between s's back-off state and s is no state (the back-off state is
    # the longest proper suffix that is one), yet the back-off rule still uses the explicit n-grams u.k (bow(u) = 0 then).  Such
    # an arc goes on the lowest chain state o ending in u (len(backoff(o)) < len(u) < len(o)), where every state above it
    # finds it: term(k | s) = cb[s] - cb[backoff(o)] + alpha * ln10 * log10p(u.k), so arc_w = alpha * ln10 * log10p -
    # cb[backoff(o)].  An explicit arc of o itself, or one from a longer u, takes precedence.  Well-formed (suffix-closed)
    # ARPA files have no such gaps.
    gaps: Dict[Tuple[int, ...], List[int]] = {}
    for s in range(1, S):
        c, bl = contexts[s], int(level[backoff[s]])
        for m in range(len(c) - 1, bl, -1):                    # longest u first
            gaps.setdefault(c[-m:], []).append(s)
    if gaps:
        cont: Dict[Tuple[int, ...], List[Tuple[int, float]]] = {}
        for n in range(2, N + 1):
            for g, (p, _) in grams[n].items():
                if g[-1] < V and g[:-1] in gaps:
                    cont.setdefault(g[:-1], []).append((g[-1], p))
        placed = set(explicit)
        for u in sorted(cont, key=len, reverse=True):
            for s in gaps[u]:
                for k, p in cont[u]:
                    if (s, k) not in placed:
                        placed.add((s, k))
                        own.append(s); tok.append(k); to.append(longest_state(contexts[s] + (k,)))
                        w64.append(scale * p - cb[backoff[s]])
    own_a, tok_a = np.array(own, np.int64), np.array(tok, np.int64)
    to_a, w64_a = np.array(to, np.int32), np.array(w64, np.float64)
    order = np.lexsort((tok_a, own_a))
    n_arcs = len(order)
    arc_begin = np.zeros(S + 1, np.int32)
    arc_begin[1:] = np.cumsum(np.bincount(own_a, minlength=S))
    pad = max(n_arcs, 1)
    arc_tok = np.zeros(pad, np.int32); arc_tok[:n_arcs] = tok_a[order]
    arc_to = np.zeros(pad, np.int32); arc_to[:n_arcs] = to_a[order]
    arc_w = np.zeros(pad, np.float32); arc_w[:n_arcs] = w64_a[order]
    pitch = (V + 3) // 4 * 4
    uni64 = np.full(pitch, scale * unk)
    uni_to = np.zeros(pitch, np.int32)
    for g, (p, _) in grams[1].items():
        if g[0] < V:
            uni64[g[0]] = scale * p
            uni_to[g[0]] = sid[g]
    uni64[V:] = 0.0
    return NgramLMTables(order=N, vocab_size=V, pitch=pitch, start_state=sid.get((V,), 0),
                         n_ngrams=sum(len(d) for d in grams.values()), contexts=contexts, backoff=backoff, level=level,
                         cb=cb.astype(np.float32), chain=chain, arc_begin=arc_begin, arc_tok=arc_tok, arc_to=arc_to, arc_w=arc_w,
                         uni_w=uni64.astype(np.float32), uni_to=uni_to, build_seconds=time.perf_counter() - t0)


# -------------------------------------------------------------------------------------------------------------------- lookup
def lookup(tables: NgramLMTables, state, token):
    """The decode kernel's lookup, step for step: fp32 ``cb[s] + uni_w[k]`` and ``uni_to[k]`` (the root row), then every chain
    level from the lowest to the highest overwrites with ``cb[s] + arc_w`` / ``arc_to`` of its arc for k.  ``state`` and
    ``token`` are scalars or arrays of one shape; a state outside [0, n_states) counts as the root.  -> (score f32, next i32)."""
    t = tables
    s = np.asarray(state, np.int64)
    k = np.asarray(token, np.int64)
    scalar = s.ndim == 0 and k.ndim == 0
    s, k = np.broadcast_arrays(np.atleast_1d(s), np.atleast_1d(k))
    if np.any((k < 0) | (k >= t.vocab_size)):
        raise ValueError("token outside [0, vocab_size)")
    s = np.where((s >= 0) & (s < t.n_states), s, 0)
    if t._keys is None:                                         # arcs are sorted by (state, token): one global key
        owner = np.repeat(np.arange(t.n_states, dtype=np.int64), np.diff(t.arc_begin))
        t._keys = owner * t.pitch + t.arc_tok[:t.n_arcs].astype(np.int64)
    cbs = t.cb[s]
    score = (cbs + t.uni_w[k]).astype(np.float32)
    nxt = t.uni_to[k].astype(np.int32)
    for d in reversed(range(t.order - 1)):
        o = t.chain[s, d].astype(np.int64)
        key = o * t.pitch + k
        pos = np.searchsorted(t._keys, key)
        hit = (o > 0) & (pos < t.n_arcs)
        hit[hit] = t._keys[pos[hit]] == key[hit]
        score = np.where(hit, cbs + t.arc_w[np.minimum(pos, len(t.arc_w) - 1)], score).astype(np.float32)
        nxt = np.where(hit, t.arc_to[np.minimum(pos, len(t.arc_to) - 1)], nxt).astype(np.int32)
    if scalar:
        return np.float32(score[0]), int(nxt[0])
    return score, nxt
