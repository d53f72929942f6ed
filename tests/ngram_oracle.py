"""Test oracle of the n-gram LM fusion (never imported by the product).

``ArpaOracle``: a brute-force float64 ARPA scorer written from the module docstring of reazonspeech_b200/ngram_lm.py alone --
dictionary lookup with the back-off recursion, and the longest-suffix state.  ``write_arpa``: a seeded ARPA writer (absolute
discounting over token sequences of a seeded sparse Markov source), for the tests and scripts/bench_ngram_lm.py.
``greedy_fused``: the boosted greedy oracle of tests/boosting_oracle.py with the LM term (and optionally the boosting bonus)
added to the fp32 logits of every non-blank class."""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np

LN10 = math.log(10.0)


class ArpaOracle:
    """Contexts are tuples of token ids with ``<s>`` as ``V``; ``score`` is alpha * ln10 * log10 P(k | h) in float64."""

    def __init__(self, path: str, V: int, alpha: float, token_offset: int = 100):
        self.V, self.alpha = V, alpha
        self.grams: Dict[Tuple[int, ...], Tuple[float, float]] = {}
        section = 0
        for raw in open(path, encoding="utf-8").read().split("\n"):
            line = raw.rstrip("\r")
            if line.startswith("\\") and line.endswith("-grams:"):
                section = int(line[1:-7])
                continue
            if section == 0 or not line.strip(" \t") or line.startswith("\\"):
                continue
            f = line.split("\t")
            words = f[1].split(" ")
            ids = []
            for w in words:
                ids.append({"<s>": V, "</s>": V + 1, "<unk>": V + 2}.get(w, ord(w) - token_offset if len(w) == 1 else None))
            self.grams[tuple(ids)] = (float(f[0]), float(f[2]) if len(f) > 2 else 0.0)
        self.order = max(len(g) for g in self.grams)
        self.states = {g for g in self.grams if len(g) < self.order and all(w < V for w in g[1:]) and g[0] <= V}
        self.states.add(())
        self.start = (V,) if (V,) in self.grams else ()
        self._rows: Dict[Tuple[int, ...], np.ndarray] = {}
        self._cont: Dict[Tuple[int, ...], list] = {}

    def log10p(self, h: Tuple[int, ...], k: int) -> float:
        if h + (k,) in self.grams:
            return self.grams[h + (k,)][0]
        if not h:
            return self.grams[(self.V + 2,)][0]                     # <unk>
        bow = self.grams[h][1] if h in self.grams else 0.0
        return bow + self.log10p(h[1:], k)

    def row(self, h) -> np.ndarray:
        """score(h, k) for every token k at once (float64), by the same back-off recursion; memoised per context."""
        h = tuple(h)
        r = self._rows.get(h)
        if r is None:
            if not self._cont:
                for g, (lp, _) in self.grams.items():
                    if g[-1] < self.V:
                        self._cont.setdefault(g[:-1], []).append((g[-1], lp))
            if not h:
                r = np.full(self.V, self.grams[(self.V + 2,)][0])
            else:
                r = (self.grams[h][1] if h in self.grams else 0.0) + self.row(h[1:]) / (self.alpha * LN10)
            for k, lp in self._cont.get(h, ()):
                r[k] = lp
            r = self.alpha * LN10 * r
            self._rows[h] = r
        return r

    def score(self, h, k) -> float:
        return self.alpha * LN10 * self.log10p(tuple(h), int(k))

    def next(self, h, k) -> Tuple[int, ...]:
        g = tuple(h) + (int(k),)
        for i in range(len(g) + 1):
            if g[i:] in self.states:
                return g[i:]
        return ()


def write_arpa(path: str, V: int, order: int, n_sentences: int, seed: int = 0, token_offset: int = 100, discount: float = 0.5,
               fanout: int = 12, sentence_len: Tuple[int, int] = (8, 40), p_unk: float = 0.01, min_count_top: int = 1) -> int:
    """A seeded ARPA of the given order over tokens 0..V-1 (about 5 % of the tokens never occur: they back off to <unk>).  The
    source is a sparse first-order Markov chain (``fanout`` Zipf-weighted successors per token); n-gram probabilities use
    absolute discounting, bow(h) = the discounted mass, not renormalised (the scorer needs no normalised LM).  n-grams of the
    highest order seen fewer than ``min_count_top`` times are dropped.  Returns the number of n-grams written."""
    rng = np.random.default_rng(seed)
    W = V + 2                                                       # ids: tokens, <s> = V, </s> = V + 1
    assert W ** order < 2 ** 62
    live = np.sort(rng.choice(V, size=max(2, int(V * 0.95)), replace=False))
    succ = rng.choice(live, size=(V, fanout))
    zipf = 1.0 / np.arange(1, fanout + 1)
    zipf /= zipf.sum()
    lens = rng.integers(sentence_len[0], sentence_len[1] + 1, size=n_sentences)
    T = int(lens.max())
    seq = np.empty((n_sentences, T), np.int64)
    seq[:, 0] = rng.choice(live, size=n_sentences)
    for t in range(1, T):
        seq[:, t] = succ[seq[:, t - 1], rng.choice(fanout, size=n_sentences, p=zipf)]
    padded = np.full((n_sentences, T + 2), -1, np.int64)
    padded[:, 0] = V
    for i, n in enumerate(lens):
        padded[i, 1:n + 1] = seq[i, :n]
        padded[i, n + 1] = V + 1
    keys, counts = {}, {}
    for n in range(1, order + 1):
        win = np.lib.stride_tricks.sliding_window_view(padded, n, axis=1).reshape(-1, n)
        win = win[(win >= 0).all(axis=1)]
        k = np.zeros(len(win), np.int64)
        for j in range(n):
            k = k * W + win[:, j]
        u, c = np.unique(k, return_counts=True)
        if n == order and min_count_top > 1:
            u, c = u[c >= min_count_top], c[c >= min_count_top]
        keys[n], counts[n] = u, c

    def words(key: np.ndarray, n: int) -> np.ndarray:
        out = np.empty((len(key), n), np.int64)
        for j in range(n - 1, -1, -1):
            out[:, j] = key % W
            key = key // W
        return out

    def name(w: int) -> str:
        return "<s>" if w == V else "</s>" if w == V + 1 else chr(w + token_offset)

    lines: Dict[int, List[str]] = {}
    logp: Dict[int, np.ndarray] = {}
    bows: Dict[int, Dict[int, float]] = {}
    total = counts[1].sum()
    for n in range(1, order + 1):
        if n == 1:
            p = counts[1] / total * (1.0 - p_unk)
        else:
            prefix = keys[n] // W
            up, inv, ctx_types = np.unique(prefix, return_inverse=True, return_counts=True)
            ctx_count = np.bincount(inv, weights=counts[n])
            p = (counts[n] - discount) / ctx_count[inv]
            bows[n - 1] = dict(zip(up.tolist(), np.log10(discount * ctx_types / ctx_count).tolist()))
        logp[n] = np.log10(np.maximum(p, 1e-99))
    out_counts = {}
    for n in range(1, order + 1):
        ws = words(keys[n].copy(), n)
        bw = bows.get(n, {})
        L = []
        for key, row, lp in zip(keys[n].tolist(), ws.tolist(), logp[n].tolist()):
            if n == 1 and row[0] == V:
                lp = -99.0
            b = bw.get(key)
            text = " ".join(name(w) for w in row)
            L.append(f"{lp:.6f}\t{text}\t{b:.6f}" if b is not None and n < order else f"{lp:.6f}\t{text}")
        if n == 1:
            L.append(f"{math.log10(p_unk):.6f}\t<unk>")
        lines[n] = L
        out_counts[n] = len(L)
    with open(path, "w", encoding="utf-8") as f:
        f.write("\\data\\\n")
        for n in range(1, order + 1):
            f.write(f"ngram {n}={out_counts[n]}\n")
        for n in range(1, order + 1):
            f.write(f"\n\\{n}-grams:\n")
            f.write("\n".join(lines[n]))
            f.write("\n")
        f.write("\n\\end\\\n")
    return sum(out_counts.values())


def greedy_fused(enc, sd, cfg, lm: "ArpaOracle", boost=None, follow=None):
    """``boosting_oracle.greedy_boosted`` with the LM: the fp32 logits + (boosting bonus +) the oracle's LM row of the
    utterance's context (float64 brute force, rounded to fp32) over the V non-blank columns.  Returns a BoostedResult
    (``changed``: decisions whose fused argmax differs from the unfused one) with ``orders``: the order of the LM context
    (``<s>`` counted) each decision was made in."""
    import torch
    import torch.nn.functional as F
    from boosting_oracle import BoostedResult
    from oracle import nemo_restated as O
    V = cfg.vocab_size
    res = BoostedResult()
    res.orders = []
    ep = O.joint_enc_proj(O._q(enc, True), sd)
    bonus = None if boost is None else torch.as_tensor(np.asarray(boost[0]), dtype=torch.float32)
    n_threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        with torch.no_grad():
            emb = sd["decoder.prediction.embed.weight"]
            h = torch.zeros(cfg.pred_hidden); c = torch.zeros(cfg.pred_hidden)
            h_new, c_new = O.lstm_step(torch.zeros(cfg.pred_hidden), h, c, sd)
            pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
            W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
            ctx, bs, i = lm.start, 0, 0
            for t in range(ep.shape[0]):
                for _ in range(cfg.max_symbols):
                    logits = F.linear(torch.relu(ep[t] + pp), W, b)
                    add = torch.from_numpy(lm.row(ctx).astype(np.float32))
                    if bonus is not None:
                        add = bonus[bs, :V] + add
                    scores = logits.clone()
                    scores[:V] = logits[:V] + add
                    top2 = torch.topk(scores, 2)
                    best = int(top2.indices[0])
                    res.margins.append(float(top2.values[0] - top2.values[1]))
                    res.changed += int(best != int(torch.argmax(logits)))
                    res.orders.append(len(ctx))
                    if follow is None:
                        k = best
                    else:
                        if i >= len(follow):
                            res.complete = False
                            return res
                        k = int(follow[i])
                        if k != best:
                            res.gaps.append((i, t, k, best, float(top2.values[0] - scores[k])))
                    i += 1
                    res.decisions.append(k)
                    if k == cfg.blank:
                        break
                    res.tokens.append(k); res.frames.append(t)
                    ctx = lm.next(ctx, k)
                    if boost is not None:
                        nx = int(boost[1][bs, k])
                        bs = nx if 0 <= nx < bonus.shape[0] else 0
                    h, c = h_new, c_new
                    h_new, c_new = O.lstm_step(emb[k], h, c, sd)
                    pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
        if follow is not None:
            res.complete = i == len(follow)
        return res
    finally:
        torch.set_num_threads(n_threads)
