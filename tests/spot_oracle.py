"""Restatement of keyword spotting (reazonspeech_b200/keywords.py): the per-end-frame segment recursion with its backtrace,
brute-force enumeration of every segment path ending at each frame, and the hit policy in two forms (the iterative rule and
a sort-then-accept scan).  ``dtype=np.float32`` repeats the kernel's fp32 arithmetic step for step (every value is one
rounded addition, so numpy's float32 gives the kernel's bits); the default is float64."""
import itertools

import numpy as np

import segment_oracle as SO


def spot(lpb, lpe, T, U, dtype=np.float64):
    """-> dict(E [T], S [T] (int), choice [T, U + 1] (1: the emission from (t, u - 1)), margin [T]: the smallest
    predecessor gap |blank - emission| along the path to (e, U))."""
    lpb = np.asarray(lpb, dtype=dtype); lpe = np.asarray(lpe, dtype=dtype)
    d = np.zeros((T, U + 1), dtype=dtype)
    st = np.zeros((T, U + 1), dtype=np.int64)
    ch = np.zeros((T, U + 1), dtype=np.int8)
    pm = np.full((T, U + 1), np.inf)
    for t in range(T):
        st[t, 0] = t
        for u in range(1, U + 1):
            ve = dtype(d[t, u - 1] + lpe[t, u - 1])
            vb = dtype(d[t - 1, u] + lpb[t - 1, u]) if t > 0 else dtype(-np.inf)
            ch[t, u] = 1 if (t == 0 or ve > vb) else 0
            if ch[t, u]:
                d[t, u], st[t, u] = ve, st[t, u - 1]
                pm[t, u] = pm[t, u - 1] if u > 1 else np.inf
            else:
                d[t, u], st[t, u] = vb, st[t - 1, u]
                pm[t, u] = pm[t - 1, u]
            if t > 0:
                pm[t, u] = min(pm[t, u], abs(float(vb) - float(ve)))
    E = np.array([dtype(d[e, U] + lpb[e, U]) for e in range(T)], dtype=dtype)
    return dict(E=E, S=st[:, U].copy(), choice=ch, margin=pm[:, U].copy())


def backtrace(choice, lpe, e, U):
    """The path to (e, U) through ``choice`` -> (frames [U], token_lp [U])."""
    frames, token_lp = np.full(U, -1, dtype=np.int64), np.full(U, np.nan, dtype=np.asarray(lpe).dtype)
    t, u = e, U
    while u > 0:
        if choice[t, u]:
            frames[u - 1] = t; token_lp[u - 1] = lpe[t, u - 1]; u -= 1
        else:
            t -= 1
    return frames, token_lp


def frame_lp(lpb, lpe, frames, e, U):
    """Per-frame log-probabilities of the segment path with token frames ``frames`` ending at e (segment_oracle's frame_lp):
    frame t holds its emissions and the blank that leaves it."""
    s = int(frames[0])
    out = np.zeros(e - s + 1)
    for u, t in enumerate(frames):
        out[t - s] += lpe[t, u]
        nxt = frames[u + 1] if u + 1 < U else e + 1
        for k in range(t, nxt):
            out[k - s] += lpb[k, u + 1]
    return out


def brute_force(lpb, lpe, T, U):
    """For every end frame e, the best segment path ending there over every choice of token frames t_1 <= ... <= t_U <= e,
    under the tie rule (the smallest t_U, then t_{U-1}, ...: the blank predecessor wins) -> (E [T], S [T], frames [T][U])."""
    E, S, F = np.full(T, -np.inf), np.full(T, -1, dtype=np.int64), []
    for e in range(T):
        best = None
        for frames in itertools.combinations_with_replacement(range(e + 1), U):
            key = (-SO.path_score(lpb, lpe, frames, e, U), frames[::-1])
            if best is None or key < best[0]:
                best = (key, frames)
        E[e], S[e] = -best[0][0], best[1][0]
        F.append(np.array(best[1], dtype=np.int64))
    return E, S, F


def mean_lp(E, S):
    """m(e) = E(e) / (e - S(e) + 1) in float32, as the kernel divides."""
    E = np.asarray(E, dtype=np.float32)
    n = (np.arange(len(E)) - np.asarray(S) + 1).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (E / n).astype(np.float32)


def pick(E, S, T, threshold, max_hits):
    """The hit policy, iteratively: the candidate with the largest m (the smaller e on a tie), then every candidate whose
    span intersects it dropped -> [(s, e, m)] in pick order."""
    m = mean_lp(E[:T], S[:T])
    alive = [e for e in range(T) if S[e] >= 0 and m[e] >= np.float32(threshold)]
    hits = []
    while alive and len(hits) < max_hits:
        e = min(alive, key=lambda x: (-m[x], x))
        s = int(S[e])
        hits.append((s, e, m[e]))
        alive = [x for x in alive if not (S[x] <= e and x >= s)]
    return hits


def pick_sorted(E, S, T, threshold, max_hits):
    """The same policy as a scan: the candidates sorted by (-m, e), each accepted unless it intersects an accepted hit."""
    m = mean_lp(E[:T], S[:T])
    cands = sorted((e for e in range(T) if S[e] >= 0 and m[e] >= np.float32(threshold)), key=lambda x: (-m[x], x))
    hits = []
    for e in cands:
        if len(hits) == max_hits:
            break
        if all(S[e] > he or e < hs for hs, he, _ in hits):
            hits.append((int(S[e]), e, m[e]))
    return hits
