"""Float64 restatement of the segment alignment (reazonspeech_b200/alignment.py, "Segment alignment") and a brute-force
enumeration of every segment path that pins it on small shapes."""
import itertools

import numpy as np

import align_oracle as A

# share of planted captions whose located segment must overlap the planted frames on lattices where the caption's tokens are
# likely only where they were said, as a trained model's are; the DPs without a free start or without a free end stay below
# it (tests/test_align_captions_cpu.py::test_free_start_and_free_end_are_needed)
PLANTED_BAR = 0.9


def segment_align(lpb, lpe, T, U, free_start=True, free_end=True):
    """Viterbi with a free start (row 0 costs nothing at every frame) and a free end (the best t of delta[t][U] +
    lp_blank[t][U], the smallest on a tie), the backtrace (blank wins an exact tie), frame_lp and the forward recursion on
    rows [s, e] -> dict(score, s, e, frames [U], token_lp [U], frame_lp [T] (NaN outside [s, e]), loglik, margin), margin the
    smallest gap of any decision the result rests on: the predecessor choices along the path and the end frame.
    ``free_start`` / ``free_end`` False give the variants that start at (0, 0) through row 0's blanks / end at T - 1 (they
    show what the free ends buy)."""
    d = np.full((T, U + 1), -np.inf)
    ch = np.zeros((T, U + 1), dtype=np.int8)
    gap = np.full((T, U + 1), np.inf)
    for t in range(T):
        for u in range(U + 1):
            if u == 0:
                d[t, 0] = 0.0 if free_start else (0.0 if t == 0 else d[t - 1, 0] + lpb[t - 1, 0])
                continue
            vb = d[t - 1, u] + lpb[t - 1, u] if t > 0 else -np.inf
            ve = d[t, u - 1] + lpe[t, u - 1]
            ch[t, u] = 1 if (t == 0 or ve > vb) else 0
            d[t, u] = ve if ch[t, u] else vb
            if t > 0:
                gap[t, u] = abs(vb - ve)
    ends = d[:, U] + lpb[:T, U]
    e = int(np.argmax(ends)) if free_end else T - 1                # argmax: the first maximum
    score = float(ends[e])
    others = np.delete(ends, e)
    margin = float(score - others.max()) if (free_end and others.size) else np.inf
    frames = np.full(U, -1, dtype=np.int64); token_lp = np.full(U, np.nan); frame_lp = np.full(T, np.nan)
    t, u = e, U
    acc = lpb[e, U]
    while u > 0:
        margin = min(margin, gap[t, u])
        if ch[t, u]:
            frames[u - 1] = t; token_lp[u - 1] = lpe[t, u - 1]; acc += lpe[t, u - 1]; u -= 1
        else:
            frame_lp[t] = acc; t -= 1; acc = lpb[t, u]
    if not free_start:                                              # row 0's blanks before token 1 are frames of the path too
        while t > 0:
            frame_lp[t] = acc; t -= 1; acc = lpb[t, 0]
    frame_lp[t] = acc
    s = t if free_start else int(frames[0])
    loglik = A.align(lpb[s:e + 1], lpe[s:e + 1], e - s + 1, U)["loglik"]
    return dict(score=score, s=s, e=e, frames=frames, token_lp=token_lp, frame_lp=frame_lp, loglik=loglik, margin=margin)


def path_score(lpb, lpe, frames, e, U):
    """Score of the segment path with token frames t_1 <= ... <= t_U <= e: the emissions, the blanks between them on each
    row, and the blanks of row U from t_U through the final one at e."""
    s = 0.0
    for u, tu in enumerate(frames):
        if u > 0:
            s += sum(lpb[k, u] for k in range(frames[u - 1], tu))
        s += lpe[tu, u]
    return s + sum(lpb[k, U] for k in range(frames[-1], e + 1))


def brute_force(lpb, lpe, T, U):
    """Every segment path (token frames t_1 <= ... <= t_U, end e >= t_U) -> (score, s, e, frames) of the best one under
    the tie rules: the largest score, then the smallest e, then the smallest t_U, t_{U-1}, ... (the blank predecessor wins)."""
    best = None
    for frames in itertools.combinations_with_replacement(range(T), U):
        for e in range(frames[-1], T):
            key = (-path_score(lpb, lpe, frames, e, U), e, frames[::-1])
            if best is None or key < best[0]:
                best = (key, frames, e)
    (neg, _, _), frames, e = best
    return -neg, frames[0], e, np.array(frames, dtype=np.int64)
