"""Float64 restatement of banded alignment (reazonspeech_b200/alignment.py, "Banded alignment"): forced alignment's recursions
and backtrace with every cell outside lo[u] <= t < hi[u] at -inf, the edge count, and a brute-force enumeration of the
band-restricted lattice paths that pins them on small shapes."""
import itertools

import numpy as np

import align_oracle as A


def masked(lpb, lpe, lo, hi, T, U):
    """lp_blank / lp_emit [T, U + 1] with every cell outside the band at -inf."""
    t = np.arange(T)[:, None]
    inside = (t >= np.asarray(lo)[None, : U + 1]) & (t < np.asarray(hi)[None, : U + 1])
    return np.where(inside, lpb[:T, : U + 1], -np.inf), np.where(inside, lpe[:T, : U + 1], -np.inf)


def edge_count(frames, lo, hi, T):
    """Tokens u = 1..U (the step from row u - 1 to u at frame frames[u - 1]) with t = lo[u] > 0 or t = hi[u - 1] - 1 < T - 1."""
    return int(sum((t == lo[u] and lo[u] > 0) or (t == hi[u - 1] - 1 and hi[u - 1] < T) for u, t in enumerate(frames, 1)))


def align(lpb, lpe, lo, hi, T, U):
    """The recursions of align_oracle.align on the band: the blank predecessor exists iff (t - 1, u) is in the band, so an
    in-band cell at t = lo[u] takes its emission predecessor, as the kernel does -> align_oracle's dict plus edge."""
    b, e = masked(lpb, lpe, lo, hi, T, U)
    fa = np.full((T, U + 1), -np.inf); va = np.full((T, U + 1), -np.inf)
    ch = np.zeros((T, U + 1), dtype=np.int8); margin = np.full((T, U + 1), np.inf)
    for t in range(T):
        for u in range(U + 1):
            if not lo[u] <= t < hi[u]:
                continue
            if t == 0 and u == 0:
                fa[0, 0] = va[0, 0] = 0.0
                continue
            has_b = t - 1 >= lo[u]
            has_e = u > 0 and lo[u - 1] <= t < hi[u - 1]
            fb = vb = fe = ve = -np.inf
            if has_b:
                fb, vb = fa[t - 1, u] + b[t - 1, u], va[t - 1, u] + b[t - 1, u]
            if has_e:
                fe, ve = fa[t, u - 1] + e[t, u - 1], va[t, u - 1] + e[t, u - 1]
            fa[t, u] = np.logaddexp(fb, fe)
            ch[t, u] = 1 if (not has_b or ve > vb) else 0
            va[t, u] = ve if ch[t, u] else vb
            if has_b and has_e:
                margin[t, u] = abs(vb - ve)
    frames = np.full(U, -1, dtype=np.int64); token_lp = np.full(U, np.nan)
    t, u, path_margin = T - 1, U, np.inf
    while u > 0:
        path_margin = min(path_margin, margin[t, u])
        if ch[t, u]:
            frames[u - 1] = t; token_lp[u - 1] = e[t, u - 1]; u -= 1
        else:
            t -= 1
    return dict(loglik=fa[T - 1, U] + b[T - 1, U], viterbi=va[T - 1, U] + b[T - 1, U], frames=frames, token_lp=token_lp,
                path_margin=path_margin, edge=edge_count(frames, lo, hi, T))


def brute_force(lpb, lpe, lo, hi, T, U):
    """Every monotone path that stays inside the band (align_oracle.brute_force's enumeration and tie rule) -> (logsumexp of
    the path scores, max score, frames of the best path)."""
    scores, best, best_frames = [], -np.inf, None
    for frames in itertools.combinations_with_replacement(range(T), U):
        cells = []
        t = 0
        for u, tu in enumerate(frames):
            cells += [(k, u) for k in range(t, tu + 1)]
            t = tu
        cells += [(k, U) for k in range(t, T)]
        if not all(lo[u] <= k < hi[u] for k, u in cells):
            continue
        s, t = 0.0, 0
        for u, tu in enumerate(frames):
            s += sum(lpb[k, u] for k in range(t, tu)) + lpe[tu, u]; t = tu
        s += sum(lpb[k, U] for k in range(t, T))
        scores.append(s)
        if best_frames is None or s > best or (s == best and frames[::-1] < best_frames[::-1]):
            best, best_frames = s, frames
    return float(np.logaddexp.reduce(scores)), float(best), np.array(best_frames, dtype=np.int64)


def valid_bands(T, U):
    """Every valid band over T frames and U labels (small shapes only)."""
    rows = [(l, h) for l in range(T) for h in range(l + 1, T + 1)]
    for band in itertools.product(rows, repeat=U + 1):
        lo = [x for x, _ in band]; hi = [y for _, y in band]
        if lo[0] != 0 or hi[U] != T:
            continue
        if any(lo[u + 1] < lo[u] or hi[u + 1] < hi[u] or lo[u + 1] >= hi[u] for u in range(U)):
            continue
        yield np.array(lo), np.array(hi)


def rows_of(x, lo, hi):
    """A [T, U + 1] lattice as banded rows: row u = x[lo[u]:hi[u], u]."""
    return [np.asarray(x[lo[u]:hi[u], u], dtype=np.float64) for u in range(len(lo))]


def align_rows(lpb_rows, lpe_rows, lo, hi, T, U):
    """The recursions of ``align`` row by row on banded rows (row u: the frames [lo[u], hi[u])), for shapes too large for the
    dense loops: within a row the blank chain is a running max / logaddexp of the emission terms minus the row's blank prefix
    sums -> dict(loglik, viterbi, frames, path_margin, edge)."""
    prev_f = prev_v = None
    choice, margin = [], []
    for u in range(U + 1):
        l, h = int(lo[u]), int(hi[u])
        b = lpb_rows[u]
        e_f = np.full(h - l, -np.inf); e_v = np.full(h - l, -np.inf)
        if u == 0:
            e_f[0] = e_v[0] = 0.0
        else:
            pl, s, t1 = int(lo[u - 1]), max(l, int(lo[u - 1])), min(h, int(hi[u - 1]))
            e_f[s - l:t1 - l] = prev_f[s - pl:t1 - pl] + lpe_rows[u - 1][s - pl:t1 - pl]
            e_v[s - l:t1 - l] = prev_v[s - pl:t1 - pl] + lpe_rows[u - 1][s - pl:t1 - pl]
        C = np.concatenate([[0.0], np.cumsum(b[:-1])])
        v = C + np.maximum.accumulate(e_v - C)
        f = C + np.logaddexp.accumulate(e_f - C)
        vb = np.concatenate([[-np.inf], v[:-1] + b[:-1]])
        ch = (e_v > vb)
        ch[0] = True
        choice.append(ch)
        margin.append(np.where(np.isfinite(vb) & np.isfinite(e_v), np.abs(vb - e_v), np.inf))
        prev_f, prev_v = f, v
    frames = np.full(U, -1, dtype=np.int64)
    t, u, path_margin = T - 1, U, np.inf
    while u > 0:
        path_margin = min(path_margin, margin[u][t - lo[u]])
        if choice[u][t - lo[u]]:
            frames[u - 1] = t; u -= 1
        else:
            t -= 1
    last = T - 1 - int(lo[U])
    return dict(loglik=prev_f[last] + lpb_rows[U][last], viterbi=prev_v[last] + lpb_rows[U][last], frames=frames,
                path_margin=path_margin, edge=edge_count(frames, lo, hi, T))
