"""Restatement of streaming keyword spotting (reazonspeech_b200/keywords.py, "Streaming"): the recursion of
``spot_oracle.spot`` run chunk by chunk from a carried column, with the forward traceback (each row keeps the token frames and
lp_emit of the path to its current cell), and after every chunk the natural cut, the forced cut, the greedy pick over the
decided candidates and the barrier.  ``decide`` is the policy alone, on given E and S, so it can be applied to the kernel's."""
import numpy as np

import spot_oracle as K


def decide(pending, E, S, sigma, t, last, D, barrier):
    """One step's decisions.  pending: the candidate end frames not yet decided (ascending); sigma: sigma(t) after the step;
    t: the step's last frame; barrier: the largest reported end frame (-1: none) -> (hits [(s, e, m, forced)] in e order,
    still pending, new barrier, forced cut?, the natural cut L)."""
    m = {e: K.mean_lp(np.array([E[e]]), np.array([S[e] - e]))[0] for e in pending}   # m(e) in fp32: E / (e - S + 1)
    if last:
        L = np.inf
    else:
        L = sigma
        while True:
            nl = min([L] + [S[e] for e in pending if e >= L])
            if nl == L:
                break
            L = nl
    cut = L
    if not last and any(e >= L and t - e >= D for e in pending):
        cut = t + 1 - D
    decided = [e for e in pending if e < cut]
    alive = [e for e in decided if S[e] > barrier]
    hits = []
    while alive:
        e = min(alive, key=lambda x: (-m[x], x))
        s = int(S[e])
        hits.append((s, e, m[e], bool(e >= L)))
        alive = [x for x in alive if not (S[x] <= e and x >= s)]
    hits.sort(key=lambda h: h[1])
    barrier = max([barrier] + [h[1] for h in hits])
    return hits, [e for e in pending if e >= cut], barrier, cut > L, L


def stream(lpb, lpe, T, U, chunks, threshold, D, dtype=np.float64):
    """The recursion over frames [0, T) in chunks of the given sizes (their sum is T; empty chunks allowed), the stream closed
    at the last one -> dict(E [T], S [T], sigma [per chunk, after it], hits [(s, e, m, forced, frames, token_lp)] in decision
    order, hit_step [the chunk that decided each hit], forced_cuts, pending_after [per chunk: the candidates still pending],
    natural [per chunk: the natural cut])."""
    lpb = np.asarray(lpb, dtype=dtype); lpe = np.asarray(lpe, dtype=dtype)
    v = np.zeros(U + 1, dtype=dtype); lb = np.zeros(U + 1, dtype=dtype); st = np.zeros(U + 1, dtype=np.int64)
    lists = [[] for _ in range(U + 1)]
    E = np.full(T, np.nan, dtype=dtype); S = np.full(T, -1, dtype=np.int64)
    paths, pending, barrier = {}, [], -1
    out = dict(sigma=[], hits=[], hit_step=[], forced_cuts=0, pending_after=[], natural=[])
    t0 = 0
    for i, n in enumerate(chunks):
        for t in range(t0, t0 + n):
            nv, nst, nlists = v.copy(), st.copy(), [list(x) for x in lists]
            nv[0], nst[0], nlists[0] = dtype(0), t, []
            for u in range(1, U + 1):
                ve = dtype(nv[u - 1] + lpe[t, u - 1])
                vb = dtype(v[u] + lb[u]) if t > 0 else dtype(-np.inf)
                if t == 0 or ve > vb:                         # an exact tie goes to the blank predecessor
                    nv[u], nst[u] = ve, (t if u == 1 else nst[u - 1])
                    nlists[u] = nlists[u - 1] + [(t, lpe[t, u - 1])]
                else:
                    nv[u], nst[u] = vb, st[u]
            v, st, lists = nv, nst, nlists
            lb = lpb[t].copy()
            E[t], S[t] = dtype(v[U] + lpb[t, U]), st[U]
            if K.mean_lp(np.array([E[t]]), np.array([S[t] - t]))[0] >= np.float32(threshold):
                pending.append(t)
                paths[t] = lists[U]
        t0 += n
        if t0 == 0:
            out["sigma"].append(-1); out["pending_after"].append([]); out["natural"].append(None)
            continue
        sigma = int(st[1:].min())
        last = i == len(chunks) - 1
        hits, pending, barrier, forced, L = decide(pending, E, S, sigma, t0 - 1, last, D, barrier)
        out["forced_cuts"] += forced
        out["sigma"].append(sigma); out["pending_after"].append(list(pending)); out["natural"].append(L)
        for s, e, m, f in hits:
            fr = np.array([x[0] for x in paths[e]]); tl = np.array([x[1] for x in paths[e]], dtype=dtype)
            out["hits"].append((s, e, m, f, fr, tl))
            out["hit_step"].append(i)
    out.update(E=E, S=S)
    return out
