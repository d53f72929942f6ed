"""Shared pieces of the ALSD N-best tests (tests/test_alsd_nbest_cpu.py without a GPU, tests/test_gpu_alsd_nbest.py on one):
the insertion rule of alsd_select_kernel restated in Python, NeMo's `final` list rebuilt from the engine's trace or from a
crafted constant-row joint with the oracle's own step (oracle/alsd_restated.py::alsd_step), and the comparison of
rs_rnnt_alsd_nbest's output with such a list."""
import torch

import alsd_cases as AC
from oracle.alsd_restated import BeamHyp, alsd_step


def key_fn(score_norm):
    return (lambda h: h.score / len(h.y)) if score_norm else (lambda h: h.score)


def insert(held, key, item, n_best):
    """The kernel's rule: ``held`` is a list of (key, item) sorted best first; the new entry goes after every held entry whose
    key is >= its key; a full list drops it when no held key is below it, and otherwise loses its last entry."""
    pos = sum(1 for k, _ in held if k >= key)          # held is sorted: the entries whose key is >= key are a prefix
    if pos == n_best:
        return
    held.insert(pos, (key, item))
    del held[n_best:]


def ranked(pool, score_norm, n_best=None):
    """NeMo's list: the stable sorted(pool, key, reverse=True), first n_best."""
    out = sorted(pool, key=key_fn(score_norm), reverse=True)
    return out if n_best is None else out[:n_best]


def final_from_trace(tr, b, T, beam, u_max, score_norm, recombine_returns_input, blank):
    """NeMo's `final` of utterance b rebuilt by replaying the engine's trace through the oracle's step (each step starts from
    the engine's own beam and log-probabilities, as alsd_cases.replay does) -> (pool, from_final): the finished hypotheses in
    append order, or the last beam in slot order when none finished."""
    prev = [BeamHyp([blank], 0.0, [-1], None)]
    final = []
    for i in range(T + u_max):
        rows = []
        for k, h in enumerate(prev):
            t = i - (len(h.y) - 1)
            if t > T - 1:
                rows.append(None)
                continue
            lp = tr["cand_logp"][i, b, k]
            rows.append((float(lp[0]), [float(x) for x in lp[1:1 + beam]], [int(x) for x in tr["cand_tok"][i, b, k, :beam]], None))
        new = alsd_step(prev, rows, i, T, beam, recombine_returns_input, final)
        if new is None:
            break
        assert int(tr["n_hyp"][i, b]) == len(new), (b, i)
        prev = [BeamHyp(h.y, float(tr["beam_score"][i, b, k]), h.timestamp, None) for k, h in enumerate(new)]
    return (final, True) if final else (prev, False)


def constant_row_pool(sd, cfg, T, beam, u_max, recombine_returns_input=True, row=None):
    """The oracle's search on a crafted joint where every row has the same log-probabilities (alsd_cases.crafted_sd) ->
    (pool, from_final) as ``final_from_trace`` returns them.  ``row``: (log p(blank), top values, top classes) to use instead
    of the oracle's float32 log_softmax of the bias (e.g. the engine's own row)."""
    blank = cfg.blank
    if row is None:
        lp = torch.log_softmax(sd["joint.joint_net.2.bias"], -1)
        top = torch.cat((lp[:blank], lp[blank + 1:])).topk(beam)
        row = (float(lp[blank]), top.values.tolist(), [k + (1 if k >= blank else 0) for k in top.indices.tolist()])
    row = tuple(row) + (None,)
    B, final = [BeamHyp([blank], 0.0, [-1], None)], []
    for i in range(T + u_max):
        nxt = alsd_step(B, [row] * len(B), i, T, beam, recombine_returns_input, final)
        if nxt is None:
            break
        B = nxt
    return (final, True) if final else (B, False)


def check_entries(out, b, pool, from_final, score_norm, n_best, tol=1e-12):
    """rs_rnnt_alsd_nbest's outputs (CPU tensors y, steps, n, score, count, pool, from_final) for utterance b against the
    first n_best of ``pool`` ranked: sequences, alignment steps and token counts identical, scores within ``tol``
    relative, count / pool / from_final exact."""
    y, steps, n, score, count, pool_n, ff = out
    want = ranked(pool, score_norm, n_best)
    assert int(count[b]) == len(want) and int(pool_n[b]) == len(pool) and int(ff[b]) == int(from_final), \
        (b, int(count[b]), len(want), int(pool_n[b]), len(pool), int(ff[b]), from_final)
    for e, h in enumerate(want):
        k = int(n[b, e])
        assert k == len(h.y) - 1 and y[b, e, : k + 1].tolist() == h.y, (b, e, y[b, e, : k + 1].tolist(), h.y)
        assert steps[b, e, :k].tolist() == h.timestamp[1:], (b, e)
        assert abs(float(score[b, e]) - h.score) <= tol * max(1.0, abs(h.score)), (b, e, float(score[b, e]), h.score)


def crafted_cases():
    """(name, T, beam, u_max_ratio, score_norm, token5_bias) of the crafted joints: alsd_cases' recombination and u_max cases,
    and one where no hypothesis finishes (u_max = 0 with token 5 far likelier than blank)."""
    cases = [(f"recombined-T{T}-{'norm' if sn else 'raw'}", T, beam, 2.0, sn, 0.0) for T, beam, sn, _, _ in AC.RECOMBINED_FINAL_CASES]
    c = AC.U_MAX_CASE
    cases.append(("u_max", c["T"], c["beam"], c["ratio"], True, c["token5_bias"]))
    cases += [(f"fallback-beam{beam}", 5, beam, 0.0, True, 5.0) for beam in (1, 4)]
    return cases
