"""Greedy decoding with phrase boosting, for the tests: ``oracle.nemo_restated``'s greedy loop with the boosting tables
(reazonspeech_b200/boosting.py) applied -- ``bonus[n]`` added to the fp32 logits before the argmax (blank column: no bonus),
the automaton state n advanced on every emission -- and a brute-force statement of the bonus by direct string matching."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F


@dataclass
class BoostedResult:
    tokens: List[int] = field(default_factory=list)
    frames: List[int] = field(default_factory=list)
    decisions: List[int] = field(default_factory=list)    # argmax of the boosted scores of every joint evaluation
    margins: List[float] = field(default_factory=list)    # top1 - top2 of the boosted scores
    changed: int = 0                                      # evaluations whose boosted argmax differs from the plain one
    gaps: List[tuple] = field(default_factory=list)       # following: (index, frame, given, oracle argmax, boosted gap)
    complete: bool = True


def boosted_scores(logits: torch.Tensor, bonus: torch.Tensor, state: int) -> torch.Tensor:
    """fp32 logits [V + 1] + the state's bonus row over the V non-blank columns (the blank's score is its logit)."""
    V = logits.shape[0] - 1
    out = logits.clone()
    out[:V] = logits[:V] + bonus[state, :V]
    return out


def greedy_boosted(enc: torch.Tensor, sd, cfg, bonus, next_state, emulate: bool = True,
                   follow: Optional[Sequence[int]] = None) -> BoostedResult:
    """enc [T, d_model] -> the boosted greedy hypothesis.  With ``follow`` (a decision sequence, blanks included, as
    ``parity.decisions_from`` rebuilds it) the walk is teacher-forced along it instead and records in ``gaps`` every decision
    where the oracle's boosted argmax differs, with the boosted score gap (as ``greedy_follow`` does for plain logits)."""
    from oracle import nemo_restated as O
    bonus = torch.as_tensor(np.asarray(bonus), dtype=torch.float32)
    nxt = np.asarray(next_state)
    S = bonus.shape[0]
    res = BoostedResult()
    ep = O.joint_enc_proj(O._q(enc, emulate), sd)
    n_threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        with torch.no_grad():
            emb = sd["decoder.prediction.embed.weight"]
            h = torch.zeros(cfg.pred_hidden); c = torch.zeros(cfg.pred_hidden)
            h_new, c_new = O.lstm_step(torch.zeros(cfg.pred_hidden), h, c, sd)
            pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
            W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
            state, i = 0, 0
            for t in range(ep.shape[0]):
                for _ in range(cfg.max_symbols):
                    logits = F.linear(torch.relu(ep[t] + pp), W, b)
                    scores = boosted_scores(logits, bonus, state)
                    top2 = torch.topk(scores, 2)
                    best = int(top2.indices[0])
                    res.margins.append(float(top2.values[0] - top2.values[1]))
                    res.changed += int(best != int(torch.argmax(logits)))
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
                    nx = int(nxt[state, k])
                    state = nx if 0 <= nx < S else 0
                    h, c = h_new, c_new
                    h_new, c_new = O.lstm_step(emb[k], h, c, sd)
                    pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
        if follow is not None:
            res.complete = i == len(follow)
        return res
    finally:
        torch.set_num_threads(n_threads)


def brute_force_bonus(phrases: Sequence[Sequence[int]], stream: Sequence[int], score: float) -> float:
    """lambda * (sum over phrase occurrences completed in ``stream`` of |p| + f(n_t)) by direct string matching: n_t = the
    longest suffix of the stream that is a prefix of a phrase, f(n_t) = |n_t| - (longest prefix of n_t that is a phrase)."""
    P = {tuple(p) for p in phrases}
    prefixes = {()} | {p[:i] for p in P for i in range(len(p) + 1)}
    s = tuple(stream)
    done = sum(len(p) for end in range(1, len(s) + 1) for p in P if len(p) <= end and s[end - len(p):end] == p)
    n = next(s[len(s) - L:] for L in range(len(s), -1, -1) if s[len(s) - L:] in prefixes)
    D = max((L for L in range(len(n) + 1) if n[:L] in P), default=0)
    return score * (done + len(n) - D)


def follow_stats_emitted(enc: torch.Tensor, sd, cfg, decisions: Sequence[int], alpha: float, emulate: bool = True) -> List[List[float]]:
    """Confidence statistics along a given (boosted) decision sequence, of the UNBOOSTED softmax: per emitted token k,
    [log p_k, sum p log p, sum p^alpha, sum p^alpha log p] from log_softmax (float64) of the oracle's fp32 logits.  Unlike
    ``confidence_oracle.follow_stats`` the first entry is the emitted token's, which under boosting need not be the argmax."""
    from confidence_oracle import stats_of_logprobs
    from oracle import nemo_restated as O
    ep = O.joint_enc_proj(O._q(enc, emulate), sd)
    out, i = [], 0
    with torch.no_grad():
        emb = sd["decoder.prediction.embed.weight"]
        h = torch.zeros(cfg.pred_hidden); c = torch.zeros(cfg.pred_hidden)
        h_new, c_new = O.lstm_step(torch.zeros(cfg.pred_hidden), h, c, sd)
        pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
        W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
        for t in range(ep.shape[0]):
            for _ in range(cfg.max_symbols):
                k = int(decisions[i]); i += 1
                if k == cfg.blank:
                    break
                x = torch.log_softmax(F.linear(torch.relu(ep[t] + pp), W, b).double(), -1)
                out.append([float(x[k])] + stats_of_logprobs(x, alpha)[1:])
                h, c = h_new, c_new
                h_new, c_new = O.lstm_step(emb[k], h, c, sd)
                pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
    assert i == len(decisions)
    return out
