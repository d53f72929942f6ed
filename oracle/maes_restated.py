"""CPU oracle of NeMo's MAES beam search (``BeamRNNTInfer.modified_adaptive_expansion_search`` with ``prefix_search``,
``select_k_expansions``, ``recombine_hypotheses`` and ``sort_nbest``, nemo/collections/asr/parts/submodules/rnnt_beam_decoding.py)
-- modified adaptive expansion search (Kim et al. 2020, "Accelerating RNN transducer inference via adaptive expansion search"),
the transducer beam search into which NeMo fuses an n-gram LM (``ngram_lm_model`` / ``ngram_lm_alpha`` are accepted with
``search_type="maes"`` only (R)).

THIS IS TEST INFRASTRUCTURE (see oracle/nemo_restated.py): only tests/, smoke() and bench.py's CPU legs may import it.

PARITY UNPINNED (R): NeMo is absent offline, so this restates the algorithm as recalled; every recalled detail is marked (R).

    K = min(beam, V); C = K + expansion_beta                                          (R: max_candidates = beam + beta)
    kept = [hyp(y=[blank], score=0, dec_out=[pred(SOS)], lm_state=<s>)]                (R)
    for t in range(enc_len):
        hyps = prefix_search(sorted(kept, key=len(y), reverse=True), t)               (R: stable, longest first)
        duplication_check = [h.y for h in hyps]                                       (R: built once per frame, never updated)
        list_b = []
        for n in range(num_steps):
            logp = log_softmax(joint(enc[t], h.dec_out[-1])) for h in hyps; the C best classes of all V + 1, blank included
                   (ties: lower class index)
            select_k_expansions: per hypothesis the candidates with score + logp >= best - gamma, ordered by score
                   ASCENDING (R; stable); none passing: the best alone
            blank -> list_b (y unchanged; list_b keeps filling across rounds)
            token k with y + [k] not in duplication_check -> list_exp (frame t; with an LM: + lm term, LM state advanced)
            list_exp empty: kept = sorted(recombine(list_b), desc)[:K]; the frame ends   (R: recombine before the sort)
            otherwise the predictor runs on list_exp (dec_out appended); not the last round: hyps = list_exp;
            last round: each entry + logp(enc[t], new dec_out)[blank], kept = sorted(recombine(list_b + list_exp), desc)[:K]
    return sort_nbest(kept): by score / len(y) with score_norm, else by score; stable

prefix_search(hyps, t) (R): for j < i in that order, where y_i is a strict prefix of y_j and len(y_j) - len(y_i) <= prefix_alpha:
    curr = score_i + logp(enc[t], dec_out_i[-1])[y_j[len_i]] + sum_{k in [len_i, len_j - 1)} logp(enc[t], dec_out_j[k])[y_j[k + 1]]
    score_j = logaddexp(score_j, curr)
Every score_i read is the one before this frame's updates (i comes after j, so its own turn is later).  No LM term (R).

LM terms come from a callable ``lm(state, token) -> (term, next_state)`` with the start state ``lm_start``: the tests pass
tests/ngram_oracle.py's ArpaOracle, term = alpha * ln10 * log10 P(k | h) as reazonspeech_b200/ngram_lm.py defines it (NeMo adds
``ngram_lm_alpha * lm_score`` with lm_score = log10 P / log10(e) (R), the same value).

Switches: ``recombine_returns_input`` as in oracle/alsd_restated.py.  An utterance with enc_len = 0 returns [blank], score 0.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from reazonspeech_b200.config import ModelConfig
from .alsd_restated import BeamHyp, _recombine
from .nemo_restated import StateDict, _q, joint_enc_proj, lstm_step


@dataclass
class MaesHyp(BeamHyp):
    """BeamHyp with NeMo's dec_out list (dec_out[k]: joint.pred after y[:k + 1]) and LM state.  Here ``timestamp`` holds a
    leading -1 and then the encoder frame of every token, and ``state`` is the predictor state AFTER consuming y[-1]."""
    dec_out: List[torch.Tensor] = field(default_factory=list)
    lm_state: Any = None


@dataclass
class MaesResult:
    y_sequence: List[int]
    frames: List[int]
    score: float
    nbest: List[MaesHyp]

    @property
    def tokens(self) -> List[int]:
        return self.y_sequence[1:]


def is_prefix(x: List[int], pref: List[int]) -> bool:
    """NeMo's is_prefix: pref is a strict prefix of x."""
    return 0 < len(pref) < len(x) and x[:len(pref)] == pref


def prefix_search(hyps: List[MaesHyp], logp: Callable[[torch.Tensor], torch.Tensor], prefix_alpha: int) -> List[MaesHyp]:
    """NeMo's prefix_search on hyps (already sorted longest first); logp(dec_out) = log-softmax of the joint at this frame."""
    old = [h.score for h in hyps]
    for j, hj in enumerate(hyps[:-1]):
        for i in range(j + 1, len(hyps)):
            hi = hyps[i]
            lj, li = len(hj.y), len(hi.y)
            if is_prefix(hj.y, hi.y) and lj - li <= prefix_alpha:
                curr = old[i] + float(logp(hi.dec_out[-1])[hj.y[li]])
                for k in range(li, lj - 1):
                    curr += float(logp(hj.dec_out[k])[hj.y[k + 1]])
                hi_, lo = max(hj.score, curr), min(hj.score, curr)
                hj.score = hi_ + math.log1p(math.exp(lo - hi_))                # np.logaddexp
    return hyps


def topk_stable(logp: torch.Tensor, C: int) -> Tuple[List[int], List[float]]:
    """The C best classes, ties -> lower class index."""
    order = torch.sort(logp, descending=True, stable=True).indices[:C]
    return order.tolist(), [float(logp[k]) for k in order.tolist()]


def select_k_expansions(hyps: List[MaesHyp], idx: List[List[int]], lps: List[List[float]], gamma: float) -> List[List[Tuple[int, float]]]:
    """NeMo's select_k_expansions: per hypothesis [(class, score + logp)] within gamma of its best, ascending by score (stable)."""
    out = []
    for h, ks, vs in zip(hyps, idx, lps):
        cand = [(int(k), h.score + float(v)) for k, v in zip(ks, vs)]
        best = max(cand, key=lambda x: x[1])
        exp = sorted([c for c in cand if best[1] - gamma <= c[1]], key=lambda x: x[1])
        out.append(exp if exp else [best])
    return out


def sort_nbest(hyps: List[MaesHyp], score_norm: bool) -> List[MaesHyp]:
    key = (lambda x: x.score / len(x.y)) if score_norm else (lambda x: x.score)
    return sorted(hyps, key=key, reverse=True)


def maes_beam(enc: torch.Tensor, sd: StateDict, cfg: ModelConfig, beam: int = 4, num_steps: int = 2, prefix_alpha: int = 1,
              expansion_beta: int = 2, expansion_gamma: float = 2.3, score_norm: bool = True, recombine_returns_input: bool = True,
              lm: Optional[Callable[[Any, int], Tuple[float, Any]]] = None, lm_start: Any = None, emulate: bool = False) -> MaesResult:
    """enc: float32[T, d_model] -> the sort_nbest list of the MAES search (see the module docstring)."""
    T = enc.shape[0]
    ep = joint_enc_proj(_q(enc, emulate), sd)
    emb = sd["decoder.prediction.embed.weight"]
    Wp, bp = sd["joint.pred.weight"], sd["joint.pred.bias"]
    W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
    hp, blank = cfg.pred_hidden, cfg.blank
    K = min(beam, cfg.vocab_size)
    C = K + expansion_beta
    n_threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        cache: Dict[tuple, Tuple[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]] = {}

        def predictor(y: List[int], state):
            """joint.pred after consuming y[-1] from `state`, and the state after it (cached per sequence, as
            batch_score_hypothesis caches it)."""
            key = tuple(y)
            if key not in cache:
                x = torch.zeros(hp) if y[-1] == blank else emb[y[-1]]          # SOS: the zero vector
                h2, c2 = lstm_step(x, state[0], state[1], sd)
                cache[key] = (F.linear(h2, Wp, bp), (h2, c2))
            return cache[key]

        pp0, st0 = predictor([blank], (torch.zeros(hp), torch.zeros(hp)))
        kept = [MaesHyp([blank], 0.0, [-1], st0, [pp0], lm_start)]
        for t in range(T):
            def logp(pp, t=t):
                return torch.log_softmax(F.linear(torch.relu(ep[t] + pp), W, b), dim=-1)

            hyps = prefix_search(sorted(kept, key=lambda x: len(x.y), reverse=True), logp, prefix_alpha)
            dup = [h.y for h in hyps]
            list_b: List[MaesHyp] = []
            for n in range(num_steps):
                rows = [topk_stable(logp(h.dec_out[-1]), C) for h in hyps]
                exps = select_k_expansions(hyps, [r[0] for r in rows], [r[1] for r in rows], expansion_gamma)
                list_exp: List[MaesHyp] = []
                for h, ex in zip(hyps, exps):
                    for k, s in ex:
                        if k == blank:
                            list_b.append(MaesHyp(h.y[:], s, h.timestamp[:], h.state, h.dec_out[:], h.lm_state))
                        elif h.y + [k] not in dup:
                            new = MaesHyp(h.y + [k], s, h.timestamp + [t], h.state, h.dec_out[:], h.lm_state)
                            if lm is not None:
                                term, new.lm_state = lm(h.lm_state, k)
                                new.score += float(term)
                            list_exp.append(new)
                if not list_exp:
                    kept = sorted(_recombine(list_b, recombine_returns_input), key=lambda x: x.score, reverse=True)[:K]
                    break
                for h in list_exp:
                    pp, h.state = predictor(h.y, h.state)
                    h.dec_out.append(pp)
                if n < num_steps - 1:
                    hyps = list_exp
                else:
                    for h in list_exp:
                        h.score += float(logp(h.dec_out[-1])[blank])
                    kept = sorted(_recombine(list_b + list_exp, recombine_returns_input), key=lambda x: x.score, reverse=True)[:K]
        nbest = sort_nbest(kept, score_norm)
        if not nbest:
            return MaesResult([blank], [], float("-inf"), [])
        best = nbest[0]
        return MaesResult(best.y, best.timestamp[1:], best.score, nbest)
    finally:
        torch.set_num_threads(n_threads)
