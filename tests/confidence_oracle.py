"""Second statement of greedy-decode confidence, for the tests: the statistics straight from ``torch.log_softmax`` of the
oracle's fp32 logits (float64), and NeMo's confidence measure bank (R) evaluated directly on the log-probability vector --
the formulas as NeMo writes them, not the statistics-based forms of ``reazonspeech_b200/confidence.py``."""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F


def stats_of_logprobs(x: torch.Tensor, alpha: float) -> List[float]:
    """x: float64 log-probabilities -> [lp (of the argmax), sum p log p, sum p^alpha, sum p^alpha log p]."""
    p = x.exp()
    pa = (x * alpha).exp()
    return [float(x.max()), float((p * x).sum()), float(pa.sum()), float((pa * x).sum())]


def _bank():
    """NeMo's get_confidence_measure_bank (R): x = log-probabilities [V], v = V, t = alpha."""
    neg_entropy_gibbs = lambda x: (x.exp() * x).sum(-1)
    neg_entropy_alpha = lambda x, t: (x * t).exp().sum(-1)
    neg_entropy_alpha_gibbs = lambda x, t: ((x * t).exp() * x).sum(-1)
    gibbs_lin_baseline = lambda x, v: 1 + neg_entropy_gibbs(x) / math.log(v)
    gibbs_exp_baseline = lambda x, v: (neg_entropy_gibbs(x).exp() * v - 1) / (v - 1)

    def tsallis_exp(x, v, t):
        exp_neg_max_ent = math.exp((1 - math.pow(v, 1 - t)) / (1 - t))
        return (((1 - neg_entropy_alpha(x, t)) / (1 - t)).exp() - exp_neg_max_ent) / (1 - exp_neg_max_ent)

    def gibbs_exp(x, v, t):
        exp_neg_max_ent = math.pow(v, -t * math.pow(v, 1 - t))
        return ((neg_entropy_alpha_gibbs(x, t) * t).exp() - exp_neg_max_ent) / (1 - exp_neg_max_ent)

    return {
        "max_prob": lambda x, v, t: ((x.max(dim=-1)[0].exp() * v - 1) / (v - 1) if t == 1.0
                                     else ((x.max(dim=-1)[0] * t).exp() * math.pow(v, t) - 1) / (math.pow(v, t) - 1)),
        "entropy_gibbs_lin": lambda x, v, t: (gibbs_lin_baseline(x, v) if t == 1.0
                                              else 1 + neg_entropy_alpha_gibbs(x, t) / math.log(v) / math.pow(v, 1 - t)),
        "entropy_gibbs_exp": lambda x, v, t: gibbs_exp_baseline(x, v) if t == 1.0 else gibbs_exp(x, v, t),
        "entropy_tsallis_lin": lambda x, v, t: (gibbs_lin_baseline(x, v) if t == 1.0
                                                else 1 + (1 - neg_entropy_alpha(x, t)) / (math.pow(v, 1 - t) - 1)),
        "entropy_tsallis_exp": lambda x, v, t: gibbs_exp_baseline(x, v) if t == 1.0 else tsallis_exp(x, v, t),
        "entropy_renyi_lin": lambda x, v, t: (gibbs_lin_baseline(x, v) if t == 1.0
                                              else 1 + neg_entropy_alpha(x, t).log2() / (t - 1) / math.log(v, 2)),
        "entropy_renyi_exp": lambda x, v, t: (gibbs_exp_baseline(x, v) if t == 1.0
                                              else (neg_entropy_alpha(x, t).pow(1 / (t - 1)) * v - 1) / (v - 1)),
    }


MEASURE_BANK = _bank()


def direct_measure(x: torch.Tensor, name: str, alpha: float) -> float:
    """NeMo's measure ``name`` ("max_prob" or "entropy_<type>_<norm>") of one log-probability vector (float64)."""
    return float(MEASURE_BANK[name](x, x.shape[-1], alpha))


def follow_stats(enc: torch.Tensor, sd, cfg, decisions: Sequence[int], alphas: Sequence[float], emulate: bool = True) -> Dict[float, List[List[float]]]:
    """The oracle's predictor + joint walked along a GIVEN decision sequence (blanks included, as ``parity.decisions_from``
    rebuilds it): per alpha, the statistics of every emitted token from log_softmax (float64) of the fp32 logits."""
    from oracle import nemo_restated as O
    ep = O.joint_enc_proj(O._q(enc, emulate), sd)
    out = {a: [] for a in alphas}
    with torch.no_grad():
        emb = sd["decoder.prediction.embed.weight"]
        h = torch.zeros(cfg.pred_hidden); c = torch.zeros(cfg.pred_hidden)
        h_new, c_new = O.lstm_step(torch.zeros(cfg.pred_hidden), h, c, sd)
        pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
        W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
        i = 0
        for t in range(ep.shape[0]):
            for _ in range(cfg.max_symbols):
                k = int(decisions[i]); i += 1
                if k == cfg.blank:
                    break
                x = torch.log_softmax(F.linear(torch.relu(ep[t] + pp), W, b).double(), -1)
                for a in alphas:
                    out[a].append(stats_of_logprobs(x, a))
                h, c = h_new, c_new
                h_new, c_new = O.lstm_step(emb[k], h, c, sd)
                pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
    assert i == len(decisions)
    return out
