"""CPU oracle of NeMo's ALSD beam search (``BeamRNNTInfer.align_length_sync_decoding``,
nemo/collections/asr/parts/submodules/rnnt_beam_decoding.py) -- the decoding strategy the shipped
reazonspeech-nemo-v2 checkpoint runs by default, as the reference's own post-processing shows
(pkg/nemo-asr/src/decode.py:29 "Decode ALSD beam search info", :38-40 leading blank in y_sequence,
:48 ``step - idx - 1``).

THIS IS TEST INFRASTRUCTURE (see oracle/nemo_restated.py): only tests/, smoke() and bench.py's CPU legs may import it.

PARITY UNPINNED (R): NeMo is absent offline and no port of its transducer beam search exists in the image, so this is a
restatement from the published algorithm (Saon et al. 2020, "Alignment-length synchronous decoding for RNN transducer")
in the form NeMo took over from ESPnet:

    B = [hyp(y=[blank], score=0, timestamp=[-1])]
    for i in range(T + u_max):                                   # i = t + u: one anti-diagonal of the (t, u) lattice per step
        A = []
        for hyp in B with t = i - (len(hyp.y) - 1) <= T - 1:
            logp = log_softmax(joint(enc[t], pred(hyp.y)))
            A += [hyp + blank  (score + logp[blank]; also appended to `final` when t == T - 1)]
            A += [hyp + k      (score + logp[k], timestamp + [i]) for k in top-`beam` non-blank tokens]
        B = top-`beam` of A by score; hypotheses with equal token sequences are recombined (logaddexp)
    return the best of `final` by score / len(y) (score_norm=True, NeMo's default)

Afterwards NeMo's ``pack_hypotheses`` drops the leading -1 of ``timestamp`` and keeps the leading blank of
``y_sequence`` -- the shape pkg/nemo-asr/src/decode.py:40-48 consumes: token idx was emitted at alignment step
``timestamp[idx] = t + idx``.

Recalled details that cannot be verified offline and are therefore switches: ``beam`` (the checkpoint's
``decoding.beam.beam_size``), ``u_max`` (``alsd_max_target_len``, NeMo default 2.0 x T), ``score_norm``, and
``recombine_returns_input``: NeMo's ``recombine_hypotheses`` adds the scores of equal sequences into the first of them
but, as recalled, returns its INPUT list, duplicates included (ESPnet returns the merged list).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from reazonspeech_b200.config import ModelConfig
from .nemo_restated import StateDict, _q, joint_enc_proj, lstm_step


@dataclass
class BeamHyp:
    y: List[int]                       # leading blank, then the tokens
    score: float
    timestamp: List[int]               # leading -1, then the alignment step (t + u) of every token
    state: Tuple[torch.Tensor, torch.Tensor]   # predictor (h, c) BEFORE consuming y[-1]


@dataclass
class AlsdResult:
    y_sequence: List[int]              # with the leading blank (decode.py:38-40)
    timestamp: List[int]               # pack_hypotheses: the leading -1 removed
    score: float
    nbest: List[BeamHyp] = field(default_factory=list)
    from_final: bool = True            # False: no hypothesis finished, the winner is the best of the last beam

    @property
    def tokens(self) -> List[int]:
        return self.y_sequence[1:]

    @property
    def frames(self) -> List[int]:
        """Encoder frame of every token: alignment step minus the tokens emitted before it."""
        return [s - i for i, s in enumerate(self.timestamp)]


def alsd_beam(enc: torch.Tensor, sd: StateDict, cfg: ModelConfig, beam: int = 4, u_max_ratio: float = 2.0,
              score_norm: bool = True, recombine_returns_input: bool = True, emulate: bool = False) -> AlsdResult:
    """enc: float32[T, d_model] -> best ALSD hypothesis (see the module docstring)."""
    T = enc.shape[0]
    ep = joint_enc_proj(_q(enc, emulate), sd)
    emb = sd["decoder.prediction.embed.weight"]
    Wp, bp = sd["joint.pred.weight"], sd["joint.pred.bias"]
    W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
    hp = cfg.pred_hidden
    blank = cfg.blank
    beam = min(beam, cfg.vocab_size)
    u_max = int(u_max_ratio * T)
    n_threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        cache: Dict[tuple, Tuple[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]] = {}

        def predictor(h: BeamHyp):
            """joint.pred of the predictor output after consuming y[-1], and the state after it (cached per sequence:
            the predictor is a deterministic function of the token sequence -- batch_score_hypothesis's cache)."""
            key = tuple(h.y)
            if key not in cache:
                x = torch.zeros(hp) if h.y[-1] == blank else emb[h.y[-1]]      # SOS / blank_as_pad: the zero vector
                h2, c2 = lstm_step(x, h.state[0], h.state[1], sd)
                cache[key] = (F.linear(h2, Wp, bp), (h2, c2))
            return cache[key]

        B = [BeamHyp([blank], 0.0, [-1], (torch.zeros(hp), torch.zeros(hp)))]
        final: List[BeamHyp] = []
        for i in range(T + u_max):
            rows = []
            for h in B:
                t = i - (len(h.y) - 1)
                if t > T - 1:
                    rows.append(None)
                    continue
                pp, state_after = predictor(h)
                logp = torch.log_softmax(F.linear(torch.relu(ep[t] + pp), W, b), dim=-1)
                nb = torch.cat((logp[:blank], logp[blank + 1:]))              # beam_logp[:, ids]: every class but the blank
                top = nb.topk(beam)
                idx = [k + (1 if k >= blank else 0) for k in top.indices.tolist()]   # index back into the full class list
                rows.append((float(logp[blank]), top.values.tolist(), idx, state_after))
            B2 = alsd_step(B, rows, i, T, beam, recombine_returns_input, final)
            if B2 is None:
                break
            B = B2
        pool = final if final else B
        key = (lambda x: x.score / len(x.y)) if score_norm else (lambda x: x.score)
        nbest = sorted(pool, key=key, reverse=True)
        best = nbest[0]
        return AlsdResult(best.y, best.timestamp[1:] if best.timestamp and best.timestamp[0] == -1 else best.timestamp,
                          best.score, nbest, from_final=bool(final))
    finally:
        torch.set_num_threads(n_threads)


def alsd_step(B: List[BeamHyp], rows, i: int, T: int, beam: int, recombine_returns_input: bool, final: List[BeamHyp],
              final_aliases_beam: bool = True) -> Optional[List[BeamHyp]]:
    """One step (the anti-diagonal i = t + u) of align_length_sync_decoding.  rows[k] = (log p(blank), the `beam` best non-blank
    log-probabilities, their class indices, the predictor state after y[-1]) of B[k] when it is live at step i (t = i - (len(y)
    - 1) <= T - 1), anything otherwise.  Appends the stays at the last frame to ``final`` and returns the new beam, or None when
    no hypothesis is live (the search ends).  As in NeMo, an entry of ``final`` is the very object that enters the beam, so
    recombination in this step adds into it; final_aliases_beam=False records a copy instead, the score before recombination."""
    A: List[BeamHyp] = []
    for h, row in zip(B, rows):
        t = i - (len(h.y) - 1)
        if t > T - 1:
            continue
        lp_blank, values, indices, state_after = row
        stay = BeamHyp(h.y[:], h.score + lp_blank, h.timestamp[:], h.state)
        A.append(stay)
        if t == T - 1:
            final.append(stay if final_aliases_beam else BeamHyp(stay.y, stay.score, stay.timestamp, stay.state))
        for lp, k in zip(values, indices):
            A.append(BeamHyp(h.y + [k], h.score + lp, h.timestamp + [i], state_after))
    if not A:
        return None
    B = sorted(A, key=lambda x: x.score, reverse=True)[:beam]              # stable, like Python's sorted in NeMo
    return _recombine(B, recombine_returns_input)


def _recombine(hyps: List[BeamHyp], returns_input: bool) -> List[BeamHyp]:
    merged: List[BeamHyp] = []
    for h in hyps:
        seen = [m.y for m in merged]
        if h.y in seen:
            m = merged[seen.index(h.y)]
            hi, lo = max(m.score, h.score), min(m.score, h.score)
            m.score = hi + math.log1p(math.exp(lo - hi))                       # np.logaddexp
        else:
            merged.append(h)
    return hyps if returns_input else merged
