"""Forced alignment of a known transcript: where each token lies in the audio, and how well the audio supports the text.

The lattice is the standard RNN-T one (Graves 2012), the same as NeMo's RNN-T loss and ``torchaudio.functional.rnnt_loss``.
For an utterance with encoder frames t < T, labels y_1..y_U (each in [0, V), never blank) and predictor outputs g_0..g_U
(g_0 the blank / start state, exactly as the greedy decode starts; g_u the output after feeding y_1..y_u):

    lp_blank[t][u] = log softmax(joint(f_t, g_u))[blank]
    lp_emit[t][u]  = log softmax(joint(f_t, g_u))[y_{u+1}]          (u < U)
    joint(f, g)    = W_out relu(enc_proj(f) + pred_proj(g)) + b_out

    alpha[0][0] = 0
    alpha[t][u] = (+)( alpha[t-1][u] + lp_blank[t-1][u],  alpha[t][u-1] + lp_emit[t][u-1] )
    score       = alpha[T-1][U] + lp_blank[T-1][U]

with (+) = logaddexp for the log-likelihood log P(y | x) (= -RNN-T loss) and max for the Viterbi score.  The Viterbi path
gives each token u its emission frame t_u (the t of its vertical step) and its path log-probability lp_emit[t_u][u-1]; on an
exact tie the blank predecessor wins.  There is no max_symbols cap (a frame may emit any number of tokens), U > T is allowed,
and U = 0 is the all-blank path.

On the GPU (csrc/align.cu): a teacher-forced predictor, the lattice on wgmma (the joint's activation split into two IEEE-half
terms and bf16-exact weights, as the greedy decode's joint: a cell's logits are the decode's for that (t, u) up to summation
order) and one CTA per utterance for the recursions and the backtrace.  This module holds the host-side helpers."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


def validate_labels(token_lists: Sequence[Sequence[int]], vocab_size: int, n_audio: int) -> List[List[int]]:
    """Token-id lists as plain ints; ValueError when their count differs from the audio count or an id is outside
    [0, vocab_size) (the blank, vocab_size, is not a label)."""
    if len(token_lists) != n_audio:
        raise ValueError(f"{len(token_lists)} transcripts for {n_audio} audio inputs")
    out = []
    for n, ids in enumerate(token_lists):
        ids = [int(k) for k in ids]
        bad = [k for k in ids if not 0 <= k < vocab_size]
        if bad:
            raise ValueError(f"transcript {n}: token id {bad[0]} outside [0, {vocab_size})")
        out.append(ids)
    return out


def pack_labels(token_lists: Sequence[Sequence[int]]) -> Tuple[np.ndarray, np.ndarray]:
    """-> labels int32 [B, U_max] (zero padded, U_max >= 1), label_len int32 [B]."""
    U = max([len(ids) for ids in token_lists] + [1])
    labels = np.zeros((len(token_lists), U), dtype=np.int32)
    for r, ids in enumerate(token_lists):
        labels[r, : len(ids)] = ids
    return labels, np.array([len(ids) for ids in token_lists], dtype=np.int32)


def alignment_hypothesis(ids: Sequence[int], frames: Sequence[int], token_lp: Sequence[float], viterbi: float, loglik: float,
                         blank: int):
    """One utterance's alignment -> the ``Hypothesis`` a transcription of the same tokens at the same frames would give
    (so ``decode_hypothesis`` times its subwords and segments the same way), with score = the Viterbi score,
    log_likelihood = log P(y | x) and token_logprob = each token's log-probability on the Viterbi path."""
    from .nemo.asr.transcribe import Hypothesis
    hyp = Hypothesis.from_greedy(ids, frames, blank)
    hyp.score = float(viterbi)
    hyp.log_likelihood = float(loglik)
    hyp.token_logprob = [float(x) for x in token_lp]
    return hyp
