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
order) and one CTA per utterance for the recursions and the backtrace.  This module holds the host-side helpers.

Segment alignment (``rs_rnnt_align_segment``; captions.py uses it to locate a caption inside its audio window).  The
lattice is the one above, of a window with T frames and labels y_1..y_U, U >= 1.  The predictor starts from the SOS state
at u = 0, as in forced alignment: it does not see the text that precedes the caption.  The tokens may start at any frame
and end at any frame, and the frames outside are not charged:

    delta[t][0] = 0                                   for every t      (the caption may start at any frame)
    delta[t][u] = max(delta[t-1][u] + lp_blank[t-1][u],  delta[t][u-1] + lp_emit[t][u-1])      u >= 1 (no blank term at t = 0)
    score       = max_t  delta[t][U] + lp_blank[t][U]                  (the end is free too)

The end frame e is the smallest maximising t; on an exact tie between predecessors the blank one wins.  The backtrace from
(e, U) gives each token's emission frame; s is the frame of token 1, and the segment [s, e] holds U emissions and one blank
per frame, the final blank at (e, U) included.  frame_lp[t] (t in [s, e]) is the sum of the path's steps charged to frame t
(its emissions at t plus the blank that leaves t), so sum(frame_lp) = score.  loglik is the forward recursion above restricted
to rows [s, e] (alpha[s][0] = 0, ending with the blank at (e, U)): log P(caption | the audio of its segment).  Hence
loglik >= score >= the full-window Viterbi score of the same lattice.  U = 0, a label outside [0, V) or enc_len outside
[1, T_max] gives s = e = -1, frames -1 and NaN scores.  On the GPU: rnnt_segment_dp_kernel, one CTA per window, on the
lattice the forced alignment computes.

Banded alignment (``rs_rnnt_align_banded``; longform.py builds the band for transcripts of long recordings).  The lattice,
recursions, tie rule, outputs and their meaning are forced alignment's, but only the cells lo[u] <= t < hi[u] exist; every
other cell is -inf.  The band is given per label row u in [0, U] and must satisfy 0 <= lo[u] < hi[u] <= T, lo and hi
non-decreasing in u, lo[0] = 0, hi[U] = T, and lo[u + 1] < hi[u]: consecutive rows overlap, and every path's vertical step
from row u to u + 1 (token u + 1) happens at a frame in [lo[u + 1], hi[u]).  Then every diagonal d = t + u meets the band in
one contiguous run of rows, every cell but (0, 0) has a predecessor inside the band, and so:

- a full band (lo = 0, hi = T) gives exactly forced alignment's results;
- a band that contains the full lattice's Viterbi path gives the same Viterbi path and score;
- for any valid band, viterbi_band <= viterbi_full and loglik_band <= loglik_full.

edge counts the tokens whose emission frame t lies on an interior edge of the band's constraint on that step: token u (the
step from row u - 1 to row u) with t = lo[u] > 0, or with t = hi[u - 1] - 1 < T - 1.  It signals that the band may have cut
the path.  It is a heuristic: a path clear of the edges does not prove that the banded path is the global Viterbi path.  On
the GPU: rnnt_lattice_kernel's banded instance computes the tiles of the full lattice's grid that meet the band (so every
cell is bit-identical to the full lattice's) into banded storage, and rnnt_band_dp_kernel runs the recursions with shared
memory bounded by the band's largest diagonal extent instead of U."""
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
