"""Keyword spotting: every occurrence of a list of keywords in long recordings, found on the RNN-T lattice.

Searching a greedy transcript for a keyword misses the words that matter most: rare names are the words the model
misrecognises.  The lattice scores the keyword's own tokens at every frame, so a keyword the greedy path spelled wrongly can
still be found.

Inputs.  A recording is prepared as ``transcribe`` prepares audio (norm_audio, then 0.5 s of silence on both sides); it has
encoder frames t < T.  A keyword is text or a sequence of token ids.  Text is tokenised as phrase boosting tokenises a phrase
(``tokenizer.text_to_ids``: the lone leading word-boundary piece dropped) and validated like ``boosting.phrase_ids``; a keyword
has labels y_1..y_U with 1 <= U <= 32 (longer text is a caption: ``align_captions``).

Lattice.  The lattice of a (recording, keyword) pair is the one alignment.py defines; the predictor starts from SOS.

Recursion.  The segment recursion of alignment.py, unchanged, with the score of every end frame kept:

    delta[t][0] = 0                                                     every t
    delta[t][u] = max(delta[t-1][u] + lp_blank[t-1][u], delta[t][u-1] + lp_emit[t][u-1])      u >= 1
    E(e) = delta[e][U] + lp_blank[e][U]            the best segment path that ends at frame e
    S(e) = the frame of token 1 on that path       (exact predecessor ties: the blank one wins, as in the segment DP)
    m(e) = E(e) / (e - S(e) + 1)                   in fp32, exactly so: the mean per-frame log-probability

So max_e E(e) is the segment alignment's score and its smallest maximising e is the segment alignment's end frame.

Hits of one (recording, keyword) pair:
  1. the candidates are every e with m(e) >= threshold;
  2. repeatedly take the candidate with the largest m (on an exact tie, the smaller e),
  3. record it as a hit [S(e), e],
  4. and drop every remaining candidate whose [S(e'), e'] intersects the hit's span;
  5. stop when no candidate is left or after ``max_hits`` hits.
Each hit carries its tokens' frames and lp_emit from the backtrace of the path to (e, U), score = E(e) and confidence = m(e).
For segments of at most 15 frames m(e) is ``captions.confidence`` of the hit's per-frame log-probabilities, up to rounding.

Seconds.  Frame f lies at max(0.08 f - 0.5, 0) s, as in ``decode_hypothesis`` and ``captions.frame_seconds``; a hit ends at
the end of frame e, clamped to the recording.

Defaults.  threshold = -1.0 and max_hits = 64 per keyword per recording (at most 256).  The threshold is NOT calibrated: only
synthetic weights were reachable when it was chosen, and their joint is nearly flat.  Calibrate it on labelled audio of the
released checkpoint before trusting a hit list.

On the GPU (rs_rnnt_spot): joint.enc once per recording, the teacher-forced predictor once per keyword, the lattice of every
pair on wgmma (rnnt_lattice_kernel<true>), one warp per pair for the recursion (rnnt_spot_dp_kernel) and one CTA per pair for
the hit policy and the backtraces (rnnt_spot_pick_kernel).  This module holds the host-side helpers.

Streaming.  Keyword hits on live streams (``StreamingTranscriber(keywords=StreamKeywordsConfig(...))``), decided chunk by
chunk on the encoder output the streaming decode produces.  Nothing above changes: lattice, recursion, E(e), S(e), m(e), the
threshold and the pick rule are the offline ones.  A stream's frames are the streaming frame grid (streaming.py), and the
lattice of a chunk's frames is the lattice of the same frames offline, cell for cell.

  1. Carried recursion.  delta[t][u] depends on frames <= t only.  So a (stream, keyword) pair carries one column from step
     to step: delta[t][u], the start frame start[t][u] and lp_blank[t][u] for u = 1..U at its last decoded frame t, and each
     step extends the recursion over its frames.  E(e) and S(e) of every frame are bit-identical to rs_rnnt_spot's on the
     same lattice cells: the same fp32 operations in the same order, the same tie rule.
  2. Frontier bound.  sigma(t) = min over u in 1..U of start[t][u].  Every candidate that ends after t has S >= sigma(t): the
     best path to (e', U), e' > t, either emits token 1 after t (S > t >= sigma(t)), or leaves frame t from some cell (t, u)
     with u >= 1, and the prefix of that path up to (t, u) is that cell's best path (the recursion's backtrace), whose first
     token is at start[t][u] >= sigma(t).  sigma never decreases: start[t + 1][u] is start[t][u] (blank) or start[t + 1][u - 1]
     (emission), by induction over u >= sigma(t) with start[t + 1][0] = t + 1.
  3. Exact decisions (the natural cut).  After each step, L = sigma(t), then L <- min(L, min{S(e) : pending candidate with
     e >= L}) until it stops changing.  No known or future candidate at or after L can intersect a candidate that ends before
     L, so the candidates with e < L form complete overlap components, and the offline greedy rule (the largest m first, the
     smaller e on a tie, drop whatever intersects a hit) applied to them gives exactly the offline decisions, provided the
     offline list did not reach ``max_hits`` (the stream has no such limit).  When a stream is closed and its last frame
     decoded, L = infinity.
  4. Bounded delay (the forced cut).  ``max_delay_seconds`` = D frames (default 10 s, NOT calibrated) bounds the time from a
     candidate's end frame to its decision: if a pending candidate has t - e >= D, the cut becomes max(L, t + 1 - D).  The
     candidates before the cut are decided by the same greedy rule among themselves, and every later candidate whose span
     reaches back to a reported hit is dropped (the barrier: the largest reported end frame).  Hits decided beyond the natural
     cut carry ``forced = True``, and the stream counts its forced cuts.  A stream without a forced cut reproduces the offline
     hits exactly; after one, only this is promised: hits never overlap, and each is a true segment path with its score.
     Forcing will be common on real audio, though none is reachable here to measure it: blanks in silence are nearly free, so
     stretching a span over silence raises m(e).  The offline rule therefore likes long spans, and sigma lags while a channel
     is silent.
  5. Hits.  The fields of ``find_keywords`` (span, score = E(e), confidence = m(e), the tokens' frames and lp_emit) plus
     ``forced``; seconds from ``hit_seconds`` over the audio pushed so far (the trailing pad exists only after close).

On the GPU (rs_stream_step_spot, rs_rnnt_spot_resume; spot_stream.cu): the chunk's joint.enc rows gathered into a compact
block, the pairs' lattice on rnnt_lattice_kernel<true>, the recursion resumed from a per-(stream, keyword) record with a
forward traceback instead of predecessor bytes (a hit's span can be much longer than any window kept on the device), the
candidates appended to a ring of D + C entries per pair, and one warp per pair for the cuts and the pick.  The keywords'
predictor rows are computed once, when the set is installed."""
from __future__ import annotations

import math
import numbers
from dataclasses import dataclass, field
from typing import Any, List, Sequence, Union

from .captions import segment_seconds
from .streaming import _frames

THRESHOLD = -1.0
MAX_HITS = 64
MAX_HITS_LIMIT = 256         # include/rs_engine.h rs_rnnt_spot
MAX_KEYWORD_TOKENS = 32      # one warp lane per lattice row in the recursion
# lattice scratch of one rs_rnnt_spot call (9 bytes per cell, 8 per frame of E and S): the keywords are cut into groups below it
SCRATCH_CAP_BYTES = 1 << 30

Keyword = Union[str, Sequence[int]]


@dataclass
class KeywordHit:
    """One occurrence of a keyword: its span in seconds of the recording, score = E(e) (the best segment path's
    log-probability), confidence = m(e) (its mean per frame), and the keyword's tokens as subwords timed in seconds."""
    keyword: Any
    start_seconds: float
    end_seconds: float
    score: float = math.nan
    confidence: float = math.nan
    subwords: List[Any] = field(default_factory=list)
    forced: bool = False      # streaming: decided by the bounded delay, beyond the natural cut (the offline list may differ)


@dataclass(frozen=True)
class StreamKeywordsConfig:
    """The keywords of a ``StreamingTranscriber``: text or token-id sequences (validated by ``keyword_ids`` when the
    transcriber is built), the per-frame threshold, and the alert delay, a non-negative multiple of 0.08 s (default 10 s,
    NOT calibrated)."""
    keywords: Sequence[Keyword]
    threshold: float = THRESHOLD
    max_delay_seconds: float = 10.0

    def __post_init__(self):
        check_search(self.threshold, 1)
        self.delay_frames()
        if len(self.keywords) == 0:
            raise ValueError("StreamKeywordsConfig needs at least one keyword")

    def delay_frames(self) -> int:
        """D in encoder frames."""
        return _frames(self.max_delay_seconds, "max_delay_seconds")


def stream_record_bytes(U_max: int, delay_frames: int, chunk_frames: int) -> int:
    """Bytes of one (stream, keyword) record (rs_spot_state_bytes): header, carried column, token lists, and a ring of D + C
    candidates of 12 + 8 U_max bytes, rounded up to 16."""
    n = 32 + 12 * U_max + 8 * U_max * U_max + (delay_frames + chunk_frames) * (12 + 8 * U_max)
    return (n + 15) // 16 * 16


def keyword_ids(keywords: Sequence[Keyword], vocab_size: int, tokenizer=None) -> List[List[int]]:
    """The keywords as token-id lists: text through ``tokenizer.text_to_ids``, id sequences as they are.  ValueError for an
    empty keyword, an id outside [0, vocab_size) or more than 32 tokens."""
    out = []
    for kw in keywords:
        if isinstance(kw, str):
            if tokenizer is None:
                raise ValueError(f"keyword {kw!r} is text but no tokenizer was given")
            ids = list(tokenizer.text_to_ids(kw))
        else:
            ids = [int(i) for i in kw]
        if len(ids) == 0:
            raise ValueError(f"keyword {kw!r} tokenises to nothing")
        bad = [i for i in ids if not 0 <= i < vocab_size]
        if bad:
            raise ValueError(f"keyword {kw!r}: token ids {bad} outside [0, {vocab_size}) (blank is never part of a keyword)")
        if len(ids) > MAX_KEYWORD_TOKENS:
            raise ValueError(f"keyword {kw!r} has {len(ids)} tokens, at most {MAX_KEYWORD_TOKENS} are searched: use align_captions "
                             "for longer text")
        out.append(ids)
    return out


def check_search(threshold: float, max_hits: int) -> None:
    """ValueError unless threshold is a number other than NaN and +inf, and max_hits an integer in [1, 256]."""
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real) or math.isnan(threshold) or threshold == math.inf:
        raise ValueError(f"threshold must be a finite number or -inf, got {threshold!r}")
    if isinstance(max_hits, bool) or not isinstance(max_hits, numbers.Integral) or not 1 <= max_hits <= MAX_HITS_LIMIT:
        raise ValueError(f"max_hits must be an integer in 1..{MAX_HITS_LIMIT}, got {max_hits!r}")


def scratch_bytes(n_rec: int, T_max: int, n_kw: int, U_max: int) -> int:
    """rs_rnnt_spot's per-pair scratch: the lattice and predecessor bytes of every cell, E and S of every frame."""
    return n_rec * n_kw * T_max * (9 * (U_max + 1) + 8)


def keyword_groups(lengths: Sequence[int], n_rec: int, T_max: int, cap: int = SCRATCH_CAP_BYTES) -> List[List[int]]:
    """Keyword indices sorted by token count and cut into groups whose scratch (``scratch_bytes`` with the group's longest
    keyword) stays at most ``cap``; a keyword alone above the cap is a group of its own."""
    order = sorted(range(len(lengths)), key=lambda k: lengths[k])
    groups: List[List[int]] = []
    for k in order:
        if groups and scratch_bytes(n_rec, T_max, len(groups[-1]) + 1, lengths[k]) <= cap:
            groups[-1].append(k)
        else:
            groups.append([k])
    return groups


def hit_seconds(s: int, e: int, duration: float):
    """Frames [s, e] of a recording of ``duration`` seconds -> (start, end): the seconds of frame s and the end of frame e,
    both clamped to the recording."""
    return segment_seconds(s, e, 0.0, duration)
