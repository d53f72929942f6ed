"""Long-form forced alignment: the band of the RNN-T lattice that a transcript without timestamps is aligned in.

The full lattice of an hour of speech (T ~ 45 000 frames, U ~ 30 000 tokens) has more than a billion cells, so the
transcript is anchored on the recording's greedy transcript and aligned only in a band around the anchors (banded
alignment, alignment.py), as recursive / anchor-based aligners do.

1. Anchors.  The transcript's tokens are matched to the greedy transcript's by
   ``difflib.SequenceMatcher(None, transcript, greedy, autojunk=False).get_matching_blocks()`` (deterministic, in the
   standard library).  A matched transcript token takes its greedy token's frame as its anchor; the others have none.
2. Band per row.  Token k (0-based) is the vertical step from label row k to row k + 1, so row r lies between the emissions
   of tokens r - 1 and r.  Token k spans [a_k, b_k]: a matched token [f_k, f_k]; an unmatched one the whole gap
   [f_prev, f_next] between its neighbouring anchors (0 before the first anchor, T - 1 after the last), so a stretch the ASR
   missed is searched over all of it.  Row r gets [a_{r-1} - W, b_r + W] (row 0 starts at 0, row U ends at T), clipped to
   [0, T): every anchor f gets at least [f - W, f + W] in both rows it joins.
3. Validity.  The rows are only ever widened: lo takes the running minimum from the top row down and hi the running
   maximum upward (so both are non-decreasing), then hi[r] >= lo[r + 1] + 1 makes consecutive rows overlap.
4. Widening.  When the alignment reports edge > 0 (a token on an interior band edge), W doubles and the transcript is aligned
   once more, at most ``max_widen`` times; the W used is reported.

W = band_seconds / 0.08 frames.  The default of 4 s is NOT calibrated: only synthetic weights are reachable offline, and how
far real speech strays from its greedy frames cannot be measured with them."""
from __future__ import annotations

import difflib
from typing import Callable, List, Sequence, Tuple

import numpy as np

BAND_SECONDS = 4.0
MAX_WIDEN = 2
SECONDS_PER_FRAME = 0.08          # encoder frame period (decode.SECONDS_PER_STEP)
MAX_PITCH = 227 * 1024 // 16      # rows of one diagonal the banded DP holds in shared memory (align.cu, band_dp_smem)


def band_frames(band_seconds: float) -> int:
    """W in frames; ValueError unless band_seconds is a positive finite number."""
    if isinstance(band_seconds, bool) or not isinstance(band_seconds, (int, float)) or not 0 < float(band_seconds) < float("inf"):
        raise ValueError(f"band_seconds must be a positive number of seconds, got {band_seconds!r}")
    return max(1, int(round(float(band_seconds) / SECONDS_PER_FRAME)))


def check_widen(max_widen) -> int:
    if isinstance(max_widen, bool) or not isinstance(max_widen, (int, np.integer)) or int(max_widen) < 0:
        raise ValueError(f"max_widen must be an integer >= 0, got {max_widen!r}")
    return int(max_widen)


def anchors(transcript: Sequence[int], greedy: Sequence[int], greedy_frames: Sequence[int]) -> np.ndarray:
    """-> int64 [U]: the greedy frame of each transcript token matched to a greedy token, -1 for the others."""
    out = np.full(len(transcript), -1, dtype=np.int64)
    sm = difflib.SequenceMatcher(None, list(transcript), list(greedy), autojunk=False)
    for i, j, n in sm.get_matching_blocks():
        out[i:i + n] = np.asarray(greedy_frames[j:j + n], dtype=np.int64)
    return out


def build_band(anchor: Sequence[int], T: int, W: int) -> Tuple[np.ndarray, np.ndarray]:
    """The band (steps 2 and 3 above) of a transcript of U = len(anchor) tokens over T frames -> lo, hi int32 [U + 1]."""
    a = np.asarray(anchor, dtype=np.int64)
    U = len(a)
    if T < 1:
        raise ValueError(f"no encoder frame to align in (T = {T})")
    known = a >= 0
    idx = np.arange(U)
    # previous / next anchor of every token (itself when matched)
    prev_i = np.maximum.accumulate(np.where(known, idx, -1)) if U else idx
    next_i = np.minimum.accumulate(np.where(known, idx, U)[::-1])[::-1] if U else idx
    a_k = np.where(prev_i >= 0, a[np.maximum(prev_i, 0)], 0) if U else a
    b_k = np.where(next_i < U, a[np.minimum(next_i, U - 1)], T - 1) if U else a
    lo = np.zeros(U + 1, dtype=np.int64)
    hi = np.full(U + 1, T, dtype=np.int64)
    lo[1:] = a_k - W
    hi[:U] = b_k + W + 1
    lo = np.clip(lo, 0, T - 1)
    hi = np.clip(hi, 1, T)
    lo = np.minimum.accumulate(lo[::-1])[::-1]
    hi[:U] = np.maximum(hi[:U], lo[1:] + 1)
    hi = np.maximum.accumulate(hi)
    lo[0], hi[U] = 0, T
    return lo.astype(np.int32), hi.astype(np.int32)


def check_band(lo: Sequence[int], hi: Sequence[int], T: int) -> None:
    """ValueError unless lo / hi [U + 1] are a valid band over T frames (alignment.py, "Banded alignment")."""
    lo, hi = np.asarray(lo, dtype=np.int64), np.asarray(hi, dtype=np.int64)
    if lo.ndim != 1 or lo.shape != hi.shape or len(lo) < 1:
        raise ValueError("the band needs lo and hi of one equal length U + 1 >= 1")
    if lo[0] != 0 or hi[-1] != T:
        raise ValueError(f"the band must start at frame 0 in row 0 and end at T = {T} in the last row (got {lo[0]}, {hi[-1]})")
    bad = np.nonzero((lo < 0) | (lo >= hi) | (hi > T))[0]
    if len(bad):
        raise ValueError(f"row {bad[0]}: band [{lo[bad[0]]}, {hi[bad[0]]}) is empty or outside [0, {T})")
    bad = np.nonzero((np.diff(lo) < 0) | (np.diff(hi) < 0))[0]
    if len(bad):
        raise ValueError(f"row {bad[0] + 1}: the band decreases")
    bad = np.nonzero(lo[1:] >= hi[:-1])[0]
    if len(bad):
        raise ValueError(f"rows {bad[0]} and {bad[0] + 1} do not overlap")


def band_offsets(lo: np.ndarray, hi: np.ndarray, label_len: Sequence[int]) -> Tuple[List[np.ndarray], int]:
    """Banded storage of a batch (lo / hi [B, >= U_b + 1]): the offset of every row u <= U_b, in (b, u) order -> ([off_b], cells)."""
    out, cells = [], 0
    for b, n in enumerate(label_len):
        w = (np.asarray(hi[b][: n + 1], dtype=np.int64) - np.asarray(lo[b][: n + 1], dtype=np.int64))
        out.append(cells + np.concatenate([[0], np.cumsum(w)[:-1]]))
        cells += int(w.sum())
    return out, cells


def widest_diagonal(lo: Sequence[int], hi: Sequence[int], T: int) -> Tuple[int, int, int]:
    """The diagonal d = t + u that meets the most rows: -> (extent, u0, u1), the rows [u0, u1] it meets."""
    lo, hi = np.asarray(lo, dtype=np.int64), np.asarray(hi, dtype=np.int64)
    r = np.arange(len(lo))
    d = np.arange(T + len(lo) - 1)
    u1 = np.searchsorted(r + lo, d, side="right") - 1
    u0 = np.searchsorted(r + hi, d, side="right")
    k = int(np.argmax(u1 - u0))
    return int(u1[k] - u0[k] + 1), int(u0[k]), int(u1[k])


def check_extent(lo, hi, T: int) -> None:
    """ValueError naming the stretch of the transcript whose band is too wide for the banded DP."""
    n, u0, u1 = widest_diagonal(lo, hi, T)
    if n > MAX_PITCH:
        raise ValueError(f"tokens {u0}..{u1} share one stretch of frames [{int(lo[u1])}, {int(hi[u0])}): {n} rows on one diagonal, more "
                         f"than the banded alignment holds ({MAX_PITCH}); the transcript leaves a gap the audio does not fill, or "
                         f"band_seconds is too large")


def align_widening(run: Callable[[int], tuple], W: int, max_widen: int):
    """run(W) -> a result whose item 4 is edge; aligns with W, then with 2W, 4W, ... while edge > 0, at most max_widen more
    times -> (result, W used, alignments run)."""
    n = 1
    res = run(W)
    while int(res[4]) > 0 and n <= max_widen:
        W *= 2
        n += 1
        res = run(W)
    return res, W, n
