"""Caption alignment: locate each caption of a long recording inside its audio window, as ReazonSpeech's corpus builder
does for broadcast captions (pkg/espnet-oneseg/src/align.py:9-95), on the RNN-T lattice instead of a CTC trellis.

Live captions appear about 25 s after the speech.  So each caption gets the window [max(start - before, 0),
min(end + after, duration)) (before = 25 s, after = 0 as in the reference), and the segment alignment of alignment.py
finds where its tokens lie inside the window: the best segment [s, e] of encoder frames, its Viterbi score, and
log P(caption | the segment's audio).  The window is prepared as ``align_batch`` prepares an audio (norm_audio, 0.5 s of
silence on both sides), so frame f of the window lies at max(0.08 f - 0.5, 0) seconds into it, exactly as
``decode_hypothesis`` times a token.

``confidence`` ports CTC segmentation's score (R): the minimum, over windows of L consecutive frames of the segment, of the
mean per-frame log-probability of the path (the plain mean when the segment is at most L frames).  L = 15 frames is 1.2 s,
the span of CTC segmentation's default 30 frames at ESPnet's 40 ms.  A caption that is said in its window scores near 0; one
whose audio is missing has a stretch of frames with low log-probabilities and scores far below.

This module holds the host-side arithmetic; ``nemo.asr.align_captions`` runs it."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np

BEFORE_SECONDS = 25.0        # live captions trail the speech by about this much (align.py:22, _MARGIN)
AFTER_SECONDS = 0.0
CONFIDENCE_FRAMES = 15
SECONDS_PER_FRAME = 0.08     # encoder frame period (decode.SECONDS_PER_STEP)
PAD_SECONDS = 0.5            # silence added on both sides of a window (decode.PAD_SECONDS)


@dataclass
class Caption:
    """A caption and the program time it was shown at (the fields of pkg/espnet-oneseg/src/interface.py's Caption)."""
    start_seconds: float
    end_seconds: float
    text: str


@dataclass
class AlignedCaption:
    """Where a caption was found: its segment in program seconds, the caption's tokens as subwords timed in program seconds,
    score = the segment path's log-probability, log_likelihood = log P(caption | the segment's audio), confidence (see the
    module docstring); with ``transcribe=True``, asr = the transcript of the segment and cer = its CER against the caption."""
    caption: Caption
    start_seconds: float
    end_seconds: float
    text: str
    subwords: List[Any] = field(default_factory=list)
    score: float = math.nan
    log_likelihood: float = math.nan
    confidence: float = math.nan
    asr: Optional[str] = None
    cer: Optional[float] = None


def caption_window(caption: Caption, duration: float, before: float = BEFORE_SECONDS,
                   after: float = AFTER_SECONDS) -> Optional[Tuple[float, float]]:
    """-> (w0, w1) = [max(start - before, 0), min(end + after, duration)) in program seconds, or None when that is empty.
    ValueError when the caption ends before it starts."""
    if caption.end_seconds < caption.start_seconds:
        raise ValueError(f"caption ends at {caption.end_seconds} s before it starts at {caption.start_seconds} s: {caption.text!r}")
    w0 = max(float(caption.start_seconds) - before, 0.0)
    w1 = min(float(caption.end_seconds) + after, float(duration))
    return (w0, w1) if w1 > w0 else None


def window_samples(w0: float, w1: float, samplerate: int) -> Tuple[int, int]:
    """Sample range of a window, cut as the reference cuts it (align.py:17-20)."""
    return int(w0 * samplerate), int(w1 * samplerate)


def frame_seconds(frame: int) -> float:
    """Seconds of encoder frame ``frame`` of a window into the window (the 0.5 s pad removed, as decode_hypothesis does)."""
    return max(SECONDS_PER_FRAME * frame - PAD_SECONDS, 0.0)


def segment_seconds(s: int, e: int, w0: float, w1: float) -> Tuple[float, float]:
    """Frames [s, e] of the window [w0, w1) -> (start, end) program seconds: start = the seconds of frame s, end = the end of
    frame e; both clamped to the window."""
    start = min(w0 + frame_seconds(s), w1)
    end = min(w0 + frame_seconds(e + 1), w1)
    return start, max(end, start)


def confidence(frame_lp: Sequence[float], frames: int = CONFIDENCE_FRAMES) -> float:
    """The minimum over windows of ``frames`` consecutive entries of their mean (the plain mean of a shorter run), float64."""
    x = np.asarray(frame_lp, dtype=np.float64)
    if frames < 1:
        raise ValueError(f"confidence frames must be >= 1, got {frames}")
    if x.size == 0:
        return math.nan
    if x.size <= frames:
        return float(x.mean())
    c = np.concatenate([[0.0], np.cumsum(x)])
    return float(((c[frames:] - c[:-frames]) / frames).min())


def read_captions_tsv(path: str) -> List[Caption]:
    """``start<TAB>end<TAB>text`` lines (what the TSV writer writes, its header line included) -> captions.  Blank lines are
    skipped; any other line that is not two numbers and a text raises ValueError naming the line."""
    out = []
    with open(path, encoding="utf-8") as f:
        for n, line in enumerate(f.read().splitlines(), 1):
            if not line.strip() or (n == 1 and line.startswith("start_seconds\t")):
                continue
            parts = line.split("\t", 2)
            try:
                out.append(Caption(float(parts[0]), float(parts[1]), parts[2]))
            except (IndexError, ValueError):
                raise ValueError(f"{path}:{n}: expected start<TAB>end<TAB>text, got {line!r}") from None
    return out
