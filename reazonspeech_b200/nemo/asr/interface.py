"""Argument / result types of the ``reazonspeech.nemo.asr`` API.

Field names, order and defaults follow the reference dataclasses
(pkg/nemo-asr/src/interface.py:4-36) so results are interchangeable; the extra helpers are ours."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, List, Optional

import numpy as np


@dataclass
class AudioData:
    """A waveform (float array, mono [n] or channels-first [c, n]) and its sample rate."""
    waveform: np.ndarray
    samplerate: int

    @property
    def seconds(self) -> float:
        return self.waveform.shape[-1] / float(self.samplerate)


@dataclass
class Subword:
    """One emitted token with the time of the encoder frame that emitted it, and its confidence when the model was loaded
    with a ``ConfidenceConfig`` (None otherwise)."""
    seconds: float
    token_id: int
    token: str
    confidence: Optional[float] = None

    def as_dict(self) -> dict:
        d = {"seconds": self.seconds, "token_id": self.token_id, "token": self.token}
        if self.confidence is not None:
            d["confidence"] = self.confidence
        return d


@dataclass
class Segment:
    """A run of subwords ending at a sentence mark, a comma or a pause (decode.find_end_of_segment)."""
    start_seconds: float
    end_seconds: float
    text: str

    @property
    def duration(self) -> float:
        return self.end_seconds - self.start_seconds

    def as_dict(self) -> dict:
        return {"start_seconds": self.start_seconds, "end_seconds": self.end_seconds, "text": self.text}


@dataclass
class TranscribeResult:
    """What ``transcribe`` / ``transcribe_batch`` return.  ``hypothesis`` is only filled when the call was made with
    ``TranscribeConfig(raw_hypothesis=True)``; it then carries the engine's token ids and ALSD-shaped step counters."""
    text: str
    subwords: List[Subword]
    segments: List[Segment]
    hypothesis: Any = None

    def as_dict(self) -> dict:
        """Plain-Python form (no hypothesis) for JSON-lines outputs such as the evaluator's."""
        return {"text": self.text, "subwords": [w.as_dict() for w in self.subwords],
                "segments": [g.as_dict() for g in self.segments]}

    @property
    def token_ids(self) -> List[int]:
        return [w.token_id for w in self.subwords]


@dataclass
class TranscribeConfig:
    verbose: bool = True
    raw_hypothesis: bool = False
