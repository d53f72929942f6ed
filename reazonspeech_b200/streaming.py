"""Streaming transcription: live 16 kHz mono streams decoded chunk by chunk, many streams per batched engine call.

This is NeMo's buffered RNN-T inference with the "middle" merge and stateful greedy decoding (as recalled, (R)), batched
across streams.  It works with the offline-trained checkpoint: each chunk is encoded inside a buffer that adds left and right
audio context, and only the chunk's frames are decoded, continuing from the stream's carried decoder state.  Emitted tokens
are final and never revised, which is what live captioning wants.

Frame grid
    P = 1280 samples (hop 160 x subsampling 8 = 0.08 s).  A stream's signal is 0.5 s of zeros, then the pushed samples, then
    0.5 s of zeros appended at close -- exactly what ``transcribe()`` feeds the engine.  Global encoder frame f is frame f of
    that padded signal; a token at frame f gets ``seconds = max(0.08 f - 0.5, 0)``, as in ``decode_hypothesis``.

Configuration
    ``StreamingConfig(chunk_seconds, left_seconds, right_seconds)``, each a multiple of 0.08 s (anything else is rejected):
    C, Lc, R frames with C >= 1, Lc >= 0, R >= 0.  The defaults, a 1.6 s chunk in a 4.0 s buffer (1.2 s on either side),
    are NeMo's buffered-RNN-T example defaults as recalled (R).  What they cost in accuracy against offline decoding cannot
    be measured here: the project's weights are synthetic.

Schedule (``plan_row``)
    D = frames decoded so far, n = padded samples available.
    - A stream is ready when n >= (D + C + R) P, or when it is closed and has frames left.
    - Its buffer is the samples [a, b), a = max(0, D - Lc) P, b = min(n, (D + C + R) P).
    - The step decodes global frames [D, min(D + C, F)); F = ``rs_enc_valid`` of the whole padded stream once it is closed
      (what the offline decode runs over), unbounded before.
    - In buffer frames that is [D - a/P, ...).  Because a is a multiple of P, ``rs_enc_valid(b - a) = rs_enc_valid(b) - a/P``
      exactly (mel_valid 8m -> conv 4m -> 2m -> m), so the decoded range always lies inside the buffer's valid frames
      (tests/test_streaming_cpu.py checks this rather than assuming it).
    - A closed stream drains in ceil(remaining / C) steps, at most C frames per step.

Log-mel statistics are per buffer, as NeMo's buffered inference computes them: a buffer is just an utterance to the kernels.

Exactness anchor.  With Lc and R at least the stream's length and the whole audio fed and closed before the first step,
every buffer is the whole padded stream, every step's encoder output is bit-identical to the offline one, and the
concatenated chunked decode equals ``transcribe()``'s tokens, frames and statistics bit for bit.

Decoder state.  The engine keeps one record per stream on the device (``rs_stream_state_bytes``; include/rs_engine.h): the
LSTM cell state, W_hh . h, the joint's prediction projection, and the phrase-boosting and LM states.  An all-zero record is
a stream that has not started.
"""
from __future__ import annotations

from dataclasses import dataclass
from fractions import Fraction
from typing import NamedTuple, Optional

SAMPLERATE = 16000
HOP = 160
SUBSAMPLING = 8
P = HOP * SUBSAMPLING                  # samples per encoder frame (0.08 s)
PAD_SAMPLES = SAMPLERATE // 2          # 0.5 s of zeros on both sides of a stream
FRAME_SECONDS = Fraction(P, SAMPLERATE)


def _frames(seconds: float, what: str) -> int:
    q = Fraction(seconds).limit_denominator(10 ** 6) / FRAME_SECONDS
    n = round(q)
    if abs(q - n) > Fraction(1, 10 ** 4) or n < 0:
        raise ValueError(f"{what}={seconds!r} s must be a non-negative multiple of 0.08 s")
    return int(n)


@dataclass(frozen=True)
class StreamingConfig:
    """Chunk, left and right context in seconds, each a multiple of 0.08 s (one encoder frame)."""
    chunk_seconds: float = 1.6
    left_seconds: float = 1.2
    right_seconds: float = 1.2

    def __post_init__(self):
        if self.frames()[0] < 1:
            raise ValueError(f"chunk_seconds={self.chunk_seconds!r} must be at least one frame (0.08 s)")

    def frames(self):
        """(C, Lc, R) in encoder frames."""
        return (_frames(self.chunk_seconds, "chunk_seconds"), _frames(self.left_seconds, "left_seconds"),
                _frames(self.right_seconds, "right_seconds"))


def conv_len(n: int) -> int:
    return (n - 1) // 2 + 1 if n > 0 else 0


def enc_valid(n_samples: int) -> int:
    """``rs_enc_valid``: valid encoder frames of an utterance of ``n_samples`` (n_fft 512, hop 160)."""
    return conv_len(conv_len(conv_len(n_samples // HOP)))


class Row(NamedTuple):
    """One stream's row of a step: buffer samples [a, b) of the padded signal, decoded buffer frames [dec_begin, dec_end),
    and the global frame of buffer frame 0 (``offset`` = a / P)."""
    a: int
    b: int
    dec_begin: int
    dec_end: int
    offset: int


def stream_frames(n: int, closed: bool) -> Optional[int]:
    """F: the frames a stream decodes in all, known once it is closed (None before)."""
    return enc_valid(n) if closed else None


def plan_row(n: int, decoded: int, closed: bool, frames) -> Optional[Row]:
    """The step of a stream with ``n`` padded samples available and ``decoded`` frames done, or None when it is not ready.
    ``frames`` = ``StreamingConfig.frames()``."""
    C, Lc, R = frames
    D = decoded
    F = stream_frames(n, closed)
    if F is not None and D >= F:
        return None
    if not (n >= (D + C + R) * P or closed):
        return None
    a = max(0, D - Lc) * P
    b = min(n, (D + C + R) * P)
    end = D + C if F is None else min(D + C, F)
    off = a // P
    return Row(a, b, D - off, end - off, off)
