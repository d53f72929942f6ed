"""``StreamingTranscriber``: many live 16 kHz mono streams decoded chunk by chunk on one GPU (semantics:
reazonspeech_b200/streaming.py).

    st = StreamingTranscriber(model)             # a single-GPU greedy model from load_model()
    sid = st.open()
    st.feed(sid, samples)                        # float32 or int16, any piece size
    for sid, subwords in st.step().items(): ...  # the tokens that became final in this step
    st.close(sid)
    while not st.done(sid): st.step()
    result = st.result(sid)                      # TranscribeResult, as transcribe() would give

Every ``step()`` advances each ready stream by one chunk: one ``rs_stream_step`` engine call per ``model.max_batch`` ready
streams.  The decoder states live in one device tensor ``[max_streams, rs_stream_state_bytes]``; a stream holds one record
from ``open()`` until it has been closed and fully decoded.  Stream ids are the record slots, so an id is reused by a later
``open()`` once its stream has drained; ``result(id)`` stays available until then."""
from __future__ import annotations

import contextlib
import weakref
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np
import torch

from ...confidence import measure
from ...streaming import P, PAD_SAMPLES, StreamingConfig, plan_row, stream_frames
from .decode import PAD_SECONDS, SECONDS_PER_STEP, decode_hypothesis
from .interface import Subword, TranscribeResult
from .transcribe import B200RnntModel, HostStaging, greedy_hypothesis


@dataclass
class _Stream:
    slot: int
    buf: np.ndarray                    # padded samples [base, n) still needed (int16 while every piece was int16)
    base: int = 0
    n: int = PAD_SAMPLES               # padded samples available
    decoded: int = 0                   # global frames decoded
    closed: bool = False
    tokens: List[int] = field(default_factory=list)
    frames: List[int] = field(default_factory=list)
    stats: List[np.ndarray] = field(default_factory=list)


class StreamingTranscriber:
    """Live streams on one single-GPU greedy model (``B200RnntModel``).  Use one transcriber per device for several GPUs."""

    def __init__(self, model, config: StreamingConfig = StreamingConfig(), max_streams: int = 256):
        if not isinstance(model, B200RnntModel):
            raise ValueError("StreamingTranscriber runs on one GPU: pass a single-device model (one transcriber per device)")
        if model.decoding != "greedy":
            raise ValueError("streaming decodes greedily (ALSD beam search does not stream)")
        if model.cfg.n_window_stride * 8 != P or model.cfg.sample_rate != 16000:
            raise ValueError("streaming needs the 16 kHz, 10 ms hop, 8x subsampling frame grid")
        if max_streams < 1:
            raise ValueError("max_streams must be >= 1")
        self.model, self.config = model, config
        self.frames_cfg = config.frames()
        eng = model.engine
        self.states = torch.zeros(max_streams, eng.stream_state_bytes, dtype=torch.uint8, device=eng.device)
        self._free = list(range(max_streams))
        self._live: Dict[int, _Stream] = {}
        self._finished: Dict[int, TranscribeResult] = {}
        self._staging = HostStaging(torch.cuda.is_available())
        model.__dict__.setdefault("_table_listeners", []).append(weakref.WeakMethod(self._tables_changed))

    # -- stream lifetime
    def open(self) -> int:
        """A new stream -> its id (the smallest free record slot, which is zeroed: a stream that has not started)."""
        if not self._free:
            raise RuntimeError(f"all {self.states.shape[0]} stream slots are in use")
        slot = min(self._free)
        self._free.remove(slot)
        self.states[slot].zero_()
        self._finished.pop(slot, None)
        self._live[slot] = _Stream(slot, np.zeros(PAD_SAMPLES, np.int16))
        return slot

    def _stream(self, sid: int) -> _Stream:
        s = self._live.get(sid)
        if s is None:
            raise KeyError(f"no open stream {sid}")
        return s

    def feed(self, sid: int, samples) -> None:
        """Append 16 kHz mono samples (1-D float32 or int16; int16 is PCM, scaled by 2^-15).  Anything else raises: resampling
        a stream is stateful and not done here."""
        s = self._stream(sid)
        if s.closed:
            raise ValueError(f"stream {sid} is closed")
        if isinstance(samples, torch.Tensor):
            samples = samples.detach().cpu().numpy()
        x = np.asarray(samples)
        if x.ndim != 1 or x.dtype not in (np.float32, np.int16):
            raise ValueError(f"feed() takes 1-D 16 kHz mono float32 or int16 samples, got {x.dtype} {x.shape}")
        self._append(s, x)

    def _append(self, s: _Stream, x: np.ndarray) -> None:
        if s.buf.dtype == np.int16 and x.dtype == np.float32:
            s.buf = s.buf.astype(np.float32) * np.float32(1.0 / 32768.0)
        elif s.buf.dtype == np.float32 and x.dtype == np.int16:
            x = x.astype(np.float32) * np.float32(1.0 / 32768.0)
        s.buf = np.concatenate([s.buf, x])
        s.n += len(x)

    def close(self, sid: int) -> None:
        """No more audio: 0.5 s of zeros is appended and the stream drains in the following steps."""
        s = self._stream(sid)
        if not s.closed:
            self._append(s, np.zeros(PAD_SAMPLES, s.buf.dtype))
            s.closed = True

    def done(self, sid: int) -> bool:
        """The stream has been closed and every frame decoded."""
        return sid in self._finished and sid not in self._live

    def result(self, sid: int) -> TranscribeResult:
        """``decode_hypothesis`` of all of a drained stream's tokens: text, subwords, segments and (with confidence) word
        confidence over the whole stream, as ``transcribe()`` gives them.  ``result.hypothesis`` carries all of the stream's
        token ids and their global frames (``Hypothesis``, as ``TranscribeConfig(raw_hypothesis=True)`` gives it)."""
        if sid not in self._finished:
            raise KeyError(f"stream {sid} has not drained (close it and step until done)")
        return self._finished[sid]

    @property
    def open_streams(self) -> List[int]:
        return sorted(self._live)

    # -- decoding
    def plan(self) -> List[tuple]:
        """The (stream id, Row) of every ready stream, in id order."""
        out = []
        for sid in sorted(self._live):
            s = self._live[sid]
            row = plan_row(s.n, s.decoded, s.closed, self.frames_cfg)
            if row is not None:
                out.append((sid, row))
        return out

    def step(self) -> Dict[int, List[Subword]]:
        """Advance every ready stream by one chunk -> {id: subwords that became final} for the streams that stepped."""
        ready = self.plan()
        out: Dict[int, List[Subword]] = {}
        mb = max(1, int(self.model.max_batch))
        for lo in range(0, len(ready), mb):
            out.update(self._run(ready[lo:lo + mb]))
        # streams that are closed and have no frames left (e.g. closed right after a step that reached F) finish here too
        for sid in [sid for sid, s in self._live.items() if s.closed and s.decoded >= stream_frames(s.n, True)]:
            self._finish(sid)
        return out

    def _run(self, batch) -> Dict[int, List[Subword]]:
        model, eng = self.model, self.model.engine
        C = self.frames_cfg[0]
        waves = [self._live[sid].buf[row.a - self._live[sid].base: row.b - self._live[sid].base] for sid, row in batch]
        wav, lens = self._staging.stage(waves, 0)
        B, U = len(batch), C * model.cfg.max_symbols
        conf = getattr(model, "confidence", None)
        alpha = conf.alpha if conf is not None else None
        out = self._staging.outputs(B, U, stats=alpha is not None)
        col = lambda k: torch.tensor([getattr(row, k) for _, row in batch], dtype=torch.int32)
        slot = torch.tensor([self._live[sid].slot for sid, _ in batch], dtype=torch.int32)
        with torch.cuda.device(eng.device) if eng.device.type == "cuda" else contextlib.nullcontext():
            eng.stream_step(wav, lens, col("dec_begin"), col("dec_end"), slot, self.states, U, out, alpha=alpha)
        tokens, frames, ntok = out[:3]
        res: Dict[int, List[Subword]] = {}
        for r, (sid, row) in enumerate(batch):
            s = self._live[sid]
            n = int(ntok[r])
            toks = tokens[r, :n].tolist()
            frs = [f + row.offset for f in frames[r, :n].tolist()]
            st = out[3][r, :n].numpy().astype(np.float64) if alpha is not None else None
            s.tokens += toks
            s.frames += frs
            if st is not None:
                s.stats.append(st)
            s.decoded = row.dec_end + row.offset
            keep = max(0, s.decoded - self.frames_cfg[1]) * P          # the next buffer's start: earlier samples are not needed
            if keep > s.base:
                s.buf = s.buf[keep - s.base:]
                s.base = keep
            res[sid] = self._subwords(toks, frs, st)
        return res

    def _subwords(self, toks, frs, st) -> List[Subword]:
        model = self.model
        tc = None
        if st is not None and len(toks):
            tc = [float(x) for x in measure(st, model.cfg.vocab_size + 1, model.confidence.method_cfg)]
        subs = []
        for i, (k, f) in enumerate(zip(toks, frs)):
            piece = model.tokenizer.ids_to_text([k])
            if piece:
                subs.append(Subword(max(SECONDS_PER_STEP * f - PAD_SECONDS, 0), k, piece, None if tc is None else tc[i]))
        return subs

    def _finish(self, sid: int) -> None:
        s = self._live.pop(sid)
        item = (s.tokens, s.frames)
        if getattr(self.model, "confidence", None) is not None:
            item += (np.concatenate(s.stats) if s.stats else np.zeros((0, 4)),)
        hyp = greedy_hypothesis(self.model, item)
        res = decode_hypothesis(self.model, hyp)
        res.hypothesis = hyp
        self._finished[sid] = res
        self._free.append(s.slot)

    def _tables_changed(self, word: int) -> None:
        """The model's boosting (word 1) or LM (word 2) tables changed: every open stream restarts that state from the root."""
        slots = [s.slot for s in self._live.values()]
        if slots:
            self.states.view(torch.int32)[torch.tensor(slots, device=self.states.device), word] = -1
