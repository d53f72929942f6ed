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
``open()`` once its stream has drained; ``result(id)`` stays available until then.

``open(boosting=...)`` gives a stream its own key phrases.  The lists of the open streams share one table (region 0: the
model's global list; ``boosting.stack_tables``), restacked at the next ``step()`` whenever the set of lists changes; every
record's automaton state is then moved from its list's old region to its new one (``remap_boost_states``), so a stream's
open partial match survives other streams opening and closing.  A list is built and checked in ``open()``: one with bad
token ids, or one that would take the open streams' lists and the global list past ``MAX_STATES`` states together, raises
ValueError there and takes no slot; ``model.set_phrase_boosting`` likewise refuses a global list that would not fit."""
from __future__ import annotations

import contextlib
import weakref
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from ...boosting import MAX_STATES, PhraseBoostingConfig, build_tables, config_key, stack_tables
from ...confidence import measure
from ...streaming import P, PAD_SAMPLES, StreamingConfig, plan_row, stream_frames
from .decode import PAD_SECONDS, SECONDS_PER_STEP, decode_hypothesis
from .interface import Subword, TranscribeResult
from .transcribe import B200RnntModel, HostStaging, greedy_hypothesis


_ALL_STATES = 1 << 30                            # the global list's region while no stream has its own: the whole table


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
    boosting: Optional[PhraseBoostingConfig] = None    # the stream's own phrase list; None: the model's global list


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
        self._layout = {None: (0, _ALL_STATES)}      # list key -> (start, states) of its region in the table in use
        self._layout_key = None                      # (global list key, the open streams' distinct list keys); None: rebuild
        self._tables = None                          # (device tables, roots by list key) while a stream has its own list
        self._built = {}                             # list key -> its build_tables, for the lists of the open streams
        model.__dict__.setdefault("_table_listeners", []).append(weakref.WeakMethod(self._tables_changed))
        model.__dict__.setdefault("_boost_checks", []).append(weakref.WeakMethod(self._check_global))

    # -- stream lifetime
    def open(self, boosting: Optional[PhraseBoostingConfig] = None) -> int:
        """A new stream -> its id (the smallest free record slot, which is zeroed: a stream that has not started).
        ``boosting``: the stream's own key phrases; None: the model's global list (``model.set_phrase_boosting``)."""
        if not self._free:
            raise RuntimeError(f"all {self.states.shape[0]} stream slots are in use")
        if boosting is not None:
            if not isinstance(boosting, PhraseBoostingConfig):
                raise ValueError(f"boosting must be a PhraseBoostingConfig or None, got {type(boosting).__name__}")
            key = config_key(boosting)
            tables = self._built.get(key)
            if tables is None:
                tables = build_tables(boosting, self.model.cfg.vocab_size, self.model.tokenizer)   # bad phrases raise here
            keys = self._own_keys() | {key}
            need = self._global_states(self.model.boosting_tables) + sum((self._built.get(k) or tables).n_states for k in keys)
            if need > MAX_STATES:
                raise ValueError(f"this stream's phrase list would take the {len(keys)} distinct lists of the open streams and the "
                                 f"global list to {need} automaton states, more than {MAX_STATES}")
            self._built[key] = tables
        slot = min(self._free)
        self._free.remove(slot)
        self.states[slot].zero_()
        self._finished.pop(slot, None)
        self._live[slot] = _Stream(slot, np.zeros(PAD_SAMPLES, np.int16), boosting=boosting)
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
        if ready:
            self._update_tables()
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
        with contextlib.ExitStack() as stack:
            if eng.device.type == "cuda":
                stack.enter_context(torch.cuda.device(eng.device))
            if self._tables is not None:
                dev, root_of = self._tables
                stack.enter_context(model.phrase_tables_set(dev))
                eng.set_boost_roots([root_of[config_key(self._live[sid].boosting)] for sid, _ in batch])
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
        """The model's boosting (word 1) or LM (word 2) tables changed: every open stream restarts that state from the root.
        Streams with their own phrase list keep their boosting state: it moves with their region at the next step."""
        slots = [s.slot for s in self._live.values() if word == 2 or s.boosting is None]
        if slots:
            self.states.view(torch.int32)[torch.tensor(slots, device=self.states.device), word] = -1
        if word == 1:
            self._layout_key = None

    def _own_keys(self) -> set:
        return {config_key(s.boosting) for s in self._live.values() if s.boosting is not None}

    @staticmethod
    def _global_states(tables) -> int:
        return 1 if tables is None else tables.n_states       # region 0: the global list, or the 1-state empty automaton

    def _check_global(self, tables) -> None:
        """Called by the model before its global list changes: refuse one that the open streams' lists cannot share a table with."""
        keys = self._own_keys()
        need = self._global_states(tables) + sum(self._built[k].n_states for k in keys)
        if keys and need > MAX_STATES:
            raise ValueError(f"the new global phrase list and the {len(keys)} distinct lists of the open streams would need {need} "
                             f"automaton states, more than {MAX_STATES}; the global list is unchanged")

    def _update_tables(self) -> None:
        """Restack the table of the open streams' lists when their set (or the global list) changed, and move every record's
        automaton state into its list's new region.  Every list was built and the total checked when it was accepted."""
        model = self.model
        order = list(dict.fromkeys(config_key(self._live[sid].boosting) for sid in sorted(self._live)
                                   if self._live[sid].boosting is not None))
        key = (config_key(model.boosting), frozenset(order))
        if key == self._layout_key:
            return
        self._built = {k: self._built[k] for k in order}
        tables = None
        layout = {None: (0, _ALL_STATES)}            # only the global list: the model's own setting, no roots
        if order:
            base = model.boosting_tables
            if base is None:
                base = build_tables(PhraseBoostingConfig(), model.cfg.vocab_size)
            stacked, starts = stack_tables([base] + [self._built[k] for k in order], model.cfg.vocab_size)
            dev = tuple(torch.as_tensor(a).to(model.engine.device) for a in (stacked.bonus, stacked.next))
            layout = {None: (0, base.n_states)}
            layout.update({k: (at, self._built[k].n_states) for k, at in zip(order, starts[1:])})
            tables = (dev, {k: at for k, (at, _) in layout.items()})
        streams = list(self._live.values())
        if streams and (tables is not None or self._tables is not None):
            old = [self._layout.get(config_key(s.boosting), (0, 0)) for s in streams]
            new = [layout[config_key(s.boosting)][0] for s in streams]
            w = self.states.view(torch.int32)
            idx = torch.tensor([s.slot for s in streams], device=self.states.device)
            as_t = lambda v: torch.tensor(v, dtype=torch.int32, device=self.states.device)
            w[idx, 1] = remap_boost_states(w[idx, 1], as_t([o[0] for o in old]), as_t([o[1] for o in old]), as_t(new))
        self._layout, self._layout_key, self._tables = layout, key, tables


def remap_boost_states(state: torch.Tensor, old_start: torch.Tensor, old_size: torch.Tensor, new_start: torch.Tensor) -> torch.Tensor:
    """The boost_state words of stream records moved between table layouts: a state inside its list's old region
    [old_start, old_start + old_size) keeps its place in the region (new = old - old_start + new_start); anything else
    (-1, a state of another layout) becomes the region's new root."""
    inside = (state >= old_start) & (state < old_start + old_size)
    return torch.where(inside, state - old_start + new_start, new_start)
