"""``load_model`` / ``transcribe`` with the reference's signatures (pkg/nemo-asr/src/transcribe.py:9-60)
on top of the H100 engine, plus the batched ``transcribe_batch`` the reference lacks
(its evaluators leave ``_evaluate_batch`` unimplemented, pkg/evaluation/examples/rs-nemo/eval.py:31-32).

The object returned by ``load_model`` is a duck-typed stand-in for NeMo's EncDecRNNTBPEModel at
exactly the three points the reference touches it (SURVEY.md section 8b):
``model.transcribe(list_of_tensors, batch_size=..., return_hypotheses=True, verbose=...)``,
``hyp.y_sequence`` / ``hyp.timestamp`` and ``model.tokenizer.ids_to_text``; the reference's own
transcribe()/decode_hypothesis() therefore run unmodified on it (see INTEGRATION.md)."""
from __future__ import annotations

import contextlib
import dataclasses
import glob
import math
import os
from dataclasses import dataclass
from functools import partial
from typing import List, Optional, Sequence

import numpy as np
import torch

from ...alignment import alignment_hypothesis, pack_labels, validate_labels
from ...captions import AFTER_SECONDS, BEFORE_SECONDS, CONFIDENCE_FRAMES, AlignedCaption, Caption, caption_window
from ...boosting import PhraseBoostingConfig, PhraseBoostingTables, build_tables, combine_tables, config_key
from ...config import MaesConfig, ModelConfig
from ...confidence import ConfidenceConfig, measure, word_confidence
from ...engine import MAX_NBEST, Engine
from ...evaluation.utils import calculate_cer, normalize
from ...ngram_lm import NgramLMConfig, NgramLMTables, build_lm_tables
from ...tokenizer import PieceTableTokenizer, SentencePieceTokenizer, synthetic_pieces
from ...weights import load_nemo_archive, random_state_dict
from .audio import SAMPLERATE, norm_audio, pad_audio
from .decode import PAD_SECONDS, build_result, decode_hypothesis
from .interface import AudioData, TranscribeConfig, TranscribeResult

HF_REPO = "reazon-research/reazonspeech-nemo-v2"
ENV_CHECKPOINT = "REAZONSPEECH_NEMO_CHECKPOINT"
ENV_SYNTHETIC = "REAZONSPEECH_B200_SYNTHETIC"


@dataclass
class Hypothesis:
    """The two NeMo Hypothesis fields the reference reads (decode.py:40,44), ALSD-shaped:
    y_sequence = [blank, tok_0, ...]; timestamp[i] = frame_i + i + 1 so that decode.py:48's
    ``step - idx - 1`` recovers the emitting encoder frame."""
    y_sequence: torch.Tensor
    timestamp: List[int]
    score: float = 0.0
    token_confidence: Optional[List[float]] = None
    word_confidence: Optional[List[float]] = None
    log_likelihood: Optional[float] = None          # forced alignment: log P(y | x) of the given transcript (alignment.py)
    token_logprob: Optional[List[float]] = None     # forced alignment: each token's log-probability on the Viterbi path

    @staticmethod
    def from_greedy(tokens: Sequence[int], frames: Sequence[int], blank: int) -> "Hypothesis":
        y = torch.tensor([blank, *[int(t) for t in tokens]], dtype=torch.long)
        return Hypothesis(y, [int(f) + i + 1 for i, f in enumerate(frames)])


def greedy_hypothesis(model, item) -> Hypothesis:
    """One item of ``iter_token_batches`` -> Hypothesis.  With confidence on, the item carries the utterance's statistics
    rows (lp, H1, A_alpha, G_alpha) and the hypothesis gets token / word confidence and score = sum of the emitted tokens'
    log-probabilities.  (NeMo's greedy loop adds the joint's maximum output, which is a log-probability only where the joint
    is log-normalised (R): the sum of log-probabilities is the score a corpus filter can compare across utterances.)"""
    hyp = Hypothesis.from_greedy(item[0], item[1], model.cfg.blank)
    conf: Optional[ConfidenceConfig] = getattr(model, "confidence", None)
    if conf is not None:
        stats = np.asarray(item[2], dtype=np.float64).reshape(-1, 4)
        tc = [float(x) for x in measure(stats, model.cfg.vocab_size + 1, conf.method_cfg)]
        hyp.token_confidence = tc
        hyp.word_confidence = word_confidence(tc, model.tokenizer.ids_to_pieces(item[0]), conf.aggregation)
        hyp.score = float(stats[:, 0].sum())
    return hyp


class HostStaging:
    """Grow-only host buffers of one in-flight batch, reused across calls and pinned when a CUDA device is there:
    allocating (cudaHostAlloc) and zero-filling a fresh 64 MB pinned batch costs more than the batch's GPU time."""

    def __init__(self, pin: bool):
        self.pin = pin
        self._wav = self._lens = self._tok = self._frm = self._ntok = None

    def _grown(self, buf, numel: int, dtype):
        if buf is None or buf.numel() < numel:
            buf = torch.empty(int(numel * 1.25) + 16, dtype=dtype)
            if self.pin:
                buf = buf.pin_memory()
        return buf

    def stage(self, waves: Sequence[np.ndarray], pad: int):
        """Rows ``[zeros(pad) | wave | zeros(pad) | zeros to L]`` (pad_audio, audio.py:70-83, written in place) -> (wav [B, L], lens [B]).

        A batch whose waveforms are ALL 16-bit PCM (int16 arrays, e.g. ``audio_from_path(..., pcm16=True)``) is staged as
        int16 and scaled by 2^-15 on the device (rs_transcribe_batch_pcm16): half the pinned memory and PCIe bytes.  A mixed
        batch is staged as float32, int16 members converted the way a file decoder would (sample / 32768)."""
        B = len(waves)
        L = max(len(w) for w in waves) + 2 * pad
        L = (L + 3) & ~3                                # rows start 8 / 16-byte aligned: the kernel's vectorised staging load
        pcm = all(w.dtype == np.int16 for w in waves)
        if pcm:
            self._wav16 = self._grown(getattr(self, "_wav16", None), B * L, torch.int16)
            wav = self._wav16[: B * L].view(B, L)
        else:
            self._wav = self._grown(self._wav, B * L, torch.float32)
            wav = self._wav[: B * L].view(B, L)
        self._lens = self._grown(self._lens, B, torch.int32)
        lens = self._lens[:B]
        # the copies run in the library (rs_stage_rows: memcpy split over a few threads, interpreter lock released): the
        # same loop as numpy slice assignments cost ~0.5 ms per 30 s clip, as much as the GPU spends on it
        import ctypes as C
        from ...engine import load_library
        srcs = [np.ascontiguousarray(w if w.dtype in (np.int16, np.float32) else w.astype(np.float32)) for w in waves]
        ptr = (C.c_void_p * B)(*[a.ctypes.data for a in srcs])
        n = (C.c_int64 * B)(*[a.shape[0] for a in srcs])
        is16 = (C.c_int32 * B)(*[int(a.dtype == np.int16) for a in srcs])
        rc = load_library().rs_stage_rows(wav.data_ptr(), L, ptr, n, is16, int(pcm), B, pad, min(4, B))
        if rc != 0:
            raise RuntimeError(f"rs_stage_rows failed ({rc})")
        lens.copy_(torch.tensor([a.shape[0] + 2 * pad for a in srcs], dtype=torch.int32))
        return wav, lens

    def outputs(self, B: int, U: int, stats: bool = False):
        """(tokens [B, U], frames [B, U], n_tok [B]), plus the confidence statistics [B, U, 4] with ``stats``."""
        self._tok = self._grown(self._tok, B * U, torch.int32)
        self._frm = self._grown(self._frm, B * U, torch.int32)
        self._ntok = self._grown(self._ntok, B, torch.int32)
        out = self._tok[: B * U].view(B, U), self._frm[: B * U].view(B, U), self._ntok[:B]
        if not stats:
            return out
        self._stats = self._grown(getattr(self, "_stats", None), B * U * 4, torch.float32)
        return out + (self._stats[: B * U * 4].view(B, U, 4),)


class B200RnntModel:
    """Engine + tokenizer behind NeMo's model surface."""

    def __init__(self, engine: Engine, tokenizer, max_batch: int = 64, decoding: str = "greedy", beam_size: int = 4,
                 confidence: Optional[ConfidenceConfig] = None, boosting: Optional[PhraseBoostingConfig] = None,
                 lm: Optional[NgramLMConfig] = None, maes: Optional[MaesConfig] = None):
        self.engine = engine
        self.cfg = engine.cfg
        self.tokenizer = tokenizer
        self.max_batch = max_batch
        self.decoding, self.beam_size = decoding, beam_size       # "greedy" (north_star's parity target), "alsd" (the checkpoint's default) or "maes"
        self.maes = (maes or MaesConfig()).check_beam(beam_size, engine.cfg.vocab_size) if decoding == "maes" else None
        if confidence is not None and decoding != "greedy":
            raise ValueError("confidence is computed by the greedy decode only (NeMo offers none for beam search)")
        self.confidence = confidence.validate() if confidence is not None else None
        pin = torch.cuda.is_available()
        self._staging = (HostStaging(pin), HostStaging(pin))      # double buffer: stage batch k+1 while batch k runs
        self._phrase_cache = None                                 # (key, device tables, {list key: root}) of the last phrases= call
        self.boosting: Optional[PhraseBoostingConfig] = None
        self.boosting_tables: Optional[PhraseBoostingTables] = None   # host tables of the global list (streams build on them)
        if boosting is not None:
            self.set_phrase_boosting(boosting)
        self.lm: Optional[NgramLMConfig] = None
        if lm is not None:
            self.set_ngram_lm(lm)

    def set_ngram_lm(self, lm: Optional[NgramLMConfig]) -> None:
        """Fuse the n-gram LM of ``lm`` into every following greedy decode (ngram_lm.py), or stop with None.  Call it between
        calls, not while one is running."""
        self.set_ngram_lm_tables(lm_tables(self, lm), lm)

    def set_ngram_lm_tables(self, tables: Optional[NgramLMTables], lm: Optional[NgramLMConfig]) -> None:
        """Upload tables already built from ``lm`` (the multi-GPU model builds them once for all replicas)."""
        self.engine.set_ngram_lm(tables)
        self.lm = lm
        self._notify_tables(2)

    def _notify_tables(self, word: int) -> None:
        """Open streams (``StreamingTranscriber``) restart their boosting (word 1) or LM (word 2) state from the root."""
        for ref in list(self.__dict__.get("_table_listeners", ())):
            fn = ref()
            if fn is not None:
                fn(word)

    def set_phrase_boosting(self, boosting: Optional[PhraseBoostingConfig]) -> None:
        """Boost the phrases of ``boosting`` in every following greedy decode (boosting.py), or stop with None.  Call it
        between calls, not while one is running."""
        self.set_phrase_boosting_tables(boosting_tables(self, boosting), boosting)

    def set_phrase_boosting_tables(self, tables: Optional[PhraseBoostingTables], boosting: Optional[PhraseBoostingConfig]) -> None:
        """Upload tables already built from ``boosting`` (the multi-GPU model builds them once for all replicas).  Raises
        ValueError, changing nothing, when open streams with their own lists (``StreamingTranscriber``) could not share one
        table with the new global list."""
        for ref in list(self.__dict__.get("_boost_checks", ())):
            fn = ref()
            if fn is not None:
                fn(tables)
        self.engine.set_phrase_boosting(None if tables is None else tables.bonus, None if tables is None else tables.next)
        self.boosting, self.boosting_tables = boosting, tables
        self._notify_tables(1)

    # -- phrase boosting per utterance (phrases=)
    def phrase_setup(self, phrases: Sequence[Optional[PhraseBoostingConfig]], combined=None):
        """The combined table of ``phrases`` (one list or None per input; ``boosting.combine_tables`` with the model's global
        list in region 0) on this device -> (device tables, one root per input).  The upload is cached, keyed by the lists, so
        a repeated call does not upload again.  ``combined``: the result of ``combine_tables`` for the same lists, already built
        (the multi-GPU model builds it once for all replicas)."""
        key = phrases_key(self, phrases)
        if self._phrase_cache is None or self._phrase_cache[0] != key:
            tables, roots = combined if combined is not None else combine_tables(phrases, self.cfg.vocab_size, self.tokenizer, base=self.boosting)
            dev = tuple(torch.as_tensor(a).to(self.engine.device).contiguous() for a in (tables.bonus, tables.next))
            self._phrase_cache = (key, dev, {config_key(c): r for c, r in zip(phrases, roots) if c is not None})
        _, dev, root_of = self._phrase_cache
        return dev, [0 if c is None else root_of[config_key(c)] for c in phrases]

    @contextlib.contextmanager
    def phrase_tables_set(self, dev):
        """Decodes inside use the combined device tables ``dev`` (``phrase_setup``); afterwards the model's global setting is
        back (its tables' pointers only: nothing is uploaded) and the roots are cleared."""
        eng = self.engine
        prev = eng._boost
        eng.set_phrase_boosting(*dev)
        try:
            yield
        finally:
            eng.set_phrase_boosting(*(prev if prev is not None else (None,)))

    # -- token-level batched path
    def iter_token_batches(self, waveforms: Sequence[np.ndarray], pad: int = 0, *, phrases=None):
        """16 kHz mono waveforms (each gets ``pad`` zero samples on both sides) -> yields ``(indices, [(tokens, frames)])``
        batch by batch; with confidence on, ``(tokens, frames, stats)``, stats float32 [n_tokens, 4] (lp, H1, A_alpha, G_alpha).

        Utterances are sorted by length and cut into batches of at most ``max_batch`` so padding waste stays small.
        The engine call of batch k runs on a worker thread (ctypes drops the GIL) while this thread stages batch k+1
        into the other staging set and the caller post-processes batch k-1: on a long list the host work hides behind
        the GPU.  One engine call is in flight at a time (an engine is not re-entrant).

        ``phrases``: one ``PhraseBoostingConfig`` or None (the model's global list) per waveform; each utterance is decoded
        against its own list, exactly as it would be alone with that list set by ``set_phrase_boosting``."""
        if phrases is None:
            yield from self._token_batches(waveforms, pad, None)
            return
        phrases = check_phrases(self, phrases, len(waveforms))
        dev, roots = self.phrase_setup(phrases)
        with self.phrase_tables_set(dev):
            yield from self._token_batches(waveforms, pad, roots)

    def _token_batches(self, waveforms: Sequence[np.ndarray], pad: int, roots: Optional[List[int]]):
        """``iter_token_batches``; ``roots``: the boosting root of every waveform in the table that is set, or None."""
        from concurrent.futures import ThreadPoolExecutor
        if len(waveforms) == 0:
            return
        order = sorted(range(len(waveforms)), key=lambda i: len(waveforms[i]))
        batches = [order[lo:lo + self.max_batch] for lo in range(0, len(order), self.max_batch)]
        eng = self.engine
        eng.ensure_workspace(len(batches[0]), (len(waveforms[order[-1]]) + 2 * pad + 3) & ~3)   # once, on this thread (stage() rounds rows up to 4 samples)
        alpha = self.confidence.alpha if self.confidence is not None else None
        host_call = eng.transcribe_host if alpha is None else partial(eng.transcribe_host, alpha=alpha)

        def call(wav, lens, U, out, idx):
            if roots is not None:                                     # the batch's roots in its sorted row order, set on the thread that runs it
                eng.set_boost_roots([roots[i] for i in idx])
            return host_call(wav, lens, U, out)

        def run(staging, idx):
            wav, lens = staging.stage([waveforms[i] for i in idx], pad)
            U = eng.u_max(wav.shape[1])
            out = staging.outputs(len(idx), U) if alpha is None else staging.outputs(len(idx), U, stats=True)
            return wav, lens, out

        def collect(done, idx):
            return idx, _items(done, len(idx))

        if len(batches) == 1:                                         # nothing to overlap: skip the thread hand-off (one-clip calls)
            wav, lens, out = run(self._staging[0], batches[0])
            yield collect(call(wav, lens, out[0].shape[1], out, batches[0]), batches[0])
            return
        with ThreadPoolExecutor(max_workers=1) as pool:
            in_flight = None
            for k, idx in enumerate(batches):
                wav, lens, out = run(self._staging[k & 1], idx)
                nxt = (pool.submit(call, wav, lens, out[0].shape[1], out, idx), idx)
                if in_flight is not None:
                    yield collect(in_flight[0].result(), in_flight[1])
                in_flight = nxt
            yield collect(in_flight[0].result(), in_flight[1])

    def transcribe_tokens(self, waveforms: Sequence[np.ndarray], pad: int = 0, *, phrases=None):
        """-> [(tokens, frames)] in input order (``phrases``: as ``iter_token_batches``)."""
        results = [None] * len(waveforms)
        for idx, items in self.iter_token_batches(waveforms, pad, phrases=phrases):
            for i, item in zip(idx, items):
                results[i] = item
        return results

    def iter_token_batches_raw(self, waves: Sequence[np.ndarray], samplerate: int, pad: int = 0, *, phrases=None):
        """Like ``iter_token_batches`` for audio that still needs ``norm_audio`` (pkg/nemo-asr/src/audio.py:54-68): waveforms
        at ``samplerate`` (any rate), mono [n] or channels-first [c, n] with the SAME channel count, float or int16 PCM.  They
        are staged as they are (pinned), copied to the GPU and resampled / down-mixed / padded there (rs_resample_mono)
        straight into the buffer the engine transcribes from: the host never touches a sample arithmetically.  (scipy's
        resample_poly, which this kernel restates, costs the host ~10 ms per 30 s 48 kHz clip -- more than the whole engine.)
        ``phrases``: as ``iter_token_batches``."""
        if phrases is None:
            yield from self._token_batches_raw(waves, samplerate, pad, None)
            return
        phrases = check_phrases(self, phrases, len(waves))
        dev, roots = self.phrase_setup(phrases)
        with self.phrase_tables_set(dev):
            yield from self._token_batches_raw(waves, samplerate, pad, roots)

    def _token_batches_raw(self, waves: Sequence[np.ndarray], samplerate: int, pad: int, roots: Optional[List[int]]):
        if len(waves) == 0:
            return
        eng = self.engine
        waves = [w if w.ndim == 2 else w[None] for w in waves]
        C = waves[0].shape[0]
        if any(w.shape[0] != C for w in waves):
            raise ValueError("iter_token_batches_raw: all waveforms of a call must have the same number of channels")
        pcm = all(w.dtype == np.int16 for w in waves)
        order = sorted(range(len(waves)), key=lambda i: waves[i].shape[1])
        for lo in range(0, len(order), self.max_batch):
            idx = order[lo:lo + self.max_batch]
            L = (max(waves[i].shape[1] for i in idx) + 3) & ~3
            raw = torch.zeros(len(idx), C, L, dtype=torch.int16 if pcm else torch.float32)
            if torch.cuda.is_available():
                raw = raw.pin_memory()
            rows = raw.numpy()
            for r, i in enumerate(idx):
                w = waves[i]
                rows[r, :, : w.shape[1]] = w if (pcm or w.dtype != np.int16) else w.astype(np.float32) * np.float32(1.0 / 32768.0)
            lens = torch.tensor([waves[i].shape[1] for i in idx], dtype=torch.int32)
            if roots is not None:
                eng.set_boost_roots([roots[i] for i in idx])
            with torch.cuda.device(eng.device):
                wav, wl = eng.resample_mono(raw.to(eng.device, non_blocking=True), lens.to(eng.device, non_blocking=True), samplerate, pad)
                done = [a.cpu() for a in (eng.transcribe_device(wav, wl) if self.confidence is None else
                                          eng.transcribe_device(wav, wl, alpha=self.confidence.alpha))]
            yield idx, _items(done, len(idx))

    # -- forced alignment of known transcripts (alignment.py)
    def iter_align_batches(self, waveforms: Sequence[np.ndarray], token_lists: Sequence[Sequence[int]], pad: int = 0):
        """16 kHz mono waveforms (``pad`` zero samples on both sides) and their token-id lists -> yields ``(indices, items)``
        batch by batch, item = (frames, token_lp, viterbi, loglik) of one utterance: log-mel -> encode -> rs_rnnt_align.
        Utterances are batched by length as in ``transcribe_alsd``; any ``decoding`` works."""
        token_lists = validate_labels(token_lists, self.cfg.vocab_size, len(waveforms))
        eng = self.engine
        order = sorted(range(len(waveforms)), key=lambda i: len(waveforms[i]))
        for lo in range(0, len(order), self.max_batch):
            idx = order[lo:lo + self.max_batch]
            wav, lens = self._staging[0].stage([waveforms[i] for i in idx], pad)
            labels, label_len = pack_labels([token_lists[i] for i in idx])
            with torch.cuda.device(eng.device):
                x = wav.to(eng.device, non_blocking=True)
                if x.dtype == torch.int16:
                    x = x.to(torch.float32) * (1.0 / 32768.0)
                mel, mel_len = eng.log_mel(x, lens.to(eng.device))
                enc, enc_len = eng.encode(mel, mel_len)
                frames, token_lp, viterbi, loglik = [a.cpu() for a in eng.align(enc, enc_len, torch.from_numpy(labels).to(eng.device),
                                                                                 torch.from_numpy(label_len).to(eng.device))]
            yield idx, [(frames[r, :n].tolist(), token_lp[r, :n].tolist(), float(viterbi[r]), float(loglik[r]))
                        for r, n in enumerate(label_len.tolist())]

    def align_tokens(self, waveforms: Sequence[np.ndarray], token_lists: Sequence[Sequence[int]], pad: int = 0):
        """-> [(frames, token_lp, viterbi, loglik)] in input order (``iter_align_batches``)."""
        results = [None] * len(waveforms)
        for idx, items in self.iter_align_batches(waveforms, token_lists, pad):
            for i, item in zip(idx, items):
                results[i] = item
        return results

    # -- segment alignment of captions inside their windows (alignment.py, captions.py)
    def iter_align_segment_batches(self, waveforms: Sequence[np.ndarray], token_lists: Sequence[Sequence[int]], pad: int = 0):
        """Like ``iter_align_batches``, through rs_rnnt_align_segment: item = (s, e, frames, token_lp, frame_lp, viterbi,
        loglik) of one window, frame_lp holding frames [s, e] only; a window whose tokens could not be placed (no token, or
        no frame) has s = e = -1, empty lists and NaN scores."""
        token_lists = validate_labels(token_lists, self.cfg.vocab_size, len(waveforms))
        eng = self.engine
        order = sorted(range(len(waveforms)), key=lambda i: len(waveforms[i]))
        for lo in range(0, len(order), self.max_batch):
            idx = order[lo:lo + self.max_batch]
            wav, lens = self._staging[0].stage([waveforms[i] for i in idx], pad)
            labels, label_len = pack_labels([token_lists[i] for i in idx])
            with torch.cuda.device(eng.device):
                x = wav.to(eng.device, non_blocking=True)
                if x.dtype == torch.int16:
                    x = x.to(torch.float32) * (1.0 / 32768.0)
                mel, mel_len = eng.log_mel(x, lens.to(eng.device))
                enc, enc_len = eng.encode(mel, mel_len)
                seg, frames, token_lp, frame_lp, viterbi, loglik = [
                    a.cpu() for a in eng.align_segment(enc, enc_len, torch.from_numpy(labels).to(eng.device),
                                                       torch.from_numpy(label_len).to(eng.device))]
            items = []
            for r, n in enumerate(label_len.tolist()):
                s0, e0 = int(seg[r, 0]), int(seg[r, 1])
                n = n if s0 >= 0 else 0
                items.append((s0, e0, frames[r, :n].tolist(), token_lp[r, :n].tolist(),
                              frame_lp[r, s0:e0 + 1].tolist() if s0 >= 0 else [], float(viterbi[r]), float(loglik[r])))
            yield idx, items

    def align_segment_tokens(self, waveforms: Sequence[np.ndarray], token_lists: Sequence[Sequence[int]], pad: int = 0):
        """-> [(s, e, frames, token_lp, frame_lp, viterbi, loglik)] in input order (``iter_align_segment_batches``)."""
        results = [None] * len(waveforms)
        for idx, items in self.iter_align_segment_batches(waveforms, token_lists, pad):
            for i, item in zip(idx, items):
                results[i] = item
        return results

    # -- NeMo's call shape (transcribe.py:48-53): already padded tensors
    def transcribe_alsd(self, waveforms: Sequence[np.ndarray], pad: int = 0) -> List[Hypothesis]:
        """ALSD beam search (NeMo's align_length_sync_decoding, the strategy reazonspeech-nemo-v2 ships with): hypotheses exactly
        as NeMo hands them to the reference's decode.py -- y_sequence with the leading blank, timestamp = alignment steps."""
        eng = self.engine
        out: List[Optional[Hypothesis]] = [None] * len(waveforms)
        order = sorted(range(len(waveforms)), key=lambda i: len(waveforms[i]))
        for lo in range(0, len(order), self.max_batch):
            idx = order[lo:lo + self.max_batch]
            wav, lens = self._staging[0].stage([waveforms[i] for i in idx], pad)
            with torch.cuda.device(eng.device):
                x = wav.to(eng.device, non_blocking=True)
                if x.dtype == torch.int16:
                    x = x.to(torch.float32) * (1.0 / 32768.0)
                mel, mel_len = eng.log_mel(x, lens.to(eng.device))
                enc, enc_len = eng.encode(mel, mel_len)
                y, steps, n, score = [a.cpu() for a in eng.alsd(enc, enc_len, beam=self.beam_size)]
            for r, i in enumerate(idx):
                k = int(n[r])
                out[i] = Hypothesis(y[r, : k + 1].to(torch.long), steps[r, :k].tolist(), float(score[r]))
        return out

    def _maes(self, enc: torch.Tensor, enc_len: torch.Tensor, n_best: int):
        m = self.maes
        y, frames, n, score, count = [a.cpu() for a in self.engine.maes(enc, enc_len, beam=self.beam_size, n_best=n_best, num_steps=m.num_steps,
                                                                        prefix_alpha=m.prefix_alpha, expansion_beta=m.expansion_beta,
                                                                        expansion_gamma=m.expansion_gamma)]
        steps = frames + torch.arange(1, frames.shape[-1] + 1, dtype=frames.dtype)      # Hypothesis.from_greedy's timestamp convention
        return y, steps, n, score, count

    def transcribe_maes(self, waveforms: Sequence[np.ndarray], pad: int = 0) -> List[Hypothesis]:
        """MAES beam search (NeMo's modified_adaptive_expansion_search, fused with the n-gram LM when one is set): the best
        hypothesis of each waveform, shaped like ``transcribe_alsd``'s (timestamp[i] = frame_i + i + 1)."""
        return [hyps[0] for hyps in self.transcribe_beam_nbest(waveforms, 1, pad)]

    def transcribe_beam_nbest(self, waveforms: Sequence[np.ndarray], n_best: int, pad: int = 0,
                              log_likelihood: bool = False) -> List[List[Hypothesis]]:
        """The N-best lists of the model's beam search, ALSD or MAES by ``decoding`` (``transcribe_alsd_nbest`` runs either)."""
        return self.transcribe_alsd_nbest(waveforms, n_best, pad, log_likelihood)

    def transcribe_alsd_nbest(self, waveforms: Sequence[np.ndarray], n_best: int, pad: int = 0,
                              log_likelihood: bool = False) -> List[List[Hypothesis]]:
        """The N-best lists of ``transcribe_alsd``'s search (NeMo's return_best_hypothesis=False; with ``decoding="maes"`` MAES's
        sort_nbest of its kept hypotheses, n_best <= beam_size), best first, one list per
        waveform: at most ``n_best`` ALSD-shaped hypotheses each, ``score`` the candidate's beam score.  Entry 0 is
        ``transcribe_alsd``'s hypothesis.  ``log_likelihood``: every candidate is also force-aligned (``Engine.align``) on its
        batch's encoder output, so ``hypothesis.log_likelihood`` = log P(tokens | audio) (alignment.py), the score for
        rescoring the list; the log-mel and the encoder do not run again."""
        eng = self.engine
        out: List[Optional[List[Hypothesis]]] = [None] * len(waveforms)
        order = sorted(range(len(waveforms)), key=lambda i: len(waveforms[i]))
        for lo in range(0, len(order), self.max_batch):
            idx = order[lo:lo + self.max_batch]
            wav, lens = self._staging[0].stage([waveforms[i] for i in idx], pad)
            with torch.cuda.device(eng.device):
                x = wav.to(eng.device, non_blocking=True)
                if x.dtype == torch.int16:
                    x = x.to(torch.float32) * (1.0 / 32768.0)
                mel, mel_len = eng.log_mel(x, lens.to(eng.device))
                enc, enc_len = eng.encode(mel, mel_len)
                if self.decoding == "maes":
                    lists = nbest_hypotheses(*self._maes(enc, enc_len, n_best))
                else:
                    lists = nbest_hypotheses(*[a.cpu() for a in eng.alsd_nbest(enc, enc_len, n_best, beam=self.beam_size)][:5])
                if log_likelihood:
                    self._candidate_log_likelihoods(enc, enc_len, lists)
            for r, i in enumerate(idx):
                out[i] = lists[r]
        return out

    def _candidate_log_likelihoods(self, enc: torch.Tensor, enc_len: torch.Tensor, lists: List[List[Hypothesis]]) -> None:
        """Fills ``log_likelihood`` of every candidate of one batch: its encoder rows gathered with index_select and aligned in
        chunks of at most ``max_batch`` rows."""
        eng = self.engine
        cands = [(r, h) for r, hyps in enumerate(lists) for h in hyps]
        for lo in range(0, len(cands), self.max_batch):
            chunk = cands[lo:lo + self.max_batch]
            rows = torch.tensor([r for r, _ in chunk], dtype=torch.long, device=eng.device)
            labels, label_len = pack_labels([h.y_sequence.tolist()[1:] for _, h in chunk])
            loglik = eng.align(enc.index_select(0, rows).contiguous(), enc_len.index_select(0, rows).contiguous(),
                               torch.from_numpy(labels).to(eng.device), torch.from_numpy(label_len).to(eng.device))[3].cpu()
            for j, (_, h) in enumerate(chunk):
                h.log_likelihood = float(loglik[j])

    def transcribe(self, audio, batch_size: int = 1, return_hypotheses: bool = True, verbose: bool = True, **_):
        waves = [a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a) for a in audio]
        if self.decoding == "alsd":
            out = self.transcribe_alsd(waves)
        elif self.decoding == "maes":
            out = self.transcribe_maes(waves)
        else:
            out = [greedy_hypothesis(self, item) for item in self.transcribe_tokens(waves)]
        if return_hypotheses:
            return out
        return [self.tokenizer.ids_to_text(h.y_sequence.tolist()[1:]) for h in out]


def boosting_tables(model, boosting: Optional[PhraseBoostingConfig]) -> Optional[PhraseBoostingTables]:
    """Validated tables of ``boosting`` for ``model``'s vocabulary and tokenizer (None: boosting off)."""
    if boosting is None:
        return None
    if getattr(model, "decoding", "greedy") != "greedy":
        raise ValueError("phrase boosting is applied by the greedy decode only (not by ALSD beam search)")
    return build_tables(boosting, model.cfg.vocab_size, model.tokenizer)


def check_phrases(model, phrases, n: int) -> List[Optional[PhraseBoostingConfig]]:
    """``phrases=`` of a call with ``n`` inputs, validated: one ``PhraseBoostingConfig`` or None per input, greedy decoding."""
    if getattr(model, "decoding", "greedy") != "greedy":
        raise ValueError("phrase boosting is applied by the greedy decode only (not by ALSD beam search)")
    phrases = list(phrases)
    if len(phrases) != n:
        raise ValueError(f"phrases= has {len(phrases)} entries for {n} inputs (one PhraseBoostingConfig or None per input)")
    for c in phrases:
        if c is not None and not isinstance(c, PhraseBoostingConfig):
            raise ValueError(f"phrases= entries must be PhraseBoostingConfig or None, got {type(c).__name__}")
    return phrases


def phrases_key(model, phrases) -> tuple:
    """The identity of the combined table of ``phrases`` on ``model``: its global list and the distinct lists, in order."""
    return config_key(model.boosting), tuple(dict.fromkeys(config_key(c) for c in phrases if c is not None))


def lm_tables(model, lm: Optional[NgramLMConfig]) -> Optional[NgramLMTables]:
    """Validated tables of ``lm`` for ``model``'s vocabulary (None: fusion off)."""
    if lm is None:
        return None
    if getattr(model, "decoding", "greedy") not in ("greedy", "maes"):
        raise ValueError("n-gram LM fusion is applied by the greedy decode and MAES beam search only (not by ALSD beam search)")
    return build_lm_tables(lm, model.cfg.vocab_size)


def nbest_hypotheses(y: torch.Tensor, steps: torch.Tensor, n: torch.Tensor, score: torch.Tensor, count: torch.Tensor) -> List[List[Hypothesis]]:
    """Host outputs of ``Engine.alsd_nbest`` (y [B, N, U + 1], steps [B, N, U], n / score [B, N], count [B]) -> per utterance
    its first count[b] entries as ALSD-shaped hypotheses, best first.  An entry longer than U keeps its first U tokens, as
    ``transcribe_alsd`` does."""
    out = []
    for b in range(y.shape[0]):
        hyps = []
        for e in range(int(count[b])):
            k = int(n[b, e])
            hyps.append(Hypothesis(y[b, e, : k + 1].to(torch.long), steps[b, e, :k].tolist(), float(score[b, e])))
        out.append(hyps)
    return out


def _items(done, B: int):
    """Host outputs of one engine call -> per utterance (tokens, frames), or (tokens, frames, stats) with the statistics."""
    tokens, frames, ntok = done[:3]
    U = tokens.shape[1]
    counts = ntok.tolist()[:B]
    if len(done) == 3:
        return [(tokens[r, :n].tolist(), frames[r, :n].tolist()) for r, n in enumerate(counts)]
    stats = done[3]
    return [(tokens[r, :n].tolist(), frames[r, :n].tolist(), stats[r, : min(n, U)].numpy().copy()) for r, n in enumerate(counts)]


def _find_checkpoint() -> Optional[str]:
    env = os.environ.get(ENV_CHECKPOINT)
    if env:
        return env
    hub = os.path.expanduser(os.environ.get("HF_HOME", "~/.cache/huggingface"))
    hits = glob.glob(os.path.join(hub, "hub", "models--" + HF_REPO.replace("/", "--"), "snapshots", "*", "*.nemo"))
    return sorted(hits)[-1] if hits else None


def load_model(device=None, *, checkpoint: Optional[str] = None, synthetic: Optional[bool] = None,
               config: Optional[ModelConfig] = None, seed: int = 0, max_batch: int = 64, devices: Optional[Sequence] = None,
               decoding: str = "greedy", beam_size: int = 4, confidence: Optional[ConfidenceConfig] = None,
               boosting: Optional[PhraseBoostingConfig] = None, lm: Optional[NgramLMConfig] = None,
               maes: Optional[MaesConfig] = None):
    """Load the ReazonSpeech FastConformer-RNNT onto a B200.

    ``device``: None / "cuda" / "cuda:N" as in the reference (transcribe.py:9-22, eval.py:26).
    "cpu" raises: this engine has no CPU path.  ``decoding``: "greedy" (default: BASELINE.json's parity target) or "alsd", NeMo's
    align_length_sync_decoding beam search with ``beam_size`` -- the strategy the shipped checkpoint decodes with by default
    (pkg/nemo-asr/src/decode.py:29); it runs on the GPU too (csrc/decode_alsd.cu).  ``devices`` (e.g. ``range(8)`` or ``["cuda:0", "cuda:1"]``) loads one
    replica per listed GPU into THIS process and returns a model that deals every call's utterances across them
    (``multi_gpu.MultiGpuRnntModel``; same surface, results in input order).  Weights come from ``checkpoint`` (a .nemo file),
    $REAZONSPEECH_NEMO_CHECKPOINT or the local Hugging Face cache of reazonspeech-nemo-v2.
    With ``synthetic=True`` (or $REAZONSPEECH_B200_SYNTHETIC=1) seeded random weights of the same
    architecture are used instead -- the only option offline.  ``confidence``: a ``ConfidenceConfig`` turns on token / word
    confidence and log-probability scores of the greedy decode (``confidence.py``); not available with ``decoding="alsd"``.
    ``boosting``: a ``PhraseBoostingConfig`` boosts its key phrases in the greedy decode (``boosting.py``); change or clear
    them later with ``model.set_phrase_boosting``; not available with ``decoding="alsd"``.
    ``lm``: an ``NgramLMConfig`` fuses its ARPA n-gram LM into the greedy decode (``ngram_lm.py``); change or clear it later
    with ``model.set_ngram_lm``; not available with ``decoding="alsd"``.
    ``decoding="maes"``: NeMo's modified adaptive expansion search with ``beam_size`` (csrc/decode_maes.cu), the beam search
    the n-gram LM of ``lm`` is fused into; ``maes`` (a ``MaesConfig``) sets its parameters, by default the maes_* keys of the
    checkpoint's decoding.beam block or NeMo's defaults.  Confidence, phrase boosting and ``devices`` are greedy-only."""
    if decoding not in ("greedy", "alsd", "maes"):
        raise ValueError(f"decoding must be 'greedy', 'alsd' or 'maes', got {decoding!r}")
    if maes is not None:
        if decoding != "maes":
            raise ValueError("maes= sets the parameters of decoding='maes'")
        maes.validate()
    if confidence is not None:
        if decoding in ("alsd", "maes"):
            raise ValueError("confidence is computed by the greedy decode only (NeMo offers none for beam search)")
        confidence.validate()
    if boosting is not None:
        if decoding in ("alsd", "maes"):
            raise ValueError("phrase boosting is applied by the greedy decode only (not by beam search)")
        boosting.validate()
    if lm is not None:
        if decoding == "alsd":
            raise ValueError("n-gram LM fusion is applied by the greedy decode and MAES beam search only (not by ALSD beam search)")
        lm.validate()
    if device is None:
        device = "cuda"
    if str(device).startswith("cpu"):
        raise RuntimeError("reazonspeech_b200: device='cpu' is not supported (hand-written sm_90a kernels only)")
    if synthetic is None:
        synthetic = os.environ.get(ENV_SYNTHETIC, "") not in ("", "0")
    path = checkpoint or (None if synthetic else _find_checkpoint())
    if path is not None:
        cfg, sd, tok = load_nemo_archive(path)
        tokenizer = SentencePieceTokenizer(tok) if tok else PieceTableTokenizer(synthetic_pieces(cfg.vocab_size))
        if decoding == "greedy" and not cfg.checkpoint_decoding.startswith("greedy"):
            import warnings                 # the reference never overrides the checkpoint's strategy (transcribe.py:26-28): say what differs
            warnings.warn(f"{path}: the checkpoint is configured for '{cfg.checkpoint_decoding}' decoding; this model decodes greedily "
                          f"(transcripts can differ from the reference's default).  Pass decoding='alsd' for NeMo's ALSD beam search.", stacklevel=2)
    elif synthetic:
        cfg = config or ModelConfig()
        sd = random_state_dict(cfg, seed)
        tokenizer = PieceTableTokenizer(synthetic_pieces(cfg.vocab_size))
    else:
        raise FileNotFoundError(
            f"no .nemo checkpoint for {HF_REPO}: pass checkpoint=..., set ${ENV_CHECKPOINT}, populate the Hugging Face "
            f"cache, or request seeded synthetic weights with synthetic=True / ${ENV_SYNTHETIC}=1")
    if decoding == "maes":
        maes = (maes or cfg.checkpoint_maes or MaesConfig()).check_beam(beam_size, cfg.vocab_size)
    if devices is None:
        return B200RnntModel(Engine(cfg, sd, str(device), alsd=decoding in ("alsd", "maes")), tokenizer, max_batch=max_batch, decoding=decoding,
                             beam_size=beam_size, confidence=confidence, boosting=boosting, lm=lm, maes=maes)
    if decoding != "greedy":
        raise ValueError("the one-process multi-GPU model decodes greedily; load one model per device for beam search")
    names = [d if isinstance(d, str) else f"cuda:{int(d)}" for d in devices]
    if len(names) == 0 or len(set(names)) != len(names):
        raise ValueError(f"devices must name distinct GPUs, got {list(devices)!r}")
    from ...engine import pack_weights
    from .multi_gpu import MultiGpuRnntModel
    packed = pack_weights(sd, cfg)                                   # repacked once, uploaded once per device
    model = MultiGpuRnntModel([B200RnntModel(Engine(cfg, None, n, packed=packed), tokenizer, max_batch=max_batch, confidence=confidence)
                               for n in names])
    if boosting is not None:
        model.set_phrase_boosting(boosting)
    if lm is not None:
        model.set_ngram_lm(lm)
    return model


def _prepare(audio: AudioData) -> np.ndarray:
    wave = pad_audio(norm_audio(audio), PAD_SECONDS).waveform
    return wave if wave.dtype == np.int16 else wave.astype(np.float32, copy=False)     # int16 = PCM, scaled on the device


def transcribe(model, audio: AudioData, config: Optional[TranscribeConfig] = None) -> TranscribeResult:
    """One utterance, same contract as the reference (transcribe.py:30-60)."""
    if config is None:
        config = TranscribeConfig()
    wave = torch.from_numpy(_prepare(audio))
    hyp = model.transcribe([wave], batch_size=1, return_hypotheses=True, verbose=config.verbose)[0]
    result = decode_hypothesis(model, hyp)
    if config.raw_hypothesis:
        result.hypothesis = hyp
    return result


def transcribe_batch(model, audios: Sequence[AudioData], config: Optional[TranscribeConfig] = None, *,
                     phrases: Optional[Sequence[Optional[PhraseBoostingConfig]]] = None) -> List[TranscribeResult]:
    """Many utterances through one or a few engine launches; results in input order.

    Same per-utterance semantics as ``transcribe`` (norm_audio, 0.5 s of silence on both sides, greedy decode,
    decode_hypothesis); the padding is written straight into the staging buffer and the post-processing of one batch
    overlaps the engine call of the next.  A model object without ``iter_token_batches`` (e.g. a real NeMo model)
    is driven through its ``transcribe`` method instead.

    ``phrases``: one ``PhraseBoostingConfig`` or None (the model's global list) per audio: utterances with different key
    phrases share the batches, each decoded against its own list (greedy decoding only)."""
    if config is None:
        config = TranscribeConfig()
    if phrases is not None:
        phrases = check_phrases(model, phrases, len(audios))
        if not hasattr(model, "iter_token_batches"):
            raise ValueError("phrases= needs a model of this package (load_model)")
    out: List[Optional[TranscribeResult]] = [None] * len(audios)

    def finish(i, hyp):
        r = decode_hypothesis(model, hyp)
        if config.raw_hypothesis:
            r.hypothesis = hyp
        out[i] = r

    if hasattr(model, "iter_token_batches") and getattr(model, "decoding", "greedy") == "greedy":
        pad = int(PAD_SECONDS * SAMPLERATE)
        # audio that still needs norm_audio (another rate, several channels) and is uniform in both goes to the GPU as it is:
        # resampling, down-mixing and padding run there (iter_token_batches_raw); anything else is normalised on the host
        raw_ok = (hasattr(model, "iter_token_batches_raw") and len(audios) > 0 and
                  len({(a.samplerate, np.asarray(a.waveform).ndim, np.asarray(a.waveform).shape[0] if np.asarray(a.waveform).ndim == 2 else 1)
                       for a in audios}) == 1 and
                  (audios[0].samplerate != SAMPLERATE or np.asarray(audios[0].waveform).ndim == 2))
        if raw_ok:
            batches = model.iter_token_batches_raw([np.asarray(a.waveform) for a in audios], audios[0].samplerate, pad=pad, phrases=phrases)
        else:
            batches = model.iter_token_batches([np.asarray(norm_audio(a).waveform) for a in audios], pad=pad, phrases=phrases)
        for idx, items in batches:
            for i, item in zip(idx, items):
                finish(i, greedy_hypothesis(model, item))
    else:
        tensors = [torch.from_numpy(_prepare(a)) for a in audios]
        hyps = model.transcribe(tensors, batch_size=max(len(tensors), 1), return_hypotheses=True, verbose=config.verbose)
        for i, hyp in enumerate(hyps):
            finish(i, hyp)
    return out


def transcribe_nbest_batch(model, audios: Sequence[AudioData], n_best: int, config: Optional[TranscribeConfig] = None, *,
                           log_likelihood: bool = False) -> List[List[TranscribeResult]]:
    """The N-best lists of ALSD beam search (NeMo's BeamRNNTInfer with return_best_hypothesis=False), in input order: for each
    audio at most ``n_best`` results, best first (ranked by score / len(y) as NeMo ranks its finished hypotheses); entry 0 is
    what ``transcribe_batch`` returns.  The audio is prepared as ``transcribe`` prepares it, and every result comes from the
    unchanged ``decode_hypothesis``.  ``result.hypothesis`` always carries the candidate: score = its beam score and, with
    ``log_likelihood=True``, log_likelihood = log P(tokens | audio) from forced alignment (alignment.py), the usual score
    for rescoring the list.  Needs a single-GPU model loaded with ``decoding="alsd"`` or ``"maes"``; that, or ``n_best``
    outside 1..64 (MAES: 1..beam_size), raises ValueError before the GPU is touched."""
    if getattr(model, "decoding", "greedy") not in ("alsd", "maes") or not hasattr(model, "transcribe_alsd_nbest"):
        raise ValueError("N-best lists come from beam search on one GPU: use load_model(decoding=\"alsd\" or \"maes\") without devices=")
    if isinstance(n_best, bool) or not isinstance(n_best, (int, np.integer)) or not 1 <= int(n_best) <= MAX_NBEST:
        raise ValueError(f"n_best must be an integer in 1..{MAX_NBEST}, got {n_best!r}")
    if model.decoding == "maes" and int(n_best) > model.beam_size:
        raise ValueError(f"MAES keeps beam_size = {model.beam_size} hypotheses: n_best must be in 1..{model.beam_size}, got {n_best!r}")
    waves = [_prepare(a) for a in audios]
    out: List[List[TranscribeResult]] = []
    for hyps in model.transcribe_alsd_nbest(waves, int(n_best), log_likelihood=log_likelihood):
        results = []
        for hyp in hyps:
            r = decode_hypothesis(model, hyp)
            r.hypothesis = hyp
            results.append(r)
        out.append(results)
    return out


def transcribe_nbest(model, audio: AudioData, n_best: int, config: Optional[TranscribeConfig] = None, *,
                     log_likelihood: bool = False) -> List[TranscribeResult]:
    """One utterance of ``transcribe_nbest_batch``."""
    return transcribe_nbest_batch(model, [audio], n_best, config, log_likelihood=log_likelihood)[0]


def _target_ids(model, text) -> List[int]:
    """A transcript as token ids: a str is encoded like the model's training targets (``sentence_to_ids``), a sequence of
    ints is taken as it is."""
    return model.tokenizer.sentence_to_ids(text) if isinstance(text, str) else [int(k) for k in text]


def align_batch(model, audios: Sequence[AudioData], texts: Sequence, config: Optional[TranscribeConfig] = None) -> List[TranscribeResult]:
    """Forced alignment of known transcripts (alignment.py): ``texts[i]`` (a str, or a sequence of token ids) against
    ``audios[i]``, results in input order.  The audio is prepared as ``transcribe`` prepares it (norm_audio, 0.5 s of silence
    on both sides), and each result comes from the unchanged ``decode_hypothesis``: subwords are the given tokens, timed at
    their Viterbi emission frames exactly as a transcription's tokens are.  ``result.hypothesis`` always carries the
    alignment: score = the Viterbi path's log-probability, log_likelihood = log P(text | audio), token_logprob per token.
    Bad token ids or a count mismatch raise ValueError before the GPU is touched."""
    if config is None:
        config = TranscribeConfig()
    if len(texts) != len(audios):
        raise ValueError(f"{len(texts)} transcripts for {len(audios)} audio inputs")
    ids = validate_labels([_target_ids(model, t) for t in texts], model.cfg.vocab_size, len(audios))
    pad = int(PAD_SECONDS * SAMPLERATE)
    waves = [np.asarray(norm_audio(a).waveform) for a in audios]
    out: List[TranscribeResult] = []
    for k, (frames, token_lp, viterbi, loglik) in zip(ids, model.align_tokens(waves, ids, pad=pad)):
        hyp = alignment_hypothesis(k, frames, token_lp, viterbi, loglik, model.cfg.blank)
        result = decode_hypothesis(model, hyp)
        result.hypothesis = hyp
        out.append(result)
    return out


def align(model, audio: AudioData, text, config: Optional[TranscribeConfig] = None) -> TranscribeResult:
    """One utterance of ``align_batch``."""
    return align_batch(model, [audio], [text], config)[0]


def align_captions(model, audio: AudioData, captions: Sequence[Caption], *, before: float = BEFORE_SECONDS,
                   after: float = AFTER_SECONDS, confidence_frames: int = CONFIDENCE_FRAMES,
                   transcribe: bool = False) -> List[Optional[AlignedCaption]]:
    """Locate each caption of a long recording inside its audio window (captions.py): one ``AlignedCaption`` or None per
    caption, in input order.  The windows [start - before, end + after) are cut from ``audio`` after norm_audio, prepared
    as ``align_batch`` prepares an audio, batched by length and aligned on the GPU with the segment alignment of
    alignment.py.  A caption whose window is empty (it lies outside the audio), whose text has no token, or whose window
    has no encoder frame gets None.  The caption's text is tokenised with ``sentence_to_ids``.  Subwords and the segment
    are in program seconds.  ``transcribe=True`` transcribes every located segment in one ``transcribe_batch`` call and
    fills ``asr`` and ``cer`` (evaluation.utils.calculate_cer against the caption), the reference's corpus filter.
    A caption that ends before it starts raises ValueError before the GPU is touched."""
    from ...captions import confidence, segment_seconds, window_samples
    wave = np.asarray(norm_audio(audio).waveform)
    duration = len(wave) / SAMPLERATE
    windows = [caption_window(c, duration, before, after) for c in captions]
    jobs = []                                                   # (caption index, window, token ids)
    for k, (c, w) in enumerate(zip(captions, windows)):
        ids = model.tokenizer.sentence_to_ids(c.text) if w is not None else []
        if ids:
            jobs.append((k, w, ids))
    validate_labels([ids for _, _, ids in jobs], model.cfg.vocab_size, len(jobs))
    waves = []
    for _, (w0, w1), _ in jobs:
        lo, hi = window_samples(w0, w1, SAMPLERATE)
        waves.append(wave[lo:hi])
    out: List[Optional[AlignedCaption]] = [None] * len(captions)
    items = model.align_segment_tokens(waves, [ids for _, _, ids in jobs], pad=int(PAD_SECONDS * SAMPLERATE)) if jobs else []
    for (k, (w0, w1), ids), (s0, e0, frames, token_lp, frame_lp, viterbi, loglik) in zip(jobs, items):
        if s0 < 0:
            continue
        r = decode_hypothesis(model, alignment_hypothesis(ids, frames, token_lp, viterbi, loglik, model.cfg.blank))
        start, end = segment_seconds(s0, e0, w0, w1)
        out[k] = AlignedCaption(captions[k], start, end, captions[k].text,
                                [dataclasses.replace(sw, seconds=sw.seconds + w0) for sw in r.subwords],
                                float(viterbi), float(loglik), confidence(frame_lp, confidence_frames))
    if transcribe:
        found = [a for a in out if a is not None]
        spans = [AudioData(wave[slice(*window_samples(a.start_seconds, a.end_seconds, SAMPLERATE))], SAMPLERATE) for a in found]
        for a, r in zip(found, transcribe_batch(model, spans, TranscribeConfig(verbose=False)) if spans else []):
            a.asr = r.text
            a.cer = calculate_cer(a.text, r.text)["cer"] if normalize(a.text) else math.nan
    return out
