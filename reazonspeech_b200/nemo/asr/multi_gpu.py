"""One process, several B200s: the same model object surface as ``B200RnntModel`` over one engine replica per device.

north_star: "utterance batches shard embarrassingly across the 8 GPUs of one box (no NCCL on the hot path)".  The
reference's only scale-out is one spawned process per GPU, each with its own model, merged through files
(pkg/evaluation/src/base.py:194-212, examples/rs-nemo/eval.py:19-27).  Here ``load_model(devices=[0, 1, ...])`` keeps
everything in one process: a full weight replica, a worker thread and a pinned staging pair per device; the utterances of
a call are dealt to the devices by length (``sharding.shard_indices``: longest first to the least-loaded device), every
replica runs its own batched pipeline (staging of batch k+1 overlaps the engine call of batch k), results are merged by
utterance index, so the output order is the input order whatever the devices' relative speed.  No collective, no
peer-to-peer traffic: an utterance never leaves its device.  The engine's C calls select their device themselves
(cudaSetDevice per call, per thread) and ctypes drops the GIL while they run, so the replicas run concurrently.
"""
from __future__ import annotations

import contextlib
import queue
import threading
from typing import List, Sequence

import numpy as np

from ...sharding import shard_indices


class MultiGpuRnntModel:
    """``replicas``: ``B200RnntModel`` objects, one per device, same weights.  Duck-typed like a single replica:
    ``iter_token_batches`` / ``transcribe_tokens`` / ``transcribe`` / ``align_tokens`` / ``tokenizer`` / ``cfg``."""

    def __init__(self, replicas: Sequence):
        if len(replicas) == 0:
            raise ValueError("MultiGpuRnntModel needs at least one replica")
        self.replicas = list(replicas)
        self.cfg = self.replicas[0].cfg
        self.tokenizer = self.replicas[0].tokenizer
        self.max_batch = self.replicas[0].max_batch
        self.confidence = getattr(self.replicas[0], "confidence", None)
        self.boosting = getattr(self.replicas[0], "boosting", None)
        self.lm = getattr(self.replicas[0], "lm", None)

    def set_ngram_lm(self, lm) -> None:
        """``B200RnntModel.set_ngram_lm`` on every replica: the tables are built once and uploaded once per device."""
        from .transcribe import lm_tables
        tables = lm_tables(self, lm)
        for r in self.replicas:
            r.set_ngram_lm_tables(tables, lm)
        self.lm = lm

    def set_phrase_boosting(self, boosting) -> None:
        """``B200RnntModel.set_phrase_boosting`` on every replica: the tables are built once and uploaded once per device."""
        from .transcribe import boosting_tables
        tables = boosting_tables(self, boosting)
        for r in self.replicas:
            r.set_phrase_boosting_tables(tables, boosting)
        self.boosting = boosting

    @property
    def devices(self) -> List[str]:
        return [str(r.engine.device) for r in self.replicas]

    def _deal(self, waveforms: Sequence[np.ndarray], batches):
        """Deals the utterances across the replicas by length and yields ``(indices into waveforms, items)`` per finished
        engine batch of any device; ``batches(replica, mine)`` runs on the replica's worker thread and yields the replica's
        ``(indices into mine, items)``.  A caller that stops early (closes the generator) waits for every replica to finish
        its engine batch in flight: the replicas' engines are idle when this generator has ended."""
        if len(waveforms) == 0:
            return
        shards = [s for s in shard_indices([len(w) for w in waveforms], len(self.replicas))]
        out: "queue.Queue" = queue.Queue()
        stop = threading.Event()

        def work(replica, mine: List[int]):
            try:
                with contextlib.closing(batches(replica, mine)) as it:      # closing waits for the batch in flight
                    for idx, items in it:
                        out.put(([mine[j] for j in idx], items))
                        if stop.is_set():
                            break
            except BaseException as exc:          # surfaced on the caller's thread: a dead device must not look like a slow one
                out.put(exc)
            finally:
                out.put(None)

        threads = [threading.Thread(target=work, args=(r, s), daemon=True) for r, s in zip(self.replicas, shards) if s]
        for t in threads:
            t.start()
        running, error = len(threads), None
        try:
            while running:
                item = out.get()
                if item is None:
                    running -= 1
                elif isinstance(item, BaseException):
                    error = error or item
                elif error is None:
                    yield item
        finally:
            stop.set()
            for t in threads:
                t.join()
        if error is not None:
            raise error

    def iter_token_batches(self, waveforms: Sequence[np.ndarray], pad: int = 0, *, phrases=None):
        """Yields ``(indices, [(tokens, frames)])`` per finished engine batch of any device, indices into ``waveforms``
        (``(tokens, frames, stats)`` items with confidence on, as ``B200RnntModel.iter_token_batches``).  ``phrases``: one
        list or None per waveform, as there; the combined table is built once and uploaded once per device, and each replica
        sets the roots of its own batches."""
        if phrases is None:
            return self._deal(waveforms, lambda replica, mine: replica.iter_token_batches([waveforms[i] for i in mine], pad))
        return self._phrase_batches(waveforms, pad, phrases)

    def _phrase_batches(self, waveforms, pad, phrases):
        from ...boosting import combine_tables
        from .transcribe import check_phrases, phrases_key
        phrases = check_phrases(self, phrases, len(waveforms))
        key, combined = phrases_key(self, phrases), None
        if any(r._phrase_cache is None or r._phrase_cache[0] != key for r in self.replicas):
            combined = combine_tables(phrases, self.cfg.vocab_size, self.tokenizer, base=self.boosting)
        setups = [r.phrase_setup(phrases, combined) for r in self.replicas]
        roots = setups[0][1]                                  # the same table on every device
        with contextlib.ExitStack() as stack:
            for r, (dev, _) in zip(self.replicas, setups):
                stack.enter_context(r.phrase_tables_set(dev))
            yield from self._deal(waveforms, lambda replica, mine: replica._token_batches([waveforms[i] for i in mine], pad,
                                                                                          [roots[i] for i in mine]))

    def align_tokens(self, waveforms: Sequence[np.ndarray], token_lists: Sequence[Sequence[int]], pad: int = 0):
        """``B200RnntModel.align_tokens`` over all devices -> [(frames, token_lp, viterbi, loglik)] in input order."""
        from ...alignment import validate_labels
        token_lists = validate_labels(token_lists, self.cfg.vocab_size, len(waveforms))
        results = [None] * len(waveforms)
        batches = self._deal(waveforms, lambda replica, mine: replica.iter_align_batches([waveforms[i] for i in mine],
                                                                                          [token_lists[i] for i in mine], pad))
        for idx, items in batches:
            for i, item in zip(idx, items):
                results[i] = item
        return results

    def transcribe_tokens(self, waveforms: Sequence[np.ndarray], pad: int = 0, *, phrases=None):
        """-> [(tokens, frames)] in input order."""
        results = [None] * len(waveforms)
        for idx, items in self.iter_token_batches(waveforms, pad, phrases=phrases):
            for i, item in zip(idx, items):
                results[i] = item
        return results

    def transcribe(self, audio, batch_size: int = 1, return_hypotheses: bool = True, verbose: bool = True, **_):
        """NeMo's call shape (pkg/nemo-asr/src/transcribe.py:48-53) over all devices."""
        import torch
        from .transcribe import greedy_hypothesis
        waves = [a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a) for a in audio]
        hyps = [greedy_hypothesis(self, item) for item in self.transcribe_tokens(waves)]
        if return_hypotheses:
            return hyps
        return [self.tokenizer.ids_to_text(h.y_sequence.tolist()[1:]) for h in hyps]
