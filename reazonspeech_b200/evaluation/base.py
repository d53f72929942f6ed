"""Evaluator with the reference's surface (pkg/evaluation/src/base.py:38-303: ``BaseEvaluator`` with
``evaluate`` / ``calculate_cer`` / ``_evaluate`` / ``_evaluate_batch``, ``EvaluationResult``,
``EvaluationResultBatch``) plus the piece every reference evaluator leaves out: a working batched path.
``NemoB200Evaluator._evaluate_batch`` (the hook pkg/evaluation/examples/rs-nemo/eval.py:31-32 raises
NotImplementedError for) feeds whole batches to ``transcribe_batch``; with ``num_gpus`` > 1 the utterances
are sharded across one spawned process per GPU (device ``cuda:{rank % num_gpus}`` like eval.py:26), no
collective on the data path.

Differences from the reference, on purpose: rows are plain dicts (a ``datasets.Dataset`` is accepted and
returned when that package is importable, but it is not required), and the batched map really is batched
-- the reference passes ``batch_size`` to ``Dataset.map`` without ``batched=True`` (base.py:205-212)."""
from __future__ import annotations

import json
import os
from abc import ABC, abstractmethod
from typing import Any, Callable, Iterable, List, Optional, TypedDict

from .utils import CERResult, calculate_cer


class EvaluationResult(TypedDict):
    prediction: str


class EvaluationResultBatch(TypedDict):
    predictions: List[str]


def _rows(dataset) -> List[dict]:
    if dataset is None:
        raise ValueError("No dataset provided and self.dataset is None.")
    if isinstance(dataset, dict):                       # column dict, like Dataset.from_dict
        keys = list(dataset)
        return [dict(zip(keys, vals)) for vals in zip(*(dataset[k] for k in keys))]
    if callable(dataset):
        return [dict(r) for r in dataset()]
    if isinstance(dataset, (str, os.PathLike)):
        path = os.fspath(dataset)
        if not os.path.isfile(path) or not path.endswith((".json", ".jsonl")):
            raise ValueError(f"Invalid dataset path: {dataset}")
        with open(path) as f:
            return [json.loads(line) for line in f if line.strip()]
    return [dict(r) for r in dataset]                   # list of dicts or datasets.Dataset


class BaseEvaluator(ABC):
    def __init__(self, model=None, processor=None, dataset=None, output_file: Optional[os.PathLike] = None,
                 batch_size: Optional[int] = None, num_proc: Optional[int] = None, num_gpus: Optional[int] = None,
                 text_column: str = "text"):
        self.model = model
        self.processor = processor
        self.output_file = output_file
        self.batch_size = batch_size
        self.num_proc = num_proc
        self.num_gpus = num_gpus
        self.text_column = text_column
        self.dataset = _rows(dataset) if dataset is not None else None

    def _calculate_cer(self, example: dict, text_column: str) -> CERResult:
        return calculate_cer(example[text_column], example["prediction"])

    def _predict(self, rows: List[dict], batch_size: Optional[int], rank: Optional[int], num_gpus: Optional[int]) -> List[str]:
        kw = {"rank": rank, "num_gpus": num_gpus}
        if batch_size is None:
            return [self._evaluate(r, **kw)["prediction"] for r in rows]
        out: List[str] = []
        for lo in range(0, len(rows), batch_size):
            chunk = rows[lo:lo + batch_size]
            batch = {k: [r[k] for r in chunk] for k in chunk[0]}
            out.extend(self._evaluate_batch(batch, **kw)["predictions"])
        return out

    def evaluate(self, dataset=None, batch_size: Optional[int] = None, num_proc: Optional[int] = None,
                 num_gpus: Optional[int] = None, text_column: Optional[str] = None,
                 output_file: Optional[os.PathLike] = None):
        """Transcribe every row, add ``prediction`` / ``distance`` / ``length`` / ``cer``, print ``CER: x.xx%``
        (same report line as base.py:223-225), optionally write JSON lines, return the rows."""
        rows = _rows(dataset) if dataset is not None else self.dataset
        if rows is None:
            raise ValueError("No dataset provided and self.dataset is None.")
        batch_size = batch_size or self.batch_size
        num_gpus = num_gpus or self.num_gpus
        text_column = text_column or self.text_column
        output_file = output_file or self.output_file
        if num_gpus is not None and num_gpus > 1:
            preds = _predict_multi_gpu(self, rows, batch_size, num_gpus)
        else:
            preds = self._predict(rows, batch_size, None, None)
        evaluated = []
        for row, pred in zip(rows, preds):
            row = dict(row, prediction=pred)
            row.update(self._calculate_cer(row, text_column))
            evaluated.append(row)
        dist = sum(r["distance"] for r in evaluated)
        length = sum(r["length"] for r in evaluated)
        print(f"CER: {dist / length * 100:.2f}%")
        if output_file is not None:
            with open(output_file, "w") as f:
                for r in evaluated:
                    f.write(json.dumps({k: v for k, v in r.items() if _jsonable(v)}, ensure_ascii=False) + "\n")
        return evaluated

    def calculate_cer(self, dataset, text_column: Optional[str] = None, num_proc: Optional[int] = None) -> float:
        text_column = text_column or self.text_column
        scored = [self._calculate_cer(r, text_column) for r in _rows(dataset)]
        return sum(s["distance"] for s in scored) / sum(s["length"] for s in scored)

    @abstractmethod
    def _evaluate(self, example: dict, *args, **kwargs) -> EvaluationResult:
        raise NotImplementedError("Subclasses must implement _evaluate method")

    @abstractmethod
    def _evaluate_batch(self, batch: dict, *args, **kwargs) -> EvaluationResultBatch:
        raise NotImplementedError("Subclasses must implement _evaluate_batch method")


def _jsonable(v) -> bool:
    try:
        json.dumps(v)
        return True
    except TypeError:
        return False


def _gpu_worker(rank: int, evaluator: "BaseEvaluator", rows: List[dict], shards: List[List[int]], batch_size, num_gpus: int, queue):
    try:
        mine = shards[rank]
        preds = evaluator._predict([rows[i] for i in mine], batch_size, rank, num_gpus)
        queue.put((rank, dict(zip(mine, preds)), None))
    except BaseException as exc:                          # the parent re-raises: a dead worker must not look like a slow one
        import traceback
        queue.put((rank, None, f"{type(exc).__name__}: {exc}\n{traceback.format_exc()}"))


def _predict_multi_gpu(evaluator: "BaseEvaluator", rows: List[dict], batch_size, num_gpus: int, poll_s: float = 1.0) -> List[str]:
    """One spawned process per GPU, utterances dealt by length (reazonspeech_b200.sharding); results return through
    a queue and are put back in input order.  A worker that raises (missing checkpoint, out of memory, unreadable audio)
    or dies without a word makes the call raise -- like ``datasets.map(num_proc=...)`` in the reference (base.py:198-204)
    -- and the remaining workers are terminated.  The caller's ``evaluator.model`` is left as it was."""
    import copy
    import queue as queue_mod
    import torch.multiprocessing as mp
    from ..sharding import shard_indices
    lengths = [evaluator._length_of(r) for r in rows]
    shards = shard_indices(lengths, num_gpus)
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    worker_eval = copy.copy(evaluator)                    # shallow: each worker loads its own replica on its own device,
    worker_eval.model = None                              # the caller keeps the model it passed in
    procs = [ctx.Process(target=_gpu_worker, args=(r, worker_eval, rows, shards, batch_size, num_gpus, queue)) for r in range(num_gpus)]
    for p in procs:
        p.start()
    merged, done, error = {}, set(), None
    try:
        while len(done) < len(procs) and error is None:
            try:
                rank, part, err = queue.get(timeout=poll_s)
            except queue_mod.Empty:
                dead = [r for r, p in enumerate(procs) if r not in done and p.exitcode is not None]
                if dead:                                  # exited without reporting (killed, segfault, CUDA abort)
                    try:                                  # its message may still be in flight
                        rank, part, err = queue.get(timeout=poll_s)
                    except queue_mod.Empty:
                        error = f"evaluation worker {dead[0]} exited with code {procs[dead[0]].exitcode} without a result"
                        break
                else:
                    continue
            if err is not None:
                error = f"evaluation worker {rank} failed: {err}"
                break
            merged.update(part)
            done.add(rank)
    finally:
        for p in procs:
            if error is not None and p.is_alive():
                p.terminate()
            p.join()
    if error is not None:
        raise RuntimeError(error)
    return [merged[i] for i in range(len(rows))]


class NemoB200Evaluator(BaseEvaluator):
    """The reference's RSNemoEvaluator (examples/rs-nemo/eval.py:15-32) on the H100 engine, with the batch hook
    implemented.  Rows carry ``{"audio": {"path": ...}}`` (datasets' undecoded Audio feature, eval.py:29) or
    ``{"audio": {"array": ..., "sampling_rate": ...}}``.

    ``evaluate(..., batch_size=N)`` hands N rows at a time to ``transcribe_batch``, which cuts them into engine batches
    of at most ``max_batch`` (64) and overlaps staging, the engine call and the post-processing of consecutive engine
    batches: a ``batch_size`` of a few hundred keeps the GPU busy, a ``batch_size`` <= 64 runs one engine call at a time."""

    def __init__(self, load_model_kwargs: Optional[dict] = None, **kwargs):
        super().__init__(**kwargs)
        self.load_model_kwargs = load_model_kwargs or {}

    def _ensure_model(self, rank, num_gpus):
        if self.model is None:
            from ..nemo.asr import load_model
            rank = 0 if rank is None else rank
            num_gpus = 1 if num_gpus is None else num_gpus
            self.model = load_model(device=f"cuda:{rank % num_gpus}", **self.load_model_kwargs)

    @staticmethod
    def _audio_of(example: dict):
        from ..nemo.asr import audio_from_numpy, audio_from_path
        a = example["audio"]
        if isinstance(a, dict) and a.get("array") is not None:
            return audio_from_numpy(a["array"], a["sampling_rate"])
        return audio_from_path(a["path"] if isinstance(a, dict) else a)

    def _length_of(self, example: dict) -> int:
        a = example["audio"]
        if isinstance(a, dict) and a.get("array") is not None:
            return len(a["array"])
        path = a["path"] if isinstance(a, dict) else a
        return os.path.getsize(path)

    def _evaluate(self, example, rank: Optional[int] = None, num_gpus: Optional[int] = None, **kwargs) -> EvaluationResult:
        from ..nemo.asr import TranscribeConfig, transcribe
        self._ensure_model(rank, num_gpus)
        return {"prediction": transcribe(self.model, self._audio_of(example), TranscribeConfig(verbose=False)).text}

    def _evaluate_batch(self, batch, rank: Optional[int] = None, num_gpus: Optional[int] = None, **kwargs) -> EvaluationResultBatch:
        from ..nemo.asr import TranscribeConfig, transcribe_batch
        self._ensure_model(rank, num_gpus)
        audios = [self._audio_of({"audio": a}) for a in batch["audio"]]
        results = transcribe_batch(self.model, audios, TranscribeConfig(verbose=False))
        return {"predictions": [r.text for r in results]}
