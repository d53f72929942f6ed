"""Drop-in for ``reazonspeech.evaluation`` (pkg/evaluation/src/__init__.py:1-3) plus the H100 evaluator."""
from .base import BaseEvaluator, EvaluationResult, EvaluationResultBatch, NemoB200Evaluator
from .utils import calculate_cer, normalize

__all__ = ["BaseEvaluator", "EvaluationResult", "EvaluationResultBatch", "NemoB200Evaluator", "calculate_cer", "normalize"]
