"""Drop-in for ``reazonspeech.nemo.asr`` (pkg/nemo-asr/src/__init__.py:1-3) plus ``transcribe_batch``, the forced alignment
of known transcripts, ``align`` / ``align_batch``, and live streams, ``StreamingTranscriber``."""
from .interface import TranscribeConfig
from .transcribe import align, align_batch, transcribe, transcribe_batch, load_model
from .audio import audio_from_numpy, audio_from_tensor, audio_from_path
from .streaming import StreamingTranscriber
from ...streaming import StreamingConfig

__all__ = ["TranscribeConfig", "transcribe", "transcribe_batch", "align", "align_batch", "load_model",
           "audio_from_numpy", "audio_from_tensor", "audio_from_path", "StreamingTranscriber", "StreamingConfig"]
