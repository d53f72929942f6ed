"""Drop-in for ``reazonspeech.nemo.asr`` (pkg/nemo-asr/src/__init__.py:1-3) plus ``transcribe_batch``, the forced alignment
of known transcripts, ``align`` / ``align_batch``, ALSD N-best lists, ``transcribe_nbest`` / ``transcribe_nbest_batch``, live
streams, ``StreamingTranscriber``, caption alignment, ``align_captions``, and keyword spotting, ``find_keywords`` /
``find_keywords_batch``, and long-form alignment of a whole transcript, ``align_long`` / ``align_long_batch``."""
from .interface import TranscribeConfig
from .transcribe import align, align_batch, align_long, align_long_batch, align_captions, find_keywords, find_keywords_batch, transcribe, transcribe_batch, transcribe_nbest, transcribe_nbest_batch, load_model
from .audio import audio_from_numpy, audio_from_tensor, audio_from_path
from .streaming import StreamingTranscriber
from ...streaming import StreamingConfig
from ...captions import AlignedCaption, Caption
from ...keywords import KeywordHit

__all__ = ["TranscribeConfig", "transcribe", "transcribe_batch", "align", "align_batch", "transcribe_nbest", "transcribe_nbest_batch", "load_model",
           "audio_from_numpy", "audio_from_tensor", "audio_from_path", "StreamingTranscriber", "StreamingConfig",
           "align_captions", "Caption", "AlignedCaption", "find_keywords", "find_keywords_batch", "KeywordHit",
           "align_long", "align_long_batch"]
