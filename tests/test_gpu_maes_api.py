"""MAES through the package's model surface: load_model(decoding="maes"), transcribe_batch, transcribe_nbest_batch with
log_likelihood, the LM set at load time and cleared later, and the greedy-only options refused."""
import numpy as np
import pytest

from ngram_oracle import write_arpa
from reazonspeech_b200.synth import synth_clip

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def audios():
    from reazonspeech_b200.nemo import asr
    return [asr.audio_from_numpy(synth_clip(400 + i, s), 16000) for i, s in enumerate((2.0, 0.8, 3.3, 1.5))]


def test_maes_model_transcribes_and_ranks(tiny_cfg, audios, tmp_path):
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.ngram_lm import NgramLMConfig
    model = asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=3, decoding="maes", beam_size=4)
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    best = asr.transcribe_batch(model, audios, cfg)
    lists = asr.transcribe_nbest_batch(model, audios, 4, log_likelihood=True)
    for ref, rs in zip(best, lists):
        assert 1 <= len(rs) <= 4
        h = rs[0].hypothesis
        assert rs[0].text == ref.text and h.y_sequence.tolist() == ref.hypothesis.y_sequence.tolist() and h.score == ref.hypothesis.score
        assert h.y_sequence[0].item() == tiny_cfg.blank
        frames = [s - i - 1 for i, s in enumerate(h.timestamp)]             # decode.py's step - idx - 1
        assert frames == sorted(frames) and all(f >= 0 for f in frames)
        keys = [r.hypothesis.score / len(r.hypothesis.y_sequence) for r in rs]
        assert keys == sorted(keys, reverse=True)
        assert all(r.hypothesis.log_likelihood is not None and np.isfinite(r.hypothesis.log_likelihood) for r in rs)
    with pytest.raises(ValueError, match="n_best"):
        asr.transcribe_nbest_batch(model, audios, 5)
    path = str(tmp_path / "lm3.arpa")
    write_arpa(path, tiny_cfg.vocab_size, 3, n_sentences=200, seed=7)
    model.set_ngram_lm(NgramLMConfig(path, 0.5))
    fused = asr.transcribe_batch(model, audios, cfg)
    model.set_ngram_lm(None)
    again = asr.transcribe_batch(model, audios, cfg)
    assert [r.hypothesis.y_sequence.tolist() for r in again] == [r.hypothesis.y_sequence.tolist() for r in best]
    assert [r.hypothesis.score for r in again] == [r.hypothesis.score for r in best]
    assert any(f.hypothesis.score != b.hypothesis.score for f, b in zip(fused, best))
    from reazonspeech_b200.boosting import PhraseBoostingConfig
    with pytest.raises(ValueError, match="greedy"):
        model.set_phrase_boosting(PhraseBoostingConfig([[1, 2]]))
