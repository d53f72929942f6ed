"""The drop-in Python surface on a GPU (pkg/nemo-asr/src/__init__.py:1-3 names + transcribe_batch): load_model ->
transcribe / transcribe_batch / the NeMo-shaped model.transcribe, on seeded synthetic weights of the tiny config.
Engine-level parity lives in test_gpu_kernels.py / test_gpu_full_model.py; here the host path around it is held to
the engine's own outputs: padding written in place, batching by length, pinned staging reuse, the worker-thread
pipeline and decode_hypothesis must not change a single token."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from reazonspeech_b200.synth import synth_clip


@pytest.fixture(scope="module")
def model(tiny_cfg):
    from reazonspeech_b200.nemo import asr
    return asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=4)


def test_transcribe_batch_equals_transcribe_and_the_engine(model, tiny_cfg):
    from reazonspeech_b200.nemo import asr
    cfgv = asr.TranscribeConfig(verbose=False, raw_hypothesis=True)
    clips = [synth_clip(100 + i, s) for i, s in enumerate((2.0, 0.7, 3.1, 1.3, 2.6, 0.9, 4.2))]
    audios = [asr.audio_from_numpy(c, 16000) for c in clips]
    single = [asr.transcribe(model, a, cfgv) for a in audios]
    for rep in range(2):                                              # second pass reuses the (dirty) staging buffers
        batch = asr.transcribe_batch(model, audios, cfgv)
        assert len(batch) == len(audios)
        for i, (b, s) in enumerate(zip(batch, single)):
            assert b.hypothesis.y_sequence.tolist() == s.hypothesis.y_sequence.tolist(), f"clip {i}, pass {rep}"
            assert list(b.hypothesis.timestamp) == list(s.hypothesis.timestamp)
            assert b.text == s.text and b.subwords == s.subwords and b.segments == s.segments
    # the engine called directly on the reference's padded waveform (pad_audio: 0.5 s both sides)
    eng = model.engine
    n_tok = 0
    for i, c in enumerate(clips):
        w = np.pad(c.astype(np.float32), 8000)
        x = torch.from_numpy(w)[None].cuda()
        t, f, n = eng.transcribe_device(x, torch.tensor([len(w)], dtype=torch.int32).cuda())
        n = int(n[0])
        hyp = single[i].hypothesis
        assert hyp.y_sequence.tolist() == [tiny_cfg.blank] + t[0, :n].cpu().tolist()
        assert [ts - k - 1 for k, ts in enumerate(hyp.timestamp)] == f[0, :n].cpu().tolist()     # decode.py:48 recovers the frame
        n_tok += n
    assert n_tok > 0, "the synthetic checkpoint emitted nothing: the comparison above is vacuous"
    for r in single:
        assert all(s.seconds >= 0 for s in r.subwords)
        assert r.text == model.tokenizer.ids_to_text(r.hypothesis.y_sequence.tolist()[1:])


def test_nemo_call_shape(model, tiny_cfg):
    """model.transcribe(list_of_tensors, batch_size, return_hypotheses, verbose) as pkg/nemo-asr/src/transcribe.py:48-53 calls it."""
    w = torch.from_numpy(np.pad(synth_clip(120, 1.5), 8000).astype(np.float32))
    hyps = model.transcribe([w], batch_size=1, return_hypotheses=True, verbose=False)
    assert len(hyps) == 1 and int(hyps[0].y_sequence[0]) == tiny_cfg.blank
    assert len(hyps[0].timestamp) == len(hyps[0].y_sequence) - 1
    texts = model.transcribe([w, w[: len(w) // 2]], batch_size=2, return_hypotheses=False, verbose=False)
    assert len(texts) == 2 and all(isinstance(t, str) for t in texts)


def test_two_engines_on_one_device_and_second_device_are_independent(tiny_cfg, tiny_sd):
    """include/rs_engine.h promises 'distinct engines are independent' and load_model accepts 'cuda:N': the opt-in to more
    than 48 KB of dynamic shared memory is per DEVICE (cudaFuncSetAttribute), so an engine created on another GPU after one
    on cuda:0 must work (it failed with 'invalid argument' while the flag was process-wide).  Runs the second engine on the
    last visible device (the same one on a one-GPU box, where it still checks two engines side by side)."""
    from reazonspeech_b200.engine import Engine
    dev = torch.cuda.device_count() - 1
    e0 = Engine(tiny_cfg, tiny_sd, "cuda:0")
    e1 = Engine(tiny_cfg, tiny_sd, f"cuda:{dev}")
    w = np.pad(synth_clip(130, 2.2), 8000).astype(np.float32)
    x, ln = torch.from_numpy(w)[None], torch.tensor([len(w)], dtype=torch.int32)
    t0, f0, n0 = e0.transcribe_device(x.to("cuda:0"), ln.to("cuda:0"))
    with torch.cuda.device(dev):
        t1, f1, n1 = e1.transcribe_device(x.to(f"cuda:{dev}"), ln.to(f"cuda:{dev}"))
    n = int(n0[0])
    assert n > 0 and int(n1[0]) == n and torch.equal(t0[0, :n].cpu(), t1[0, :n].cpu()) and torch.equal(f0[0, :n].cpu(), f1[0, :n].cpu())


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_one_process_multi_gpu_equals_single_gpu(model, tiny_cfg):
    """load_model(devices=[0, 1]): one replica, worker thread and staging pair per device in ONE process; the merged result
    equals the one-GPU result token for token and arrives in input order (SURVEY.md section 8e; the reference's
    counterpart is one spawned process per GPU, pkg/evaluation/src/base.py:194-212)."""
    from reazonspeech_b200.nemo import asr
    multi = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=4, devices=[0, 1])
    assert multi.devices == ["cuda:0", "cuda:1"]
    cfgv = asr.TranscribeConfig(verbose=False, raw_hypothesis=True)
    audios = [asr.audio_from_numpy(synth_clip(140 + i, 0.8 + 0.45 * (i % 9)), 16000) for i in range(23)]
    one = asr.transcribe_batch(model, audios, cfgv)
    for rep in range(2):
        two = asr.transcribe_batch(multi, audios, cfgv)
        assert len(two) == len(one)
        for i, (a, b) in enumerate(zip(one, two)):
            assert a.hypothesis.y_sequence.tolist() == b.hypothesis.y_sequence.tolist(), f"clip {i}, pass {rep}"
            assert list(a.hypothesis.timestamp) == list(b.hypothesis.timestamp) and a.text == b.text
    assert sum(len(r.subwords) for r in two) > 0
    single = asr.transcribe(multi, audios[3], cfgv)                    # the reference's one-clip call shape on the multi-GPU model
    assert single.text == one[3].text


def test_transcribe_batch_normalises_foreign_rates_on_the_gpu(model, tiny_cfg):
    """A call whose clips all come at 44.1 kHz stereo PCM takes the device route (iter_token_batches_raw: H2D of the raw
    samples, rs_resample_mono, rs_transcribe_device); its results equal the host route's (norm_audio on the CPU) up to the
    two resamplers' fp32 rounding: same text on nearly all tokens, same count within a few."""
    from reazonspeech_b200.nemo import asr
    rate = 44100
    g = np.random.default_rng(3)
    clips = []
    for i, secs in enumerate((1.4, 2.3, 0.8, 3.0, 1.9)):
        t = np.arange(int(rate * secs)) / rate
        x = np.stack([0.3 * np.sin(2 * np.pi * (200 + 70 * (i + c)) * t * (1 + 0.1 * np.sin(2 * np.pi * 4 * t))) + 0.02 * g.standard_normal(len(t))
                      for c in range(2)])
        clips.append(np.round(x * 32767.0).astype(np.int16))
    audios = [asr.audio_from_numpy(c, rate) for c in clips]
    cfgv = asr.TranscribeConfig(verbose=False, raw_hypothesis=True)
    calls = {"raw": 0}
    orig = model.iter_token_batches_raw

    def spy(*a, **k):
        calls["raw"] += 1
        return orig(*a, **k)

    model.iter_token_batches_raw = spy
    try:
        dev = asr.transcribe_batch(model, audios, cfgv)
    finally:
        del model.iter_token_batches_raw
    assert calls["raw"] == 1
    host = [asr.transcribe(model, a, cfgv) for a in audios]              # one clip per call: norm_audio on the host (scipy)
    total = 0
    for d, h in zip(dev, host):
        nd, nh = len(d.hypothesis.y_sequence), len(h.hypothesis.y_sequence)
        assert abs(nd - nh) <= max(2, nh // 10)
        total += nd - 1
    assert total > 0


def test_alsd_decoding_through_the_reference_call_shape(tiny_cfg):
    """load_model(decoding="alsd"): model.transcribe hands back NeMo-shaped ALSD hypotheses (leading blank, alignment steps)
    which decode_hypothesis -- byte-compatible with the reference's decode.py -- turns into subwords with non-negative,
    non-decreasing times; beam 1 reproduces the greedy text where greedy's symbol cap does not bind."""
    from reazonspeech_b200.nemo import asr
    m = asr.load_model("cuda:0", synthetic=True, config=tiny_cfg, seed=0, max_batch=4, decoding="alsd", beam_size=4)
    audios = [asr.audio_from_numpy(synth_clip(160 + i, 1.0 + 0.7 * i), 16000) for i in range(5)]
    cfgv = asr.TranscribeConfig(verbose=False, raw_hypothesis=True)
    res = asr.transcribe_batch(m, audios, cfgv)
    assert len(res) == 5
    for r in res:
        h = r.hypothesis
        assert int(h.y_sequence[0]) == tiny_cfg.blank and len(h.timestamp) == len(h.y_sequence) - 1
        secs = [s.seconds for s in r.subwords]
        assert all(s >= 0 for s in secs) and secs == sorted(secs)
    one = asr.transcribe(m, audios[2], cfgv)
    assert one.text == res[2].text
