"""Confidence statistics of the greedy decode kernel (kConf) on the GPU: the decisions do not change, and the statistics of
every emitted token match the oracle's log_softmax (float64) of its fp32 logits, walked along the engine's own decisions."""
import numpy as np
import pytest
import torch

from confidence_oracle import follow_stats
from parity import decisions_from

pytestmark = pytest.mark.gpu

TOL = 1e-3
ALPHAS = (1.0, 0.33)


def _check_stats(eng, cfg, sd, enc, enc_len, tag, U=None):
    """Decode ``enc`` with and without statistics at every alpha; decisions byte-identical, statistics within TOL of the
    oracle for every stored token.  Returns the largest difference."""
    enc_d, len_d = enc.cuda().contiguous(), enc_len.cuda()
    base = [a.cpu() for a in eng.greedy(enc_d, len_d, U)]
    worst = 0.0
    for alpha in ALPHAS:
        tk, fr, nt, st = [a.cpu() for a in eng.greedy(enc_d, len_d, U, alpha=alpha)]
        assert torch.equal(tk, base[0]) and torch.equal(fr, base[1]) and torch.equal(nt, base[2]), f"{tag}: decisions depend on kConf"
        Ucap = tk.shape[1]
        for b in range(enc.shape[0]):
            n, T = int(nt[b]), int(enc_len[b])
            k = min(n, Ucap)
            assert torch.all(st[b, k:] == 0), f"{tag}: statistics written past the stored tokens of utterance {b}"
            if n > Ucap:
                continue                                   # the decision sequence is incomplete: compared in test_u_max_below_n_tok
            ref = follow_stats(enc[b, :T], sd, cfg, decisions_from(tk[b, :n].tolist(), fr[b, :n].tolist(), T, cfg.max_symbols, cfg.blank), [alpha])[alpha]
            if n == 0:
                continue
            d = (st[b, :n].double() - torch.tensor(ref, dtype=torch.float64)).abs()
            worst = max(worst, float(d.max()))
            assert float(d.max()) <= TOL, f"{tag} b={b} alpha={alpha}: |delta| per column {d.max(0).values.tolist()}"
    print(f"{tag}: largest |delta stats| vs the oracle {worst:.3e}")
    return worst


def _tiny_enc(cfg, lens, seed, T=None):
    g = torch.Generator().manual_seed(seed)
    T = T or max(lens)
    enc = torch.randn(len(lens), T, cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc, torch.tensor(lens, dtype=torch.int32)


def test_tiny_ragged_and_window_past_the_end(tiny_cfg, tiny_sd, tiny_engine):
    """Ragged batch; lengths that are not a multiple of the 4-frame window, so windows run past utterance ends; 1 frame."""
    enc, lens = _tiny_enc(tiny_cfg, [37, 1, 6, 23, 40, 13, 2, 31, 9], seed=1)
    _check_stats(tiny_engine, tiny_cfg, tiny_sd, enc, lens, "tiny ragged")


def test_tiny_symbol_cap(tiny_cfg, tiny_sd):
    """Blank suppressed: every frame reaches max_symbols."""
    from reazonspeech_b200.engine import Engine
    sd = dict(tiny_sd)
    b = sd["joint.joint_net.2.bias"].clone()
    b[tiny_cfg.blank] = -1e4
    sd["joint.joint_net.2.bias"] = b
    eng = Engine(tiny_cfg, sd, "cuda:0")
    enc, lens = _tiny_enc(tiny_cfg, [11, 5, 16], seed=2)
    _check_stats(eng, tiny_cfg, sd, enc, lens, "tiny symbol cap")
    tk, fr, nt = eng.greedy(enc.cuda(), lens.cuda())
    assert nt.cpu().tolist() == [int(n) * tiny_cfg.max_symbols for n in lens]


def test_u_max_below_n_tok(tiny_cfg, tiny_sd, tiny_engine):
    """U_max below the token count: the first U_max statistics equal the uncapped run's, nothing lands past U_max."""
    enc, lens = _tiny_enc(tiny_cfg, [40, 33, 21, 40], seed=3)
    full = [a.cpu() for a in tiny_engine.greedy(enc.cuda(), lens.cuda(), alpha=0.33)]
    n = full[2]
    U = max(1, int(n.min()) // 2)
    assert int(n.min()) > U
    tk, fr, nt, st = [a.cpu() for a in tiny_engine.greedy(enc.cuda(), lens.cuda(), U, alpha=0.33)]
    assert torch.equal(nt, n) and torch.equal(tk, full[0][:, :U]) and torch.equal(fr, full[1][:, :U])
    assert torch.equal(st, full[3][:, :U])


def test_alpha_is_validated(tiny_cfg, tiny_engine):
    enc, lens = _tiny_enc(tiny_cfg, [8], seed=4)
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(RuntimeError, match="rs_rnnt_greedy_confidence"):
            tiny_engine.greedy(enc.cuda(), lens.cuda(), alpha=bad)


def test_tiny_whole_path(tiny_cfg, tiny_sd, tiny_engine):
    """transcribe_device: float and PCM16 input, with and without statistics; the same statistics from the host call."""
    g = torch.Generator().manual_seed(5)
    L = 40000
    pcm = (3000 * torch.randn(5, L, generator=g)).to(torch.int16)
    lens = torch.tensor([L, 9000, 17003, 31000, 4000], dtype=torch.int32)
    wav = pcm.float() / 32768.0
    base = [a.cpu() for a in tiny_engine.transcribe_device(wav.cuda(), lens.cuda())]
    on = [a.cpu() for a in tiny_engine.transcribe_device(wav.cuda(), lens.cuda(), alpha=0.33)]
    on16 = [a.cpu() for a in tiny_engine.transcribe_device(pcm.cuda(), lens.cuda(), alpha=0.33)]
    host = tiny_engine.transcribe_host(wav.pin_memory(), lens, alpha=0.33)
    n = on[2]
    assert torch.equal(base[2], n) and torch.equal(on16[2], n) and torch.equal(host[2], n) and int(n.sum()) > 0
    for b in range(5):                   # the host call returns the workspace's rows: entries past n_tok are not part of the result
        k = int(n[b])
        for i in (0, 1, 3):
            ref = on[i][b, :k]
            assert torch.equal(on16[i][b, :k], ref) and torch.equal(host[i][b, :k], ref)
            if i < 3:
                assert torch.equal(base[i][b, :k], ref)


def test_production_geometry():
    """BASELINE.json configs[1] geometry (32 x 30 s clips in one batch, full model, V + 1 = 3001 classes over S slices): the
    decode kernel alone, fed the encoder output of the bench's clips, against the oracle at alpha = 1 and 0.33."""
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    sd = random_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, "cuda:0")
    waves = [np.pad(synth_clip(i, 30.0), 8000) for i in range(32)]
    x = torch.from_numpy(np.stack(waves)).float().cuda()
    lens = torch.full((32,), len(waves[0]), dtype=torch.int32).cuda()
    mel, mel_len = eng.log_mel(x, lens)
    enc, enc_len = eng.encode(mel, mel_len)
    base = [a.cpu() for a in eng.transcribe_device(x, lens)]
    on = [a.cpu() for a in eng.transcribe_device(x, lens, alpha=0.33)]
    for i in range(3):
        assert torch.equal(base[i], on[i]), "whole path: decisions depend on kConf"
    worst = _check_stats(eng, cfg, sd, enc.cpu(), enc_len.cpu(), "32 x 30 s")
    print(f"production geometry: {int(base[2].sum())} tokens, largest |delta stats| {worst:.3e}")


def test_transcribe_batch_confidence(tiny_cfg):
    """The public path: texts unchanged, confidences in [0, 1], score = sum lp, subword confidences, PCM16 / resampling paths."""
    from reazonspeech_b200.confidence import ConfidenceConfig
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    off = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3)
    on = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=3, confidence=ConfidenceConfig())
    clips = [synth_clip(60 + i, s) for i, s in enumerate((1.5, 3.0, 2.2, 4.0, 0.7))]
    audios = [AudioData(c.astype(np.float32), 16000) for c in clips]
    r_off = asr.transcribe_batch(off, audios, asr.TranscribeConfig(raw_hypothesis=True))
    r_on = asr.transcribe_batch(on, audios, asr.TranscribeConfig(raw_hypothesis=True))
    n_conf = 0
    for a, b in zip(r_off, r_on):
        assert a.text == b.text and [w.token_id for w in a.subwords] == [w.token_id for w in b.subwords]
        assert a.hypothesis.score == 0.0 and a.hypothesis.token_confidence is None
        h = b.hypothesis
        n = len(h.y_sequence) - 1
        assert len(h.token_confidence) == n and all(0.0 <= c <= 1.0 for c in h.token_confidence)
        assert h.word_confidence is not None and all(0.0 <= c <= 1.0 for c in h.word_confidence)
        kept = [c for c, t in zip(h.token_confidence, h.y_sequence.tolist()[1:]) if on.tokenizer.ids_to_text([t])]
        assert [w.confidence for w in b.subwords] == kept
        assert all(w.confidence is None for w in a.subwords)
        n_conf += n
    assert n_conf > 0
    # score = sum of the emitted tokens' log-probabilities (the statistics of the engine call)
    pad = 8000
    items = on.transcribe_tokens([np.asarray(c, np.float32) for c in clips], pad=pad)
    for r, (tk, fr, st) in zip(r_on, items):
        assert r.hypothesis.score == pytest.approx(float(np.asarray(st, np.float64)[:, 0].sum()), rel=1e-12, abs=1e-12)
    # PCM16 and resampling paths: the same statistics as the float path on the same samples
    pcm = [(np.clip(c, -1, 1) * 32767).astype(np.int16) for c in clips]
    r16 = asr.transcribe_batch(on, [AudioData(p, 16000) for p in pcm], asr.TranscribeConfig(raw_hypothesis=True))
    rf = asr.transcribe_batch(on, [AudioData(p.astype(np.float32) / 32768.0, 16000) for p in pcm], asr.TranscribeConfig(raw_hypothesis=True))
    for a, b in zip(r16, rf):
        assert a.text == b.text and a.hypothesis.token_confidence == b.hypothesis.token_confidence and a.hypothesis.score == b.hypothesis.score
    stereo = [np.stack([c, c]).astype(np.float32) for c in clips]       # two equal channels: down-mixing keeps the samples
    i_raw = list(on.iter_token_batches_raw(stereo, 16000, pad=pad))
    i_host = list(on.iter_token_batches([c.astype(np.float32) for c in clips], pad=pad))
    raw = {i: it for idx, its in i_raw for i, it in zip(idx, its)}
    host = {i: it for idx, its in i_host for i, it in zip(idx, its)}
    for i in range(len(clips)):
        assert raw[i][0] == host[i][0] and np.array_equal(raw[i][2], host[i][2])


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_gpu_confidence(tiny_cfg):
    from reazonspeech_b200.confidence import ConfidenceConfig
    from reazonspeech_b200.nemo import asr
    from reazonspeech_b200.nemo.asr.interface import AudioData
    from reazonspeech_b200.synth import synth_clip
    one = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, confidence=ConfidenceConfig())
    two = asr.load_model(synthetic=True, config=tiny_cfg, seed=0, max_batch=2, devices=[0, 1], confidence=ConfidenceConfig())
    audios = [AudioData(synth_clip(80 + i, 1.0 + 0.4 * i).astype(np.float32), 16000) for i in range(6)]
    cfg = asr.TranscribeConfig(raw_hypothesis=True)
    for a, b in zip(asr.transcribe_batch(one, audios, cfg), asr.transcribe_batch(two, audios, cfg)):
        assert a.text == b.text and a.hypothesis.token_confidence == b.hypothesis.token_confidence
        assert a.hypothesis.word_confidence == b.hypothesis.word_confidence and a.hypothesis.score == b.hypothesis.score
