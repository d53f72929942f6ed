"""Streaming without a GPU: the chunk planner's contract (reazonspeech_b200/streaming.py), carried-state decoding on the CPU
oracle, and StreamingTranscriber's host layer on a stub engine."""
import math
import random

import numpy as np
import pytest
import torch

from oracle import nemo_restated as O
from reazonspeech_b200.streaming import P, PAD_SAMPLES, StreamingConfig, conv_len, enc_valid, plan_row, stream_frames
from streaming_oracle import greedy_resume, oracle_stream


def mel_valid(n):                     # FilterbankFeatures.get_seq_len restated (n_fft 512, hop 160)
    return (n + 2 * 256 - 512) // 160


def enc_valid_ref(n):
    return conv_len(conv_len(conv_len(mel_valid(n))))


def test_enc_valid_shift_identity():
    """a a multiple of P: enc_valid(b - a) = enc_valid(b) - a / P for every b >= a (the decoded range lies in the buffer)."""
    for b in range(0, 40 * P, 37):
        assert enc_valid(b) == enc_valid_ref(b)
        for k in range(0, b // P + 1):
            assert enc_valid_ref(b - k * P) == enc_valid_ref(b) - k, (b, k)


@pytest.mark.parametrize("bad", [0.05, 0.1, 1.0 / 3, -0.08])
def test_config_rejects_off_grid(bad):
    with pytest.raises(ValueError):
        StreamingConfig(chunk_seconds=bad)
    with pytest.raises(ValueError):
        StreamingConfig(left_seconds=bad)
    with pytest.raises(ValueError):
        StreamingConfig(right_seconds=bad)


def test_config_frames():
    assert StreamingConfig().frames() == (20, 15, 15)
    assert StreamingConfig(0.08, 0.0, 0.0).frames() == (1, 0, 0)
    with pytest.raises(ValueError):
        StreamingConfig(chunk_seconds=0.0)


def simulate(rng, frames_cfg, total, pieces, close_after):
    """Push ``total`` samples in ``pieces``-sized bursts, closing after ``close_after`` bursts' worth; step after each push.
    Checks every planned row against the contract and returns the decoded global frame ranges."""
    C, Lc, R = frames_cfg
    n, D, closed, pushed, ranges = PAD_SAMPLES, 0, False, 0, []
    while True:
        if not closed:
            k = min(pieces(rng), total - pushed)
            pushed += k
            n += k
            if pushed >= total or rng.random() < close_after:
                n += PAD_SAMPLES
                closed = True
        F = stream_frames(n, closed)
        ready = n >= (D + C + R) * P or (closed and D < F)
        row = plan_row(n, D, closed, frames_cfg)
        assert (row is not None) == ready
        if row is None:
            if closed:
                return ranges, enc_valid(n)
            continue
        assert row.a % P == 0 and row.a == max(0, D - Lc) * P and row.b == min(n, (D + C + R) * P)
        assert row.offset == row.a // P and row.dec_begin == D - row.offset
        end = row.dec_end + row.offset
        assert D < end <= D + C and (F is None or end <= F)
        assert 0 <= row.dec_begin < row.dec_end <= enc_valid_ref(row.b - row.a)     # inside the buffer's valid frames
        ranges.append((D, end))
        D = end


@pytest.mark.parametrize("seed", range(40))
def test_planner_covers_every_frame_once(seed):
    rng = random.Random(seed)
    cfg = StreamingConfig(0.08 * rng.randint(1, 30), 0.08 * rng.randint(0, 25), 0.08 * rng.randint(0, 25))
    total = rng.randint(0, 16000 * 12)
    piece_max = rng.choice([1, 97, P, 5920, 16000 * 3])
    ranges, F = simulate(rng, cfg.frames(), total, lambda r: r.randint(1, piece_max), rng.choice([0.0, 0.01, 0.2]))
    covered = [f for lo, hi in ranges for f in range(lo, hi)]
    assert covered == list(range(F))
    C = cfg.frames()[0]
    assert all(hi - lo <= C for lo, hi in ranges)


def test_closed_stream_drains_in_ceil_steps():
    C, Lc, R = frames = StreamingConfig().frames()
    n = PAD_SAMPLES + 16000 * 7 + PAD_SAMPLES
    F = enc_valid(n)
    D = 0
    for already in range(0, F, 7):
        steps, D = 0, already
        while (row := plan_row(n, D, True, frames)) is not None:
            D = row.dec_end + row.offset
            steps += 1
        assert D == F and steps == math.ceil((F - already) / C)


# ---- carried-state decoding on the oracle
def _ep(tiny_cfg, tiny_sd, seconds, seed):
    from reazonspeech_b200.synth import synth_clip
    wave = np.pad(synth_clip(seed, seconds), PAD_SAMPLES).astype(np.float32)
    with torch.no_grad():
        enc = O.encoder(O.log_mel(torch.from_numpy(wave), tiny_cfg), tiny_sd, tiny_cfg)
        return O.joint_enc_proj(enc, tiny_sd)


def test_oracle_chunked_equals_unchunked(tiny_cfg, tiny_sd):
    rng = random.Random(3)
    for seed in (5, 6, 7):
        ep = _ep(tiny_cfg, tiny_sd, 3.0, seed)
        T = ep.shape[0]
        with torch.no_grad():
            full = O._greedy_loop(ep, tiny_sd, tiny_cfg, O.GreedyResult())
            multi = sorted({f for f in full.frames if full.frames.count(f) > 1})
            cuts = {0, T}
            cuts |= {f + 1 for f in multi}                               # right after a frame that emitted several tokens
            cuts |= {rng.randint(0, T) for _ in range(5)} | {1, T - 1}
            cuts = sorted(c for c in cuts if 0 <= c <= T)
            res, state = O.GreedyResult(), None
            for lo, hi in zip(cuts, cuts[1:] + [T]):
                res, state = greedy_resume(ep, tiny_sd, tiny_cfg, lo, hi, state, res)
        assert res.tokens == full.tokens and res.frames == full.frames and res.decisions == full.decisions
        assert res.margins == full.margins


def test_oracle_stream_unlimited_context_equals_transcribe(tiny_cfg, tiny_sd):
    from reazonspeech_b200.synth import synth_clip
    wave = synth_clip(8, 2.5).astype(np.float32)
    padded = np.pad(wave, PAD_SAMPLES).astype(np.float32)
    frames = StreamingConfig(0.4, 10.0, 10.0).frames()
    with torch.no_grad():
        ref = O.transcribe_tokens(torch.from_numpy(padded), tiny_sd, tiny_cfg)
    got = oracle_stream(wave, tiny_sd, tiny_cfg, frames)
    assert got.tokens == ref.tokens and got.frames == ref.frames and got.decisions == ref.decisions


# ---- host layer on a stub engine
class StubEngine:
    """Emits, for every decoded buffer frame f, the token (sample at f * P + P // 2 of the buffer) % V: with a signal that
    encodes its own global frame there, the host layer's frame offsets and buffer slicing are checked end to end."""

    def __init__(self, cfg, nbytes=64):
        self.cfg = cfg
        self.device = torch.device("cpu")
        self.stream_state_bytes = nbytes
        self.calls = []

    def stream_step(self, wav, lens, dec_begin, dec_end, slot, states, U, out, alpha=None):
        tokens, frames, ntok = out[:3]
        self.calls.append((wav.shape[0], slot.tolist()))
        assert len(set(slot.tolist())) == len(slot)
        for r in range(wav.shape[0]):
            n = 0
            for f in range(int(dec_begin[r]), int(dec_end[r])):
                i = f * P + P // 2
                v = int(wav[r, i]) if i < int(lens[r]) else 0
                tokens[r, n] = v % self.cfg.vocab_size
                frames[r, n] = f
                if alpha is not None:
                    out[3][r, n] = torch.tensor([-0.1, -0.2, 0.5, -0.3])
                n += 1
            ntok[r] = n
            states[int(slot[r]), 0] = 1
        return out


def _model(tiny_cfg, max_batch=2, **kw):
    from reazonspeech_b200.nemo.asr.transcribe import B200RnntModel
    from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces
    return B200RnntModel(StubEngine(tiny_cfg), PieceTableTokenizer(synthetic_pieces(tiny_cfg.vocab_size)), max_batch=max_batch, **kw)


def _signal(seconds):
    """int16 samples whose value at padded position g * P + P // 2 is g (the padding shifts it by PAD_SAMPLES)."""
    n = int(seconds * 16000)
    x = np.zeros(n, np.int16)
    for g in range(1, (PAD_SAMPLES + n) // P + 1):
        i = g * P + P // 2 - PAD_SAMPLES
        if 0 <= i < n:
            x[i] = g
    return x


def test_host_frames_offsets_and_result(tiny_cfg):
    from reazonspeech_b200.nemo.asr.decode import decode_hypothesis
    from reazonspeech_b200.nemo.asr.streaming import StreamingTranscriber
    from reazonspeech_b200.nemo.asr.transcribe import Hypothesis
    model = _model(tiny_cfg)
    st = StreamingTranscriber(model, StreamingConfig(0.4, 0.32, 0.24), max_streams=4)
    sigs = {}
    ids = []
    for k, secs in enumerate((3.0, 1.7, 4.3)):
        sid = st.open()
        ids.append(sid)
        sigs[sid] = _signal(secs)
    pos = {sid: 0 for sid in ids}
    finals = {sid: [] for sid in ids}
    rounds = 0
    while any(not st.done(s) for s in ids):
        for j, sid in enumerate(ids):
            if sid in st.open_streams and pos[sid] < len(sigs[sid]):
                step = 5920 + 1000 * j
                st.feed(sid, sigs[sid][pos[sid]:pos[sid] + step])
                pos[sid] += step
                if pos[sid] >= len(sigs[sid]):
                    st.close(sid)
        for sid, subs in st.step().items():
            finals[sid] += subs
        rounds += 1
        assert rounds < 500
    assert max(b for b, _ in model.engine.calls) <= 2                  # max_batch rows per engine call
    for sid in ids:
        n = PAD_SAMPLES * 2 + len(sigs[sid])
        F = enc_valid(n)
        hyp_frames = list(range(F))
        hyp_tokens = [(g if (g * P + P // 2 - PAD_SAMPLES) in range(len(sigs[sid])) else 0) % tiny_cfg.vocab_size for g in hyp_frames]
        ref = decode_hypothesis(model, Hypothesis.from_greedy(hyp_tokens, hyp_frames, tiny_cfg.blank))
        got = st.result(sid)
        assert got.text == ref.text and got.subwords == ref.subwords and got.segments == ref.segments
        assert [(s.token_id, s.seconds) for s in finals[sid]] == [(s.token_id, s.seconds) for s in ref.subwords]


def test_host_ids_and_slots_reused(tiny_cfg):
    from reazonspeech_b200.nemo.asr.streaming import StreamingTranscriber
    model = _model(tiny_cfg)
    st = StreamingTranscriber(model, StreamingConfig(0.4, 0.0, 0.0), max_streams=2)
    a, b = st.open(), st.open()
    assert (a, b) == (0, 1)
    with pytest.raises(RuntimeError):
        st.open()
    st.feed(a, np.zeros(8000, np.float32))
    st.close(a)
    while not st.done(a):
        st.step()
    assert st.result(a) is not None and a not in st.open_streams
    c = st.open()
    assert c == a and not st.done(c)
    assert int(st.states[c].sum()) == 0                                 # the reused record is zeroed
    with pytest.raises(KeyError):
        st.result(c)


def test_host_feed_rejects_other_dtypes(tiny_cfg):
    from reazonspeech_b200.nemo.asr.streaming import StreamingTranscriber
    st = StreamingTranscriber(_model(tiny_cfg), max_streams=1)
    sid = st.open()
    for bad in (np.zeros(10, np.float64), np.zeros((2, 10), np.float32), np.zeros(10, np.int32)):
        with pytest.raises(ValueError):
            st.feed(sid, bad)


def test_host_confidence_and_table_reset(tiny_cfg):
    from reazonspeech_b200.confidence import ConfidenceConfig
    from reazonspeech_b200.nemo.asr.streaming import StreamingTranscriber
    model = _model(tiny_cfg, confidence=ConfidenceConfig())
    st = StreamingTranscriber(model, StreamingConfig(0.4, 0.0, 0.0), max_streams=3)
    sid, other = st.open(), st.open()
    st.feed(sid, _signal(1.0))
    subs = [s for v in st.step().values() for s in v]
    assert subs and all(s.confidence is not None for s in subs)
    # a table change writes -1 into the boosting / LM word of every open stream's record
    st._tables_changed(1)
    st._tables_changed(2)
    words = st.states.view(torch.int32)
    assert words[sid, 1] == -1 and words[sid, 2] == -1 and words[other, 1] == -1 and words[2, 1] == 0


def test_rejects_alsd_and_multi_gpu(tiny_cfg):
    from reazonspeech_b200.nemo.asr.multi_gpu import MultiGpuRnntModel
    from reazonspeech_b200.nemo.asr.streaming import StreamingTranscriber
    with pytest.raises(ValueError):
        StreamingTranscriber(_model(tiny_cfg, decoding="alsd"))
    with pytest.raises(ValueError):
        StreamingTranscriber(MultiGpuRnntModel([_model(tiny_cfg), _model(tiny_cfg)]))
