"""ALSD beam search on the GPU (rs_rnnt_alsd, csrc/decode_alsd.cu) against its CPU oracle (oracle/alsd_restated.py: NeMo's
align_length_sync_decoding restated -- the reference's default decoding, pkg/nemo-asr/src/decode.py:29,38-40,48) on the SAME
encoder output: token sequences, alignment steps and scores.  Both evaluate log-probabilities to fp32 accuracy (the engine
splits activations into three bf16 terms), so the winning hypothesis must be identical; the score is compared to 1e-3."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from reazonspeech_b200.synth import synth_clip


@pytest.fixture(scope="module")
def alsd_engine(tiny_cfg, tiny_sd):
    from reazonspeech_b200.engine import Engine
    return Engine(tiny_cfg, tiny_sd, "cuda:0", alsd=True)


def _encode(eng, waves):
    L = max(len(w) for w in waves)
    x = torch.zeros(len(waves), L)
    for i, w in enumerate(waves):
        x[i, : len(w)] = torch.from_numpy(w)
    lens = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    mel, mel_len = eng.log_mel(x.cuda(), lens.cuda())
    return eng.encode(mel, mel_len)


# u_max_ratio < 2 ends most searches before any hypothesis finishes, so the winner comes from the last beam; the batch mixes
# lengths, so utterances end on steps of both parities and the beam is read from either half of the engine's double buffer
_CASES = [(1, True, True, 2.0), (2, True, True, 2.0), (4, True, True, 2.0), (4, False, True, 2.0), (4, True, False, 2.0), (8, True, True, 2.0),
          (4, True, True, 0.0), (4, True, True, 0.3)]


@pytest.mark.parametrize("beam,returns_input,score_norm,u_max_ratio", _CASES,
                         ids=[f"{b}-{r}-{s}" + ("" if u == 2.0 else f"-{u}") for b, r, s, u in _CASES])
def test_alsd_matches_the_oracle(alsd_engine, tiny_cfg, tiny_sd, beam, returns_input, score_norm, u_max_ratio):
    from oracle.alsd_restated import alsd_beam
    eng = alsd_engine
    waves = [np.pad(synth_clip(200 + i, s), 8000) for i, s in enumerate((2.0, 3.3, 0.9, 2.6, 1.4))]
    enc, enc_len = _encode(eng, waves)
    y, steps, n, score = [a.cpu() for a in eng.alsd(enc, enc_len, beam=beam, u_max_ratio=u_max_ratio, recombine_returns_input=returns_input,
                                                    score_norm=score_norm)]
    enc = enc.cpu()
    same = 0
    from_last_beam = 0
    for i in range(len(waves)):
        T = int(enc_len[i])
        ref = alsd_beam(enc[i, :T], tiny_sd, tiny_cfg, beam=beam, u_max_ratio=u_max_ratio, recombine_returns_input=returns_input,
                        score_norm=score_norm, emulate=True)
        from_last_beam += not ref.from_final
        k = int(n[i])
        got_y, got_steps = y[i, : k + 1].tolist(), steps[i, :k].tolist()
        print(f"beam {beam} utt{i}: T={T}, {k} tokens (oracle {len(ref.tokens)}), score {float(score[i]):.4f} (oracle {ref.score:.4f})")
        if got_y == ref.y_sequence and got_steps == ref.timestamp:
            same += 1
            assert abs(float(score[i]) - ref.score) < 1e-3 * max(1.0, abs(ref.score))
        else:                                        # a different winner is admissible only as a near-tie of the ranking key
            key = lambda s, ln: s / ln if score_norm else s
            assert abs(key(float(score[i]), k + 1) - key(ref.score, len(ref.y_sequence))) < 1e-3, (got_y[:12], ref.y_sequence[:12])
        assert got_y[0] == tiny_cfg.blank and all(0 <= s - j < T for j, s in enumerate(got_steps))     # frame = step - tokens before it
    assert same >= len(waves) - 1
    if u_max_ratio < 2.0:
        assert from_last_beam >= 1


def test_alsd_beam_one_equals_the_greedy_kernel_where_the_cap_does_not_bind(alsd_engine, tiny_cfg):
    """beam = 1 keeps the better of (blank, best token) at every step: the greedy decision sequence without max_symbols."""
    eng = alsd_engine
    waves = [np.pad(synth_clip(210 + i, s), 8000) for i, s in enumerate((2.2, 1.1, 3.0))]
    enc, enc_len = _encode(eng, waves)
    y, steps, n, _ = [a.cpu() for a in eng.alsd(enc, enc_len, beam=1)]
    tk, fr, nt = [a.cpu() for a in eng.greedy(enc, enc_len)]
    checked = 0
    for i in range(len(waves)):
        k = int(nt[i])
        frames = fr[i, :k].tolist()
        if k and max(np.bincount(frames)) >= tiny_cfg.max_symbols:
            continue                                 # greedy's symbol cap has no counterpart in ALSD
        assert int(n[i]) == k and y[i, 1 : k + 1].tolist() == tk[i, :k].tolist()
        assert [s - j for j, s in enumerate(steps[i, :k].tolist())] == frames
        checked += 1
    assert checked >= 1
