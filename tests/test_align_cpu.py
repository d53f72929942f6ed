"""Forced alignment without a GPU: the float64 oracle (tests/align_oracle.py) against brute-force path enumeration and
torchaudio's RNN-T loss, the lattice built from oracle/nemo_restated.py, the accuracy bars of the GPU tests against the error of
plausible mis-implementations, and the host logic (tokenisation, hypotheses, validation, the CLI)."""
import numpy as np
import pytest
import torch

import align_oracle as A
from reazonspeech_b200.alignment import alignment_hypothesis, pack_labels, validate_labels
from reazonspeech_b200.tokenizer import PieceTableTokenizer, synthetic_pieces, WORD_BOUNDARY

LATTICE_BAR = 2e-4          # max |lp - float64 reference| of the GPU lattice (tests/test_gpu_align.py)


def _random_lattice(rng, T, U):
    return np.log(rng.uniform(0.05, 1.0, (T, U + 1))), np.log(rng.uniform(0.05, 1.0, (T, U + 1)))


@pytest.mark.parametrize("T", [1, 2, 3, 4])
@pytest.mark.parametrize("U", [0, 1, 2, 3])
def test_recursions_equal_brute_force(T, U):
    rng = np.random.default_rng(10 * T + U)
    for _ in range(3):
        lpb, lpe = _random_lattice(rng, T, U)
        r = A.align(lpb, lpe, T, U)
        loglik, best, frames = A.brute_force(lpb, lpe, T, U)
        assert abs(r["loglik"] - loglik) < 1e-12 and abs(r["viterbi"] - best) < 1e-12
        assert r["frames"].tolist() == frames.tolist()
        assert np.allclose(r["token_lp"], [lpe[f, u] for u, f in enumerate(frames)])
    zero = np.zeros((T, U + 1))                                    # every path ties: the tie rule decides the frames
    r = A.align(zero, zero, T, U)
    assert r["frames"].tolist() == A.brute_force(zero, zero, T, U)[2].tolist() == [0] * U


def test_recursion_matches_torchaudio_rnnt_loss():
    ta = pytest.importorskip("torchaudio")
    rng = np.random.default_rng(3)
    B, T_max, U_max, V = 5, 9, 6, 11
    logits = torch.from_numpy(rng.normal(size=(B, T_max, U_max + 1, V + 1)) * 2).float()
    T = torch.tensor([9, 4, 1, 7, 3], dtype=torch.int32)
    U = torch.tensor([6, 0, 3, 2, 5], dtype=torch.int32)
    labels = torch.from_numpy(rng.integers(0, V, (B, U_max))).int()
    loss = ta.functional.rnnt_loss(logits, labels, T, U, blank=V, reduction="none", fused_log_softmax=True)
    for b in range(B):
        Tb, Ub = int(T[b]), int(U[b])
        lpb, lpe = A.lattice_from_logits(logits[b, :Tb, : Ub + 1].double(), labels[b, :Ub].tolist(), V)
        r = A.align(lpb, lpe, Tb, Ub)
        assert abs(r["loglik"] + float(loss[b])) < 1e-4, b
        assert r["viterbi"] <= r["loglik"] + 1e-12


def _tiny_case(cfg, sd, T=10, U=6, seed=1):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(T, cfg.d_model, generator=g)
    labels = [int(x) for x in torch.randint(0, cfg.vocab_size, (U,), generator=g)]
    return enc, labels


def test_lattice_from_the_oracle_predictor_and_joint(tiny_cfg, tiny_sd):
    """Row u of the lattice is the joint after feeding y_1..y_u: it equals the greedy oracle's own joint evaluation there."""
    import nemo_restated as O
    enc, labels = _tiny_case(tiny_cfg, tiny_sd)
    lpb, lpe = A.lattice(enc, labels, tiny_sd, tiny_cfg)
    hp = tiny_cfg.pred_hidden
    emb = tiny_sd["decoder.prediction.embed.weight"]
    h, c = O.lstm_step(torch.zeros(hp), torch.zeros(hp), torch.zeros(hp), tiny_sd)
    ep = O.joint_enc_proj(enc.to(torch.bfloat16).float(), tiny_sd)
    W, b = tiny_sd["joint.joint_net.2.weight"], tiny_sd["joint.joint_net.2.bias"]
    for u in range(len(labels) + 1):
        pp = torch.nn.functional.linear(h, tiny_sd["joint.pred.weight"], tiny_sd["joint.pred.bias"])
        for t in (0, 4, 9):
            lsm = torch.log_softmax(torch.nn.functional.linear(torch.relu(ep[t] + pp), W, b).double(), -1)
            assert abs(float(lsm[tiny_cfg.blank]) - lpb[t, u]) < 1e-5
            if u < len(labels):
                assert abs(float(lsm[labels[u]]) - lpe[t, u]) < 1e-5
        if u < len(labels):
            h, c = O.lstm_step(emb[labels[u]], h, c, tiny_sd)
    assert np.all(np.isneginf(lpe[:, len(labels)]))


@pytest.mark.parametrize("full", [False, True])
def test_lattice_bar_separates_mis_implementations(full, tiny_cfg, tiny_sd):
    """The GPU lattice bar lies at least 3x below the error of: one half term instead of two, no b_out, the target taken from
    y_u instead of y_{u+1}, lp_emit shifted by one frame (the same check as test_gpu_encoder_kernels.py's bars)."""
    if full:
        from reazonspeech_b200.config import ModelConfig
        from reazonspeech_b200.weights import random_state_dict
        cfg = ModelConfig(); sd = random_state_dict(cfg, seed=0)
    else:
        cfg, sd = tiny_cfg, tiny_sd
    enc, labels = _tiny_case(cfg, sd, T=12, U=7)
    _, pp = A.predictor(labels, sd, cfg)
    ep = A.enc_proj(enc, sd)
    U = len(labels)
    lpb, lpe = A.lattice_from_logits(A.joint_logits(ep, pp, sd), labels, cfg.blank)

    def err(b, e):
        return max(np.abs(b - lpb).max(), np.abs(e[:, :U] - lpe[:, :U]).max())

    W, bias = sd["joint.joint_net.2.weight"].double(), sd["joint.joint_net.2.bias"].double()
    act = torch.relu(ep[:, None, :] + pp[None])
    one_term = act.half().double() @ W.T + bias
    two_terms = (act.half().double() + (act - act.half().float()).half().double()) @ W.T + bias
    wrong = {
        "one half term": A.lattice_from_logits(one_term, labels, cfg.blank),
        "no b_out": A.lattice_from_logits(A.joint_logits(ep, pp, sd, b_out=False), labels, cfg.blank),
        "target y_u": A.lattice_from_logits(A.joint_logits(ep, pp, sd), [labels[0]] + labels[:-1], cfg.blank),
        "lp_emit one frame late": (lpb, np.roll(lpe, 1, axis=0)),
    }
    for name, (b, e) in wrong.items():
        assert 3 * LATTICE_BAR <= err(b, e), f"{name}: error {err(b, e):.2e}"
    assert err(*A.lattice_from_logits(two_terms, labels, cfg.blank)) < LATTICE_BAR / 10


def test_sentence_tokenisation_keeps_the_boundary_piece():
    tok = PieceTableTokenizer(synthetic_pieces(3000))
    text = tok.ids_to_text([60, 61, 2])
    ids = tok.sentence_to_ids(text)
    assert tok.pieces[ids[0]] == WORD_BOUNDARY and ids[1:] == [60, 61, 2]
    assert tok.text_to_ids(text) == ids[1:]                  # phrase tokenisation drops it
    with pytest.raises(ValueError):
        tok.sentence_to_ids("abc")


def test_validation_and_packing():
    assert validate_labels([[1, 2], []], 10, 2) == [[1, 2], []]
    for bad in ([[1, 10]], [[-1]]):
        with pytest.raises(ValueError):
            validate_labels(bad, 10, 1)
    with pytest.raises(ValueError):
        validate_labels([[1]], 10, 2)
    labels, lens = pack_labels([[3, 4, 5], []])
    assert labels.tolist() == [[3, 4, 5], [0, 0, 0]] and lens.tolist() == [3, 0]
    assert pack_labels([[]])[0].shape == (1, 1)


def test_align_builds_the_transcription_shaped_result(tiny_cfg):
    """align_batch: the hypothesis of given (ids, frames) goes through the unchanged decode_hypothesis, so subwords and segment
    times are exactly a transcription's of the same tokens at the same frames; score = Viterbi, plus the two new fields."""
    from reazonspeech_b200.nemo.asr import align_batch, audio_from_numpy
    from reazonspeech_b200.nemo.asr.decode import build_result
    from reazonspeech_b200.nemo.asr.transcribe import Hypothesis

    class FakeModel:
        cfg = tiny_cfg
        tokenizer = PieceTableTokenizer(synthetic_pieces(tiny_cfg.vocab_size))

        def align_tokens(self, waves, ids, pad):
            self.seen = (len(waves), ids, pad)
            return [([3 * i for i in range(len(k))], [-0.5] * len(k), -4.0, -3.0) for k in ids]

    m = FakeModel()
    text = m.tokenizer.ids_to_text([60, 2, 61])
    audios = [audio_from_numpy(np.zeros(16000, np.float32), 16000)] * 2
    r = align_batch(m, audios, [text, [61, 62]])
    assert m.seen[0] == 2 and m.seen[2] == 8000 and m.seen[1][1] == [61, 62]
    ids = m.tokenizer.sentence_to_ids(text)
    assert m.seen[1][0] == ids
    hyp = r[0].hypothesis
    assert hyp.y_sequence.tolist() == Hypothesis.from_greedy(ids, [0, 3, 6, 9], tiny_cfg.blank).y_sequence.tolist()
    assert hyp.score == -4.0 and hyp.log_likelihood == -3.0 and hyp.token_logprob == [-0.5] * 4
    expect = build_result(m.tokenizer, ids, [f + i + 1 for i, f in enumerate([0, 3, 6, 9])])
    assert r[0].text == expect.text and [w.seconds for w in r[0].subwords] == [w.seconds for w in expect.subwords]
    assert [w.token_id for w in r[1].subwords] == [61, 62]
    assert Hypothesis.from_greedy([1], [0], 5).log_likelihood is None        # transcriptions keep the defaults
    with pytest.raises(ValueError):
        align_batch(m, audios, [text])
    with pytest.raises(ValueError):
        align_batch(m, audios, [[tiny_cfg.vocab_size], [1]])


def test_cli_text_option(tmp_path):
    from reazonspeech_b200.nemo.asr import cli
    opt = cli.parse(["--text=t.txt", "a.wav", "b.wav"])
    assert opt.text == "t.txt" and opt.audio == ["a.wav", "b.wav"]
    assert cli.parse(["a.wav"]).text is None
    f = tmp_path / "t.txt"
    f.write_text("こんにちは\nさようなら\n", encoding="utf-8")
    assert cli.load_transcripts(str(f), 2) == ["こんにちは", "さようなら"]
    with pytest.raises(ValueError):
        cli.load_transcripts(str(f), 3)
    with pytest.raises(ValueError):
        cli.run(cli.parse([f"--text={f}", "only_one.wav"]))
