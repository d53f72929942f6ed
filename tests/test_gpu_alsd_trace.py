"""ALSD beam search on the GPU step by step, through the trace seam (rs_rnnt_alsd_trace): the log-probabilities of every row the
search scored against float64, the beam update of every step replayed exactly by the oracle's own step
(oracle/alsd_restated.py::alsd_step), the crafted inputs on which recombination and u_max decide the winner, batch invariance,
and the edges (one- and two-frame utterances, an empty one, U_cap below the winner's length)."""
import numpy as np
import pytest
import torch

import alsd_cases as AC
from oracle.alsd_restated import alsd_beam
from reazonspeech_b200.synth import synth_clip

pytestmark = pytest.mark.gpu

_WAVES = [(300, 2.0), (301, 3.3), (302, 0.9), (303, 2.6), (304, 1.4)]


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


@pytest.fixture(scope="module")
def tiny_enc(alsd_engine):
    return _encode(alsd_engine, [np.pad(synth_clip(s, d), 8000) for s, d in _WAVES])


def _check_logps(tr, enc, enc_len, sd, cfg, beam):
    """Every traced row against float64 -> (worst error, rows checked)."""
    worst, n_rows = 0.0, 0
    for b in range(enc.shape[0]):
        J = AC.Float64Joint(enc[b, : int(enc_len[b])], sd, cfg)
        for i, k, toks, t in AC.scored_rows(tr, b, cfg.blank):
            ref = J.logp(toks, t)
            lp = tr["cand_logp"][i, b, k].double()
            got = [int(x) for x in tr["cand_tok"][i, b, k, :beam]]
            want = J.top(ref, beam)
            err = abs(float(lp[0]) - float(ref[cfg.blank]))
            for c in range(beam):
                err = max(err, abs(float(lp[1 + c]) - float(ref[want[c]])), abs(float(lp[1 + c]) - float(ref[got[c]])))
                if got[c] != want[c]:                              # only a near-tie of the float64 values may swap classes
                    assert abs(float(ref[got[c]]) - float(ref[want[c]])) < AC.LP_BAR, (i, b, k, c, got, want)
            worst = max(worst, err)
            n_rows += 1
    return worst, n_rows


_CASES = [(1, True, True), (2, True, True), (4, True, True), (4, False, True), (4, True, False), (4, False, False), (8, True, True),
          (8, False, True)]
_IDS = [f"beam{b}-{'input' if r else 'merged'}-{'norm' if s else 'raw'}" for b, r, s in _CASES]
_traces = {}


def _trace(eng, enc_pair, case):
    if case not in _traces:
        beam, returns_input, score_norm = case
        enc, enc_len = enc_pair
        _traces[case] = eng.alsd_trace(enc, enc_len, beam=beam, score_norm=score_norm, recombine_returns_input=returns_input)
    return _traces[case]


@pytest.mark.parametrize("case", _CASES, ids=_IDS)
def test_alsd_log_probabilities_match_float64(alsd_engine, tiny_enc, tiny_cfg, tiny_sd, case):
    """log p(blank) and the top-k of every row the search scored, at every step, within LP_BAR of float64; the classes are
    float64's top-k (lower index first on ties) except where float64 values lie within LP_BAR of each other."""
    tr = _trace(alsd_engine, tiny_enc, case)
    enc, enc_len = tiny_enc
    worst, n_rows = _check_logps(tr, enc.cpu(), enc_len.cpu(), tiny_sd, tiny_cfg, case[0])
    print(f"{case}: {n_rows} rows, worst |log p - float64| {worst:.2e} (bar {AC.LP_BAR:.0e})")
    assert n_rows >= 100 and worst < AC.LP_BAR


@pytest.mark.parametrize("case", _CASES, ids=_IDS)
def test_alsd_select_replays_exactly(alsd_engine, tiny_enc, tiny_cfg, case):
    """The oracle's step applied to the engine's own log-probabilities and previous beam builds the engine's next beam at
    every step (same slots in order, sequences, token counts, alignment steps; scores to 1e-12 relative) and the engine's
    running best finished hypothesis; the output is that search's winner."""
    beam, returns_input, score_norm = case
    tr = _trace(alsd_engine, tiny_enc, case)
    enc_len = tiny_enc[1].cpu()
    steps = 0
    for b in range(len(_WAVES)):
        T = int(enc_len[b])
        steps += AC.replay(tr, b, T, beam, int(2.0 * T), score_norm, returns_input, tiny_cfg.blank)
    assert steps >= 100


def test_alsd_production_size_log_probabilities():
    """One clip at the production size (V = 3000, K = 1920 / 3840, the 128 x 64 GEMM instance): every row against float64,
    and the beam update replayed exactly."""
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    sd = random_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, "cuda:0", alsd=True)
    enc, enc_len = _encode(eng, [np.pad(synth_clip(61, 4.0), 8000)])
    tr = eng.alsd_trace(enc, enc_len, beam=4)
    worst, n_rows = _check_logps(tr, enc.cpu(), enc_len.cpu(), sd, cfg, 4)
    print(f"production size: {n_rows} rows, worst |log p - float64| {worst:.2e} (bar {AC.LP_BAR:.0e})")
    assert n_rows >= 100 and worst < AC.LP_BAR
    T = int(enc_len[0])
    AC.replay(tr, 0, T, 4, int(2.0 * T), True, True, cfg.blank)


def _crafted_engine(tiny_cfg, tiny_sd, token5_bias):
    from reazonspeech_b200.engine import Engine
    sd = AC.crafted_sd(tiny_sd, tiny_cfg, token5_bias)
    return Engine(tiny_cfg, sd, "cuda:0", alsd=True), sd


@pytest.mark.parametrize("T,beam,score_norm,tokens,score", AC.RECOMBINED_FINAL_CASES)
def test_alsd_recombined_final_matches_the_oracle(tiny_cfg, tiny_sd, T, beam, score_norm, tokens, score):
    """A finished hypothesis is ranked with the score recombination added into it in the step it finished (NeMo's `final`
    holds the beam's own object): the winner equals the oracle's on the crafted joint."""
    eng, sd = _crafted_engine(tiny_cfg, tiny_sd, 0.0)
    ref = alsd_beam(torch.zeros(T, tiny_cfg.d_model), sd, tiny_cfg, beam=beam, score_norm=score_norm)
    assert ref.tokens == tokens
    enc = torch.zeros(1, 8, tiny_cfg.d_model, device="cuda")
    y, steps, n, sc = [a.cpu() for a in eng.alsd(enc, torch.tensor([T], dtype=torch.int32, device="cuda"), beam=beam, score_norm=score_norm)]
    k = int(n[0])
    assert y[0, : k + 1].tolist() == ref.y_sequence
    assert AC.close(float(sc[0]), ref.score, 1e-5), (float(sc[0]), ref.score)
    AC.assert_valid_alignment(ref.tokens, steps[0, :k].tolist(), T)       # exactly tied duplicates may order differently


def test_alsd_u_max_is_rounded_in_double(tiny_cfg, tiny_sd):
    """u_max = int(1.16 * 25) = 28, as the oracle computes it (29 in float), on a joint that emits as much as u_max allows."""
    c = AC.U_MAX_CASE
    eng, sd = _crafted_engine(tiny_cfg, tiny_sd, c["token5_bias"])
    T = c["T"]
    ref = alsd_beam(torch.zeros(T, tiny_cfg.d_model), sd, tiny_cfg, beam=c["beam"], u_max_ratio=c["ratio"])
    enc = torch.zeros(1, 32, tiny_cfg.d_model, device="cuda")
    y, steps, n, sc = [a.cpu() for a in eng.alsd(enc, torch.tensor([T], dtype=torch.int32, device="cuda"), beam=c["beam"],
                                                 u_max_ratio=c["ratio"], U_cap=200)]
    k = int(n[0])
    assert k == len(ref.tokens) and y[0, : k + 1].tolist() == ref.y_sequence, (k, len(ref.tokens))
    assert AC.close(float(sc[0]), ref.score, 1e-5), (float(sc[0]), ref.score)
    AC.assert_valid_alignment(ref.tokens, steps[0, :k].tolist(), T)


@pytest.mark.parametrize("beam", [2, 8])
def test_alsd_batch_invariance(alsd_engine, tiny_enc, beam):
    """Each utterance decodes bit-identically alone (its own T_max) and inside the batch of five at two different positions."""
    enc, enc_len = tiny_enc
    B = enc.shape[0]
    U = 200

    def run(e, l):
        return [a.cpu() for a in alsd_engine.alsd(e.contiguous(), l.contiguous(), beam=beam, U_cap=U)]

    batched = []
    for shift in (0, 2):
        perm = [(j + shift) % B for j in range(B)]
        batched.append((perm, run(enc[perm], enc_len[perm])))
    for i in range(B):
        T = int(enc_len[i])
        Tp = (T + 7) // 8 * 8
        alone = run(enc[i : i + 1, :Tp], enc_len[i : i + 1])
        k = int(alone[2][0])
        for perm, (y, steps, n, sc) in batched:
            p = perm.index(i)
            assert int(n[p]) == k and y[p, : k + 1].tolist() == alone[0][0, : k + 1].tolist(), (i, p)
            assert steps[p, :k].tolist() == alone[1][0, :k].tolist() and float(sc[p]) == float(alone[3][0]), (i, p)


def test_alsd_edges_short_and_empty_utterances(alsd_engine, tiny_enc, tiny_cfg, tiny_sd):
    """Utterances of 1 and 2 frames in a batch with a long one equal the oracle; an empty one gives [blank], n = 0, score 0,
    as the oracle's search of no frame does."""
    enc, enc_len = tiny_enc
    long_i = int(enc_len.argmax())
    e = torch.stack([enc[long_i], enc[0], enc[1], enc[2]]).contiguous()
    lens = torch.tensor([int(enc_len[long_i]), 1, 2, 0], dtype=torch.int32, device="cuda")
    y, steps, n, sc = [a.cpu() for a in alsd_engine.alsd(e, lens, beam=4)]
    e = e.cpu()
    for b in range(4):
        T = int(lens[b])
        ref = alsd_beam(e[b, :T], tiny_sd, tiny_cfg, beam=4, emulate=True)
        k = int(n[b])
        assert y[b, : k + 1].tolist() == ref.y_sequence and steps[b, :k].tolist() == ref.timestamp, b
        assert abs(float(sc[b]) - ref.score) < 1e-3 * max(1.0, abs(ref.score)), b
    assert int(n[3]) == 0 and int(y[3, 0]) == tiny_cfg.blank and float(sc[3]) == 0.0


def test_alsd_u_cap_below_the_winners_length(alsd_engine, tiny_enc):
    """U_cap smaller than the winner's length: n is the full length, y / steps hold its first U_cap tokens."""
    enc, enc_len = tiny_enc
    full = [a.cpu() for a in alsd_engine.alsd(enc, enc_len, beam=4)]
    cap = 3
    assert int(full[2].min()) > cap
    y, steps, n, sc = [a.cpu() for a in alsd_engine.alsd(enc, enc_len, beam=4, U_cap=cap)]
    assert torch.equal(n, full[2]) and torch.equal(sc, full[3])
    assert torch.equal(y, full[0][:, : cap + 1]) and torch.equal(steps, full[1][:, :cap])


def test_alsd_trace_seam_arguments_and_agreement(alsd_engine, tiny_enc):
    """The seam returns rs_rnnt_alsd's results; max_steps limits what it records; bad trace buffers are rejected."""
    import ctypes as C
    from reazonspeech_b200.engine import RsAlsdTrace
    enc, enc_len = tiny_enc
    plain = [a.cpu() for a in alsd_engine.alsd(enc, enc_len, beam=4)]
    tr = alsd_engine.alsd_trace(enc, enc_len, beam=4, max_steps=5)
    assert tr["n_hyp"].shape[0] == 5
    for a, k in zip(plain, ("y", "steps", "n", "score")):
        assert torch.equal(a, tr[k]), k
    B, T, _ = enc.shape
    out = [torch.zeros(B, 3 * T + 2, dtype=torch.int32, device="cuda") for _ in range(3)] + [torch.zeros(B, dtype=torch.float64, device="cuda")]
    bad = RsAlsdTrace(1, 4, *([None] * 13))
    rc = alsd_engine.lib.rs_rnnt_alsd_trace(alsd_engine.h, enc.data_ptr(), enc_len.data_ptr(), B, T, 4, 2.0, 1, 1, out[0].data_ptr(),
                                            out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), 3 * T + 1, C.byref(bad), None)
    assert rc == -1 and b"trace" in alsd_engine.lib.rs_last_error(alsd_engine.h)
