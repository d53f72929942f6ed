"""ALSD beam search without a GPU: the log-probability bar of tests/test_gpu_alsd_trace.py against the error of plausible
mis-implementations, and the two places where the search departs from the oracle (oracle/alsd_restated.py) unless it keeps
NeMo's rules: a finished hypothesis carries the score recombination adds into it, and u_max = int(ratio * T) in double."""
import numpy as np
import pytest
import torch

import alsd_cases as AC
from oracle.alsd_restated import alsd_beam


@pytest.mark.parametrize("full", [False, True])
def test_lp_bar_separates_mis_implementations(full, tiny_cfg, tiny_sd):
    """LP_BAR lies at least 3x below the error of: one bf16 activation term instead of three, b_out dropped, the blank left out
    of the log-sum-exp, frame t - 1, and an extension scored with its parent's predictor output -- on the rows (every prefix
    of a token sequence at every frame) of a random encoder output; the engine's own three-term split stays far below it."""
    if full:
        from reazonspeech_b200.config import ModelConfig
        from reazonspeech_b200.weights import random_state_dict
        cfg = ModelConfig(); sd = random_state_dict(cfg, seed=0)
    else:
        cfg, sd = tiny_cfg, tiny_sd
    g = torch.Generator().manual_seed(5)
    T, U, k = 10, 6, 8
    enc = torch.randn(T, cfg.d_model, generator=g)
    labels = [int(x) for x in torch.randint(0, cfg.vocab_size, (U,), generator=g)]
    J = AC.Float64Joint(enc, sd, cfg)
    worst = {}
    three_terms = 0.0
    for u in range(U + 1):
        toks = labels[:u]
        for t in range(T):
            ref = J.logp(toks, t)
            top = J.top(ref, k)
            for name, lp in AC.mutant_logps(J, toks, t).items():
                worst[name] = max(worst.get(name, 0.0), AC.row_error(lp, ref, cfg.blank, top))
            a = J.act(toks, t)
            hi = a.float().to(torch.bfloat16).double()
            mid = (a.float() - hi.float()).to(torch.bfloat16).double()
            lo = (a.float() - hi.float() - mid.float()).to(torch.bfloat16).double()
            split = torch.log_softmax(J.logits(hi + mid + lo), -1)
            three_terms = max(three_terms, AC.row_error(split, ref, cfg.blank, top))
    print({n: f"{e:.2e}" for n, e in worst.items()}, f"three terms {three_terms:.2e}")
    for name, e in worst.items():
        assert 3 * AC.LP_BAR <= e, f"{name}: error {e:.2e}"
    assert three_terms < AC.LP_BAR / 10


@pytest.mark.parametrize("T,beam,score_norm,tokens,score", AC.RECOMBINED_FINAL_CASES)
def test_recombined_final_decides_the_winner(tiny_cfg, tiny_sd, T, beam, score_norm, tokens, score):
    """On the crafted joint the oracle's winner is a finished hypothesis whose score recombination raised in the step it
    finished; ranking finished hypotheses by their score before recombination picks another winner."""
    sd = AC.crafted_sd(tiny_sd, tiny_cfg)
    u_max = int(2.0 * T)
    ref = alsd_beam(torch.zeros(T, tiny_cfg.d_model), sd, tiny_cfg, beam=beam, score_norm=score_norm)
    assert ref.tokens == tokens and abs(ref.score - score) < 1e-4
    assert AC.constant_row_search(sd, tiny_cfg, T, beam, u_max, score_norm) == (ref.tokens, ref.score)
    before = AC.constant_row_search(sd, tiny_cfg, T, beam, u_max, score_norm, final_aliases_beam=False)
    assert before[0] != ref.tokens


def test_u_max_rounding_decides_the_winner(tiny_cfg, tiny_sd):
    """u_max = int(1.16 * 25) is 28 in double and 29 in float, and on the crafted joint the winner depends on it."""
    c = AC.U_MAX_CASE
    T, ratio = c["T"], c["ratio"]
    assert int(ratio * T) == 28 and int(np.float32(ratio) * np.float32(T)) == 29
    sd = AC.crafted_sd(tiny_sd, tiny_cfg, c["token5_bias"])
    enc = torch.zeros(T, tiny_cfg.d_model)
    r28 = alsd_beam(enc, sd, tiny_cfg, beam=c["beam"], u_max_ratio=ratio)
    r29 = alsd_beam(enc, sd, tiny_cfg, beam=c["beam"], u_max_ratio=29.5 / T)
    assert int(29.5 / T * T) == 29
    assert r28.tokens != r29.tokens
    assert AC.constant_row_search(sd, tiny_cfg, T, c["beam"], 28) == (r28.tokens, r28.score)
