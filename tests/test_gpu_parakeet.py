"""The sm_90a engine against the third-party Parakeet vectors (tests/golden/parakeet_cases.npz):
log-mel frontend and FastConformer encoder, through the C ABI, no oracle in between.

Tolerances: normalised log-mel max-abs 2e-3 (fp32 FFT in a different order; log of near-silent bins);
encoder output relative L2 2e-2 (bf16 GEMM operands and bf16 activation storage against an fp32
evaluation; SURVEY.md A.6)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_parakeet_golden as G  # noqa: E402

from reazonspeech_b200.engine import Engine  # noqa: E402
from reazonspeech_b200.weights import random_state_dict  # noqa: E402


@pytest.mark.parametrize("case", G.CASES, ids=[c[0] for c in G.CASES])
def test_engine_matches_parakeet_vectors(case):
    name, kw, wseed, cseed, secs = case
    z = np.load(G.OUT)
    cfg = G.case_config(kw)
    sd = random_state_dict(cfg, seed=wseed, calibrate=False)
    eng = Engine(cfg, sd, "cuda:0")
    wave = G.padded_clip(cseed, secs)
    # the clip rides in a padded batch next to a longer one: padding must not leak into it
    other = G.padded_clip(cseed + 100, secs + 1.3)
    L = max(len(wave), len(other))
    x = torch.zeros(2, L)
    x[0, : len(wave)] = torch.from_numpy(wave)
    x[1, : len(other)] = torch.from_numpy(other)
    lens = torch.tensor([len(wave), len(other)], dtype=torch.int32)
    mel, mel_len = eng.log_mel(x.cuda(), lens.cuda())
    enc, enc_len = eng.encode(mel, mel_len)
    torch.cuda.synchronize()
    feats, n, ref = z[name + ".features"], int(z[name + ".n_frames"]), z[name + ".encoder"]
    assert int(mel_len[0]) == n
    err = np.abs(mel[0, :n].cpu().numpy() - feats[:n]).max()
    assert mel[0, n: feats.shape[0]].abs().max().item() == 0.0
    T = ref.shape[0]
    assert int(enc_len[0]) == T
    got = enc[0, :T].cpu().numpy()
    rel = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    print(f"{name}: log-mel max-abs {err:.3e}, encoder rel-L2 {rel:.3e}")
    assert err < 2e-3
    assert rel < 2e-2
