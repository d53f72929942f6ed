"""MAES beam search on the GPU (rs_rnnt_maes, csrc/decode_maes.cu) against its CPU oracle (oracle/maes_restated.py: NeMo's
modified_adaptive_expansion_search restated) on the SAME encoder output, with and without an n-gram LM.  Both evaluate
log-probabilities to fp32 accuracy, so the kept hypotheses must agree; a different winner is admissible only as a near-tie of the
ranking key, at most one utterance per case."""
import dataclasses

import numpy as np
import pytest
import torch

from ngram_oracle import ArpaOracle, write_arpa

pytestmark = pytest.mark.gpu

ALPHA = 0.1
LENS = [37, 1, 6, 23, 0, 13, 2, 31]


@pytest.fixture(scope="module")
def maes_engine(tiny_cfg, tiny_sd):
    from reazonspeech_b200.engine import Engine
    return Engine(tiny_cfg, tiny_sd, "cuda:0", alsd=True)


@pytest.fixture(scope="module")
def tiny_lm(tmp_path_factory, tiny_cfg):
    path = str(tmp_path_factory.mktemp("lm") / "tiny3.arpa")
    write_arpa(path, tiny_cfg.vocab_size, 3, n_sentences=200, seed=7)
    return path


def _tiny_enc(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    enc = torch.randn(len(lens), max(lens), cfg.d_model, generator=g)
    for b, n in enumerate(lens):
        enc[b, n:] = 0
    return enc, torch.tensor(lens, dtype=torch.int32)


def _set_lm(eng, cfg, path):
    from reazonspeech_b200.ngram_lm import NgramLMConfig, build_lm_tables
    eng.set_ngram_lm(None if path is None else build_lm_tables(NgramLMConfig(path, ALPHA), cfg.vocab_size))


def _run(eng, enc, lens, **kw):
    return [a.cpu() for a in eng.maes(enc.cuda().contiguous(), lens.cuda(), **kw)]


def _oracle(enc, lens, sd, cfg, lm_path, **kw):
    from oracle.maes_restated import maes_beam
    lm = None if lm_path is None else ArpaOracle(lm_path, cfg.vocab_size, ALPHA)
    fn = None if lm is None else (lambda s, k: (lm.score(s, k), lm.next(s, k)))
    return [maes_beam(enc[b, :int(lens[b])], sd, cfg, lm=fn, lm_start=None if lm is None else lm.start, emulate=True, **kw)
            for b in range(enc.shape[0])]


def _compare(got, refs, score_norm, tag):
    """-> utterances whose whole N-best list equals the oracle's; asserts the winner bar."""
    y, frames, n, score, count = got
    same_best = same_list = 0
    for b, ref in enumerate(refs):
        key = lambda s, ln: s / ln if score_norm else s
        k = int(n[b, 0])
        gy, gf = y[b, 0, : k + 1].tolist(), frames[b, 0, :k].tolist()
        print(f"{tag} b={b}: {k} tokens (oracle {len(ref.tokens)}), score {float(score[b, 0]):.4f} (oracle {ref.score:.4f}), "
              f"count {int(count[b])} (oracle {len(ref.nbest)})")
        if gy == ref.y_sequence and gf == ref.frames:
            same_best += 1
            assert abs(float(score[b, 0]) - ref.score) < 1e-3 * max(1.0, abs(ref.score)), tag
        else:
            assert abs(key(float(score[b, 0]), k + 1) - key(ref.score, len(ref.y_sequence))) < 1e-3, (tag, b, gy[:12], ref.y_sequence[:12])
        N = min(y.shape[1], len(ref.nbest))
        ok = int(count[b]) == N
        for e in range(N if ok else 0):
            h, ke = ref.nbest[e], int(n[b, e])
            ok &= y[b, e, : ke + 1].tolist() == h.y and frames[b, e, :ke].tolist() == h.timestamp[1:]
            ok &= abs(float(score[b, e]) - h.score) < 1e-3 * max(1.0, abs(h.score))
        same_list += ok
    assert same_best >= len(refs) - 1, f"{tag}: {same_best} of {len(refs)} winners equal"
    return same_list


# (beam, num_steps, prefix_alpha, expansion_beta, score_norm, recombine_returns_input): every value of each parameter, each
# switch both ways, within the row limit (beam 8 at num_steps 3 exceeds it)
_CASES = [(1, 2, 0, 0, True, True), (1, 3, 1, 2, False, True), (2, 2, 1, 2, True, False), (2, 3, 2, 0, True, True),
          (4, 2, 1, 2, True, True), (4, 2, 2, 2, False, False), (4, 3, 0, 2, True, True), (4, 3, 2, 0, True, False),
          (8, 2, 1, 2, True, True), (8, 2, 0, 0, False, True), (8, 2, 2, 2, True, False)]


@pytest.mark.parametrize("with_lm", [False, True], ids=["no-lm", "lm"])
@pytest.mark.parametrize("beam,steps,alpha,beta,score_norm,rri", _CASES, ids=["-".join(str(v) for v in c) for c in _CASES])
def test_maes_matches_the_oracle(maes_engine, tiny_cfg, tiny_sd, tiny_lm, beam, steps, alpha, beta, score_norm, rri, with_lm):
    enc, lens = _tiny_enc(tiny_cfg, LENS, seed=31)
    kw = dict(beam=beam, num_steps=steps, prefix_alpha=alpha, expansion_beta=beta, score_norm=score_norm, recombine_returns_input=rri)
    path = tiny_lm if with_lm else None
    _set_lm(maes_engine, tiny_cfg, path)
    try:
        got = _run(maes_engine, enc, lens, n_best=beam, **kw)
    finally:
        _set_lm(maes_engine, tiny_cfg, None)
    refs = _oracle(enc, lens, tiny_sd, tiny_cfg, path, **kw)
    same_list = _compare(got, refs, score_norm, f"maes {beam}/{steps}/{alpha}/{beta}" + (" lm" if with_lm else ""))
    assert same_list >= len(refs) - 1
    assert int(got[4][4]) == 1 and got[0][4, 0, 0].item() == tiny_cfg.blank and float(got[3][4, 0]) == 0.0   # enc_len 0: [blank], 0


def test_beam_one_equals_greedy_with_max_symbols(maes_engine, tiny_cfg, tiny_sd):
    """beam 1, beta 0: one candidate per round -- a blank ends the frame, a token is kept -- so num_steps = S is greedy decoding
    with max_symbols = S."""
    from reazonspeech_b200.engine import Engine
    enc, lens = _tiny_enc(tiny_cfg, [40, 17, 3, 29], seed=5)
    enc = enc * 0.3                                   # flatter joints: several tokens per frame happen
    for S in (2, 3):
        greedy = Engine(dataclasses.replace(tiny_cfg, max_symbols=S), tiny_sd, "cuda:0")
        tk, fr, nt = [a.cpu() for a in greedy.greedy(enc.cuda().contiguous(), lens.cuda())]
        y, frames, n, _, _ = _run(maes_engine, enc, lens, beam=1, num_steps=S, prefix_alpha=1, expansion_beta=0)
        for b in range(len(lens)):
            k = int(nt[b])
            assert int(n[b, 0]) == k and y[b, 0, 1 : k + 1].tolist() == tk[b, :k].tolist(), (S, b)
            assert frames[b, 0, :k].tolist() == fr[b, :k].tolist(), (S, b)
        del greedy


def test_the_lm_changes_winners_and_clearing_it_restores(maes_engine, tiny_cfg, tiny_lm):
    enc, lens = _tiny_enc(tiny_cfg, LENS, seed=32)
    plain = _run(maes_engine, enc, lens, n_best=4)
    _set_lm(maes_engine, tiny_cfg, tiny_lm)
    fused = _run(maes_engine, enc, lens, n_best=4)
    _set_lm(maes_engine, tiny_cfg, None)
    again = _run(maes_engine, enc, lens, n_best=4)
    assert all(torch.equal(a, b) for a, b in zip(plain, again))
    changed = sum(plain[0][b, 0].tolist() != fused[0][b, 0].tolist() for b in range(len(LENS)))
    print(f"the LM changed {changed} of {len(LENS)} winners")
    assert changed >= 1
    rows, frames = maes_engine.maes_last_rows()
    assert frames == max(LENS) and rows > 0


def test_rejections_before_any_launch(maes_engine, tiny_cfg):
    enc, lens = _tiny_enc(tiny_cfg, [5, 3], seed=1)
    for kw, code in ((dict(beam=9), -1), (dict(beam=0), -1), (dict(num_steps=1), -1), (dict(num_steps=5), -1), (dict(prefix_alpha=-1), -1),
                     (dict(prefix_alpha=5), -1), (dict(expansion_beta=5), -1), (dict(expansion_gamma=0.0), -1),
                     (dict(expansion_gamma=float("inf")), -1), (dict(beam=2, n_best=3), -1), (dict(n_best=0), -1),
                     (dict(beam=8, num_steps=3, expansion_beta=2), -5), (dict(beam=4, num_steps=4, expansion_beta=2), -5)):
        with pytest.raises(RuntimeError, match=rf"rs_rnnt_maes failed \({code}\)"):
            _run(maes_engine, enc, lens, **kw)
    y, *_ = _run(maes_engine, enc, lens, beam=8, num_steps=2, expansion_beta=2)       # 8 * 10^2 = 800 rows: admitted
    assert y.shape[0] == 2


def test_full_size_against_the_oracle():
    """The 619 M synthetic model at the bench geometry (30 s clips): two clips at beam 4 with NeMo's defaults."""
    from reazonspeech_b200.config import ModelConfig
    from reazonspeech_b200.engine import Engine
    from reazonspeech_b200.synth import synth_clip
    from reazonspeech_b200.weights import random_state_dict
    cfg = ModelConfig()
    sd = random_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, "cuda:0", alsd=True)
    waves = [np.pad(synth_clip(i, 30.0), 8000) for i in range(2)]
    x = torch.from_numpy(np.stack(waves)).float().cuda()
    lens = torch.full((2,), len(waves[0]), dtype=torch.int32).cuda()
    enc, enc_len = eng.encode(*eng.log_mel(x, lens))
    got = [a.cpu() for a in eng.maes(enc, enc_len, beam=4, n_best=4)]
    refs = _oracle(enc.cpu(), enc_len.cpu(), sd, cfg, None, beam=4)
    _compare(got, refs, True, "619M")
