"""ALSD N-best lists without a GPU: the insertion rule of alsd_select_kernel against Python's stable sort, NeMo's whole sorted
`final` list of the crafted constant-row joints written down, a search in which nothing finishes, and the host packing of
``Engine.alsd_nbest``'s arrays into ``Hypothesis`` / ``TranscribeResult`` lists on a stub engine."""
import contextlib
import ctypes as C
import importlib
import random

import numpy as np
import pytest
import torch

import alsd_cases as AC
import alsd_nbest_cases as NC

T = importlib.import_module("reazonspeech_b200.nemo.asr.transcribe")     # the package exports a FUNCTION of the same name


# ------------------------------------------------------------------------------------------------ the insertion rule
@pytest.mark.parametrize("seed", range(6))
def test_insertion_rule_is_a_stable_sort_truncated(seed):
    """Entries inserted one by one as the kernel inserts them equal sorted(pool, key, reverse=True)[:N], the same objects in
    the same order, on append streams with many equal keys; N = 1, N < |pool|, N = |pool| and N > |pool|."""
    g = random.Random(seed)
    for _ in range(50):
        n = g.randint(1, 40)
        levels = [g.uniform(-5, 0) for _ in range(g.randint(1, 4))]           # few distinct keys: ties everywhere
        pool = [(g.choice(levels), object()) for _ in range(n)]
        for N in sorted({1, max(1, n // 2), n, n + 3, 64}):
            held = []
            for key, item in pool:
                NC.insert(held, key, item, N)
            want = sorted(pool, key=lambda p: p[0], reverse=True)[:N]
            assert [id(it) for _, it in held] == [id(it) for _, it in want], (n, N)


# ------------------------------------------------------------------------------------------------ crafted joints
# NeMo's whole sorted `final` list of each crafted case: (tokens, score to 4 decimals) best first.  Duplicates of a sequence
# stay (e.g. [5] at -0.9808 and at -2.0794).  Scores below are the oracle's on the tiny model's crafted joint.
_F5 = lambda k: [5] * k                                                        # noqa: E731
EXPECTED = {
    "recombined-T2-norm": [(_F5(2), -1.3863), (_F5(3), -1.8563), (_F5(4), -2.3671), (_F5(1), -0.9808), (_F5(4), -4.1589),
                           (_F5(3), -3.4657), (_F5(2), -2.7726), (_F5(1), -2.0794), ([], -1.3863)],
    "recombined-T2-raw": [(_F5(1), -0.9808), ([], -1.3863), (_F5(2), -1.3863), (_F5(3), -1.8563), (_F5(1), -2.0794),
                          (_F5(4), -2.3671), (_F5(2), -2.7726), (_F5(3), -3.4657), (_F5(4), -4.1589)],
    "recombined-T5-norm": [(_F5(5), -2.8371), (_F5(6), -3.3342), (_F5(4), -2.3882), (_F5(7), -3.8634), (_F5(8), -4.4158),
                           (_F5(9), -4.9856), (_F5(10), -5.5689), (_F5(3), -2.5007), (_F5(10), -7.8323), (_F5(9), -7.1391),
                           (_F5(8), -6.446), (_F5(7), -5.7528), (_F5(6), -5.0597), (_F5(5), -4.3665), (_F5(4), -3.6734),
                           (_F5(3), -3.4657), (_F5(2), -2.7726), (_F5(1), -3.0603)],
    "u_max": [(_F5(28), -12.6819), (_F5(27), -12.2798), (_F5(26), -11.9257), (_F5(25), -11.6511), (_F5(24), -11.5341),
              (_F5(25), -12.6135), (_F5(26), -13.2116), (_F5(27), -13.8098), (_F5(23), -11.8984), (_F5(28), -14.4079),
              (_F5(24), -12.4966)],
    "fallback-beam1": [(_F5(5), -0.0336)],
    "fallback-beam4": [(_F5(5), -0.0336), (_F5(4), -2.9541), (_F5(4), -5.0336), (_F5(4), -5.0336)],
}


def _crafted(tiny_sd, tiny_cfg, case):
    name, Tn, beam, ratio, score_norm, bias = case
    sd = AC.crafted_sd(tiny_sd, tiny_cfg, bias)
    pool, from_final = NC.constant_row_pool(sd, tiny_cfg, Tn, beam, int(ratio * Tn))
    return name, pool, from_final, score_norm


@pytest.mark.parametrize("case", NC.crafted_cases(), ids=[c[0] for c in NC.crafted_cases()])
def test_crafted_final_lists(tiny_cfg, tiny_sd, case):
    """The oracle's whole `final` of each crafted joint, ranked, is the list written down above; the kernel's rule applied to
    it in append order gives its first 4 and all of it at N = 64; the winner is alsd_cases' expected winner."""
    name, pool, from_final, score_norm = _crafted(tiny_sd, tiny_cfg, case)
    full = NC.ranked(pool, score_norm)
    assert [(h.y[1:], round(h.score, 4)) for h in full] == EXPECTED[name]
    assert from_final == (not name.startswith("fallback"))
    key = NC.key_fn(score_norm)
    for N in (4, 64):
        held = []
        for h in pool:
            NC.insert(held, key(h), h, N)
        assert [h for _, h in held] == full[:N]
    for Tn, beam, sn, tokens, score in AC.RECOMBINED_FINAL_CASES:
        if name == f"recombined-T{Tn}-{'norm' if sn else 'raw'}":
            assert full[0].y[1:] == tokens and abs(full[0].score - score) < 1e-4


def test_crafted_lists_hold_duplicates_and_exceed_four(tiny_cfg, tiny_sd):
    """The lists the GPU tests compare against are long enough for N = 4 to cut them (9, 9, 18 and 11 entries), and the same
    sequence appears in them twice with different scores."""
    sizes = {}
    for case in NC.crafted_cases():
        name, pool, from_final, _ = _crafted(tiny_sd, tiny_cfg, case)
        sizes[name] = len(pool)
    assert [sizes[c[0]] for c in NC.crafted_cases()[:4]] == [9, 9, 18, 11]
    _, pool, _, _ = _crafted(tiny_sd, tiny_cfg, NC.crafted_cases()[1])
    assert sorted(round(h.score, 4) for h in pool if h.y[1:] == [5]) == [-2.0794, -0.9808]


# ------------------------------------------------------------------------------------------------ the C ABI without a GPU
def test_nbest_rejects_bad_arguments_before_any_launch():
    """n_best outside 1..RS_MAX_NBEST (and missing list-size buffers) is RS_ERR_INVALID_ARG, decided before the engine or
    the GPU is touched."""
    from reazonspeech_b200 import engine as E
    lib = E.load_library()
    buf = (C.c_int32 * 8)()
    p = C.cast(buf, C.c_void_p)
    for n_best, counts in ((0, p), (E.MAX_NBEST + 1, p), (4, None)):
        rc = lib.rs_rnnt_alsd_nbest(None, p, p, 1, 1, 4, 2.0, 1, 1, n_best, p, p, p, p, counts, counts, counts, 1, None)
        assert rc == -1
        assert b"rs_rnnt_alsd_nbest" in lib.rs_last_error(None)


# ------------------------------------------------------------------------------------------------ host packing
class _Cfg:
    blank = 50
    vocab_size = 50


class _Tok:
    def ids_to_text(self, ids):
        return "".join(chr(0x3042 + i) for i in ids)


class NbestStubEngine:
    """Engine stand-in on the CPU: 'encodes' a batch into frames whose count is the utterance's sample count / 1000, and returns
    for each utterance min(n_best, 1 + its frame count % 3) entries; entry e has e + 2 tokens (token j = 10 + e + j at
    step 2 j + 1) and score -e - 0.5.  ``align`` returns log-likelihood = -(frames * 1000 + sum of the labels)."""
    device = "cpu"

    def __init__(self):
        self.cfg = _Cfg()
        self.align_rows = []
        self.nbest_calls = []

    def log_mel(self, x, lens):
        return x, lens

    def encode(self, mel, mel_len):
        frames = (mel_len // 1000).to(torch.int32)
        Tm = int(frames.max())
        return torch.arange(mel.shape[0], dtype=torch.float32)[:, None, None].expand(-1, Tm, 2).contiguous(), frames

    def alsd_nbest(self, enc, enc_len, n_best, beam=4, U_cap=None):
        self.nbest_calls.append((enc.shape[0], n_best, beam))
        B, U = enc.shape[0], U_cap or 12
        y = torch.zeros(B, n_best, U + 1, dtype=torch.int32)
        steps = torch.zeros(B, n_best, U, dtype=torch.int32)
        n = torch.zeros(B, n_best, dtype=torch.int32)
        score = torch.zeros(B, n_best, dtype=torch.float64)
        count = torch.zeros(B, dtype=torch.int32)
        for r in range(B):
            c = min(n_best, 1 + int(enc_len[r]) % 3)
            count[r] = c
            for e in range(c):
                k = e + 2
                n[r, e] = k
                score[r, e] = -e - 0.5
                y[r, e, 0] = self.cfg.blank
                for j in range(min(k, U)):
                    y[r, e, 1 + j] = 10 + e + j
                    steps[r, e, j] = 2 * j + 1
        return y, steps, n, score, count, count.clone() + 5, torch.ones(B, dtype=torch.int32)

    def align(self, enc, enc_len, labels, label_len):
        self.align_rows.append(enc.shape[0])
        ll = [-(float(enc_len[j]) * 1000 + float(labels[j, : int(label_len[j])].sum())) for j in range(enc.shape[0])]
        B = enc.shape[0]
        return torch.zeros(B, 1), torch.zeros(B, 1), torch.zeros(B), torch.tensor(ll, dtype=torch.float32)


def test_nbest_hypotheses_packing():
    """Leading blank, alignment steps as timestamp, best first, only count[b] entries, and U_cap truncation: n is the full
    length, the hypothesis holds the first U_cap tokens (as transcribe_alsd does)."""
    eng = NbestStubEngine()
    enc = torch.zeros(3, 4, 2)
    y, steps, n, score, count, _, _ = eng.alsd_nbest(enc, torch.tensor([3, 4, 5], dtype=torch.int32), 3, U_cap=2)
    lists = T.nbest_hypotheses(y, steps, n, score, count)
    assert [len(h) for h in lists] == [1, 2, 3]
    h = lists[2][2]                                    # 4 tokens, U_cap 2
    assert h.y_sequence.tolist() == [50, 12, 13] and h.timestamp == [1, 3] and h.score == -2.5
    assert h.y_sequence.dtype == torch.long and h.log_likelihood is None
    assert [x.score for x in lists[2]] == [-0.5, -1.5, -2.5]
    assert lists[0][0].y_sequence.tolist() == [50, 10, 11] and lists[0][0].timestamp == [1, 3]


@pytest.fixture
def no_cuda_device(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device", contextlib.nullcontext)


def _clips(n, seed=0):
    g = np.random.default_rng(seed)
    return [g.standard_normal(int(g.integers(2000, 40000))).astype(np.float32) * 0.1 for _ in range(n)]


def test_transcribe_alsd_nbest_batches_and_log_likelihood(no_cuda_device):
    """Batches of at most max_batch by length, lists back in input order, and with log_likelihood every candidate aligned on
    its own utterance's encoder rows (index_select) in chunks of at most max_batch rows."""
    eng = NbestStubEngine()
    model = T.B200RnntModel(eng, _Tok(), max_batch=3, decoding="alsd", beam_size=2)
    clips = _clips(7, seed=5)
    lists = model.transcribe_alsd_nbest(clips, 2, log_likelihood=True)
    assert [c[0] for c in eng.nbest_calls] == [3, 3, 1] and all(c[1:] == (2, 2) for c in eng.nbest_calls)
    assert all(r <= 3 for r in eng.align_rows) and sum(eng.align_rows) == sum(len(h) for h in lists)
    for w, hyps in zip(clips, lists):
        frames = len(w) // 1000
        assert 1 <= len(hyps) <= 2
        for h in hyps:
            assert h.log_likelihood == float(np.float32(-(frames * 1000 + sum(h.y_sequence.tolist()[1:]))))
    plain = model.transcribe_alsd_nbest(clips, 2)
    assert all(h.log_likelihood is None for hyps in plain for h in hyps)
    assert [[h.y_sequence.tolist() for h in hyps] for hyps in plain] == [[h.y_sequence.tolist() for h in hyps] for hyps in lists]


def test_transcribe_nbest_batch_results(no_cuda_device):
    """Every candidate goes through the unchanged decode_hypothesis, best first, with result.hypothesis set."""
    from reazonspeech_b200.nemo.asr import audio_from_numpy, transcribe_nbest, transcribe_nbest_batch
    from reazonspeech_b200.nemo.asr.decode import decode_hypothesis
    eng = NbestStubEngine()
    model = T.B200RnntModel(eng, _Tok(), max_batch=4, decoding="alsd")
    audios = [audio_from_numpy(w, 16000) for w in _clips(5, seed=6)]
    res = transcribe_nbest_batch(model, audios, 3)
    assert len(res) == 5
    for rs in res:
        assert 1 <= len(rs) <= 3
        assert [r.hypothesis.score for r in rs] == sorted((r.hypothesis.score for r in rs), reverse=True)
        for r in rs:
            d = decode_hypothesis(model, r.hypothesis)
            assert r.text == d.text and r.subwords == d.subwords and r.segments == d.segments
    one = transcribe_nbest(model, audios[0], 3)
    assert [r.text for r in one] == [r.text for r in res[0]]


def test_transcribe_nbest_batch_argument_errors(no_cuda_device):
    """A greedy model, the multi-GPU model or n_best outside 1..64 raise ValueError before the engine is called."""
    from reazonspeech_b200.nemo.asr import audio_from_numpy, transcribe_nbest_batch
    from reazonspeech_b200.nemo.asr.multi_gpu import MultiGpuRnntModel
    audios = [audio_from_numpy(np.zeros(16000, np.float32), 16000)]
    eng = NbestStubEngine()
    greedy = T.B200RnntModel(eng, _Tok())
    with pytest.raises(ValueError, match="load_model"):
        transcribe_nbest_batch(greedy, audios, 4)
    multi = MultiGpuRnntModel.__new__(MultiGpuRnntModel)
    with pytest.raises(ValueError, match="load_model"):
        transcribe_nbest_batch(multi, audios, 4)
    alsd = T.B200RnntModel(eng, _Tok(), decoding="alsd")
    for bad in (0, 65, -1, 2.0, True, None):
        with pytest.raises(ValueError, match="n_best"):
            transcribe_nbest_batch(alsd, audios, bad)
    assert eng.nbest_calls == []
