"""Shared pieces of the ALSD beam-search tests (tests/test_alsd_cpu.py without a GPU, tests/test_gpu_alsd_trace.py on one):
the float64 log-probabilities of a hypothesis at a frame, the replay of the engine's per-step trace (rs_rnnt_alsd_trace)
through the oracle's own step (oracle/alsd_restated.py::alsd_step), and the crafted joints on which recombination and u_max
decide the winner."""
import math

import torch
import torch.nn.functional as F

from oracle import nemo_restated as O
from oracle.alsd_restated import BeamHyp, alsd_step

# max |log p - float64 reference| over the traced rows' blank and top-k log-probabilities (tests/test_gpu_alsd_trace.py).
# Measured on an H100 80GB HBM3 at 700 W: 3.9e-6 on the tiny model (beams 1-8), 2.7e-5 at the production size (V = 3000).
# The mis-implementations of tests/test_alsd_cpu.py err by 1.1e-2 or more.
LP_BAR = 2e-4


class Float64Joint:
    """log_softmax of the joint in float64 for a token sequence at a frame: the predictor run in float64 over the sequence
    (cached per prefix; SOS = the zero vector, as in the oracle) and joint.enc of the bf16-rounded encoder output, as the
    engine rounds it for its projection GEMM.  enc: float32 [T, d_model] of one utterance."""

    def __init__(self, enc, sd, cfg):
        self.sd = {k: v.double() for k, v in sd.items() if k.startswith(("decoder.", "joint."))}
        self.cfg = cfg
        self.ep = O.joint_enc_proj(enc.to(torch.bfloat16).double(), self.sd)
        hp = cfg.pred_hidden
        z = torch.zeros(hp, dtype=torch.float64)
        h, c = O.lstm_step(z, z, z, self.sd)
        self._cache = {(): (h, c, self._pp(h))}

    def _pp(self, h):
        return F.linear(h, self.sd["joint.pred.weight"], self.sd["joint.pred.bias"])

    def pred(self, toks):
        """(h, c, joint.pred) after feeding toks."""
        toks = tuple(toks)
        if toks not in self._cache:
            h, c, _ = self.pred(toks[:-1])
            h2, c2 = O.lstm_step(self.sd["decoder.prediction.embed.weight"][toks[-1]], h, c, self.sd)
            self._cache[toks] = (h2, c2, self._pp(h2))
        return self._cache[toks]

    def act(self, toks, t):
        return torch.relu(self.ep[t] + self.pred(toks)[2])

    def logits(self, act, b_out=True):
        return F.linear(act, self.sd["joint.joint_net.2.weight"], self.sd["joint.joint_net.2.bias"] if b_out else None)

    def logp(self, toks, t):
        return torch.log_softmax(self.logits(self.act(toks, t)), -1)

    def top(self, lp, k):
        """The k best non-blank classes, ties to the lower index (a stable sort of -lp)."""
        order = sorted(range(self.cfg.vocab_size), key=lambda j: -float(lp[j]))
        return order[:k]


def mutant_logps(J, toks, t):
    """log-probabilities of the same row under plausible mis-implementations of the engine, in float64."""
    blank = J.cfg.blank
    a = J.act(toks, t)
    lg = J.logits(a)
    nb = J.logits(a, b_out=False)
    return {
        "one bf16 activation term": torch.log_softmax(J.logits(a.to(torch.bfloat16).double()), -1),
        "b_out dropped": torch.log_softmax(nb, -1),
        "blank outside the log-sum-exp": lg - torch.logsumexp(torch.cat((lg[:blank], lg[blank + 1:])), -1),
        "frame t - 1": torch.log_softmax(J.logits(J.act(toks, max(t - 1, 0))), -1),
        "parent's predictor output": torch.log_softmax(J.logits(J.act(toks[:-1], t)), -1),
    }


def row_error(lp, ref, blank, toks):
    """max |lp - ref| over the blank and the classes toks."""
    return max(abs(float(lp[j]) - float(ref[j])) for j in [blank] + list(toks))


# ------------------------------------------------------------------------------------------------ the trace
def sequence(tr, b, node):
    """(tokens, alignment steps) of back-pointer node `node` of utterance b."""
    toks, steps = [], []
    while node > 0:
        toks.append(int(tr["node_tok"][b, node])); steps.append(int(tr["node_step"][b, node]))
        node = int(tr["node_parent"][b, node])
    assert node == 0
    return toks[::-1], steps[::-1]


def beams(tr, b, blank):
    """The beam each step starts from: [(slot, tokens, steps, score)] per step; step 0 starts from [blank] with score 0."""
    out = [[(0, [], [], 0.0)]]
    for i in range(tr["n_hyp"].shape[0]):
        out.append([(k, *sequence(tr, b, int(tr["beam_node"][i, b, k])), float(tr["beam_score"][i, b, k])) for k in range(int(tr["n_hyp"][i, b]))])
    return out


def scored_rows(tr, b, blank):
    """Every row the engine scored for utterance b: (step, slot, tokens, frame)."""
    rows = []
    for i, beam_i in enumerate(beams(tr, b, blank)[: tr["n_hyp"].shape[0]]):
        for k, toks, _, _ in beam_i:
            t = int(tr["row_t"][i, b, k])
            if t >= 0:
                rows.append((i, k, toks, t))
    return rows


def _rel(a, b):
    return abs(a - b) <= 1e-12 * max(1.0, abs(b))


def replay(tr, b, T, beam, u_max, score_norm, recombine_returns_input, blank):
    """Applies the oracle's step to the engine's own log-probabilities and previous beam at every step and asserts that it
    builds the engine's next beam (slots in order, sequences, token counts, alignment steps; scores to 1e-12 relative) and
    the engine's running best finished hypothesis.  Returns the number of steps replayed."""
    S = tr["n_hyp"].shape[0]
    prev = [BeamHyp([blank], 0.0, [-1], None)]
    final = []
    key = (lambda x: x.score / len(x.y)) if score_norm else (lambda x: x.score)
    i = 0
    for i in range(T + u_max):
        assert i < S, f"utt {b}: the engine stopped recording at step {S}, the search runs to {T + u_max}"
        rows = []
        for k, h in enumerate(prev):
            t = i - (len(h.y) - 1)
            rt = int(tr["row_t"][i, b, k])
            if t > T - 1:
                assert rt == -1, (i, k)
                rows.append(None)
                continue
            assert rt == t, (i, k, rt, t)
            lp = tr["cand_logp"][i, b, k]
            rows.append((float(lp[0]), [float(x) for x in lp[1:1 + beam]], [int(x) for x in tr["cand_tok"][i, b, k, :beam]], None))
        new = alsd_step(prev, rows, i, T, beam, recombine_returns_input, final)
        if new is None:                                           # nothing live: the engine keeps the beam it had
            new = prev
        assert int(tr["n_hyp"][i, b]) == len(new), (i, int(tr["n_hyp"][i, b]), len(new))
        for k, h in enumerate(new):
            toks, steps = sequence(tr, b, int(tr["beam_node"][i, b, k]))
            assert [blank] + toks == h.y and steps == h.timestamp[1:], (i, k)
            assert int(tr["beam_u"][i, b, k]) == len(toks)
            assert _rel(float(tr["beam_score"][i, b, k]), h.score), (i, k, float(tr["beam_score"][i, b, k]), h.score)
        assert int(tr["has_final"][i, b]) == (1 if final else 0), i
        if final:
            best = final[0]
            for f in final[1:]:
                if key(f) > key(best):
                    best = f
            assert _rel(float(tr["final_score"][i, b]), best.score) and _rel(float(tr["final_key"][i, b]), key(best)), \
                (i, float(tr["final_score"][i, b]), best.score)
        if new is prev:
            break
        prev = [BeamHyp(h.y, float(tr["beam_score"][i, b, k]), h.timestamp, None) for k, h in enumerate(new)]
    return i + 1


# ------------------------------------------------------------------------------------------------ crafted joints
def crafted_sd(sd, cfg, token5_bias=0.0):
    """The joint's output weight zeroed: every row's logits are the bias, 0 for blank, token5_bias for token 5 and distinct
    values near -30 for every other class, whatever the encoder and predictor say."""
    out = dict(sd)
    bias = -30.0 - 0.01 * torch.arange(cfg.vocab_size + 1, dtype=torch.float32)
    bias[cfg.blank] = 0.0
    bias[5] = token5_bias
    out["joint.joint_net.2.weight"] = torch.zeros_like(sd["joint.joint_net.2.weight"])
    out["joint.joint_net.2.bias"] = bias
    return out


# (T, beam, score_norm) -> the oracle's winner (tokens, score); the entries of `final` carry the score recombination added
# in the step they finished.  Recording them before recombination picks another winner (tests/test_alsd_cpu.py).
RECOMBINED_FINAL_CASES = [(2, 4, True, [5, 5], -1.3863), (2, 4, False, [5], -0.9808), (5, 4, True, [5] * 5, -2.8371)]

# u_max = int(ratio * T) in double is 28 here; the same product rounded in float is 29.  Token 5's bias a little above
# blank's makes the search emit as much as u_max allows.
U_MAX_CASE = dict(T=25, ratio=1.16, beam=4, token5_bias=0.2)


def assert_valid_alignment(tokens, steps, T):
    """Token j emitted at alignment step steps[j] = t + j with frames t non-decreasing in [0, T)."""
    frames = [s - j for j, s in enumerate(steps)]
    assert len(steps) == len(tokens) and frames == sorted(frames) and all(0 <= f < T for f in frames), frames


def close(a, b, tol):
    return math.isfinite(a) and abs(a - b) <= tol * max(1.0, abs(b))


def constant_row_search(sd, cfg, T, beam, u_max, score_norm=True, recombine_returns_input=True, final_aliases_beam=True):
    """The oracle's search (alsd_step) on a crafted joint, where every row has the same log-probabilities -> (tokens, score)
    of the winner.  final_aliases_beam=False records finished hypotheses before recombination."""
    blank = cfg.blank
    lp = torch.log_softmax(sd["joint.joint_net.2.bias"], -1)
    top = torch.cat((lp[:blank], lp[blank + 1:])).topk(beam)
    row = (float(lp[blank]), top.values.tolist(), [k + (1 if k >= blank else 0) for k in top.indices.tolist()], None)
    B, final = [BeamHyp([blank], 0.0, [-1], None)], []
    for i in range(T + u_max):
        nxt = alsd_step(B, [row] * len(B), i, T, beam, recombine_returns_input, final, final_aliases_beam)
        if nxt is None:
            break
        B = nxt
    key = (lambda x: x.score / len(x.y)) if score_norm else (lambda x: x.score)
    best = sorted(final or B, key=key, reverse=True)[0]
    return best.y[1:], best.score
