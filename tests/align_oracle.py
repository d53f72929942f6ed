"""Float64 restatement of forced alignment on the RNN-T lattice (reazonspeech_b200/alignment.py states the contract):
the lattice from oracle/nemo_restated.py's predictor and joint, the forward / Viterbi recursions with the backtrace, and a
brute-force enumeration of every lattice path that pins the recursions on small shapes."""
import itertools
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
import nemo_restated as O  # noqa: E402


def predictor(labels, sd, cfg):
    """Teacher-forced predictor (the greedy loop's SOS step, then one lstm_step per label) -> h, pred_proj float32
    [U + 1, Hp / Hj]: row u is the state after feeding y_1..y_u."""
    hp = cfg.pred_hidden
    emb = sd["decoder.prediction.embed.weight"]
    h = torch.zeros(hp); c = torch.zeros(hp)
    hs = []
    for u in range(len(labels) + 1):
        x = torch.zeros(hp) if u == 0 else emb[int(labels[u - 1])]
        h, c = O.lstm_step(x, h, c, sd)
        hs.append(h)
    H = torch.stack(hs)
    return H, F.linear(H, sd["joint.pred.weight"], sd["joint.pred.bias"])


def enc_proj(enc, sd, bf16_input=True):
    """joint.enc of every frame; bf16_input rounds the encoder output to bf16 first, as the engine's projection GEMM does."""
    x = enc.to(torch.bfloat16).float() if bf16_input else enc
    return O.joint_enc_proj(x, sd)


def joint_logits(ep, pp, sd, dtype=torch.float64, b_out=True):
    """[T, U + 1, V + 1] joint logits of every cell from enc_proj [T, Hj] and pred_proj [U + 1, Hj]."""
    W, b = sd["joint.joint_net.2.weight"].to(dtype), sd["joint.joint_net.2.bias"].to(dtype)
    a = torch.relu(ep.to(dtype)[:, None, :] + pp.to(dtype)[None, :, :])
    return a @ W.T + (b if b_out else 0)


def lattice_from_logits(logits, labels, blank):
    """-> lp_blank [T, U + 1], lp_emit [T, U + 1] (lp_emit[:, U] = -inf) float64 numpy."""
    lsm = torch.log_softmax(logits.to(torch.float64), dim=-1)
    U = len(labels)
    lpb = lsm[:, :, blank].numpy()
    lpe = np.full(lpb.shape, -np.inf)
    for u in range(U):
        lpe[:, u] = lsm[:, u, int(labels[u])].numpy()
    return lpb, lpe


def lattice(enc, labels, sd, cfg, T=None):
    """The float64 lattice of one utterance from its encoder output [T, d_model] and labels."""
    T = enc.shape[0] if T is None else T
    _, pp = predictor(labels, sd, cfg)
    return lattice_from_logits(joint_logits(enc_proj(enc[:T], sd), pp, sd), labels, cfg.blank)


def align(lpb, lpe, T, U):
    """Forward and Viterbi recursions + backtrace on lp_blank / lp_emit (at least [T, U + 1]) ->
    dict(loglik, viterbi, frames [U], token_lp [U], margin [T, U + 1], path_margin) where margin is the |blank - emission| gap of
    the Viterbi candidates at every cell that has both predecessors (inf elsewhere) and path_margin its minimum along the path."""
    fa = np.full((T, U + 1), -np.inf); va = np.full((T, U + 1), -np.inf)
    ch = np.zeros((T, U + 1), dtype=np.int8); margin = np.full((T, U + 1), np.inf)
    for t in range(T):
        for u in range(U + 1):
            if t == 0 and u == 0:
                fa[0, 0] = va[0, 0] = 0.0
                continue
            fb = vb = fe = ve = -np.inf
            if t > 0:
                fb, vb = fa[t - 1, u] + lpb[t - 1, u], va[t - 1, u] + lpb[t - 1, u]
            if u > 0:
                fe, ve = fa[t, u - 1] + lpe[t, u - 1], va[t, u - 1] + lpe[t, u - 1]
            fa[t, u] = np.logaddexp(fb, fe)
            ch[t, u] = 1 if (t == 0 or ve > vb) else 0          # exact tie -> blank
            va[t, u] = ve if ch[t, u] else vb
            if t > 0 and u > 0:
                margin[t, u] = abs(vb - ve)
    frames = np.full(U, -1, dtype=np.int64); token_lp = np.full(U, np.nan)
    t, u = T - 1, U
    path_margin = np.inf
    while u > 0:
        path_margin = min(path_margin, margin[t, u])
        if ch[t, u]:
            frames[u - 1] = t; token_lp[u - 1] = lpe[t, u - 1]; u -= 1
        else:
            t -= 1
    return dict(loglik=fa[T - 1, U] + lpb[T - 1, U], viterbi=va[T - 1, U] + lpb[T - 1, U], frames=frames, token_lp=token_lp,
                margin=margin, path_margin=path_margin)


def brute_force(lpb, lpe, T, U):
    """Every monotone lattice path (the emission frames t_1 <= ... <= t_U, then the final blank at T - 1) -> (logsumexp of the
    path scores, max score, frames of the best path under the tie rule)."""
    scores, best, best_frames = [], -np.inf, None
    for frames in itertools.combinations_with_replacement(range(T), U):
        s, t = 0.0, 0
        for u, tu in enumerate(frames):
            s += sum(lpb[k, u] for k in range(t, tu))             # blanks from t to tu at label u
            s += lpe[tu, u]; t = tu
        s += sum(lpb[k, U] for k in range(t, T))                  # the last row, through the final blank
        scores.append(s)
        # tie rule: the backtrace takes the blank predecessor on a tie, i.e. among equal scores the last token's frame is the
        # smallest, then the one before it, ...
        if s > best or (s == best and frames[::-1] < best_frames[::-1]):
            best, best_frames = s, frames
    return float(np.logaddexp.reduce(scores)), float(best), np.array(best_frames if best_frames is not None else (), dtype=np.int64)
