"""Streaming restated on the CPU oracle (oracle/nemo_restated.py): the greedy loop of ``_greedy_loop`` with a carried decoder
state, and the chunk schedule of reazonspeech_b200/streaming.py driven through the oracle's own log-mel and encoder."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from oracle import nemo_restated as O
from reazonspeech_b200.streaming import PAD_SAMPLES, plan_row


@dataclass
class DecoderState:
    """What a stream carries between chunks: the LSTM state after the last emission (its h, c) and that state's
    joint.pred projection pp."""
    h: torch.Tensor
    c: torch.Tensor
    pp: torch.Tensor


def greedy_resume(ep: torch.Tensor, sd, cfg, t0: int, t1: int, state: Optional[DecoderState] = None, res=None):
    """``_greedy_loop`` over frames [t0, t1) of ``ep`` (joint.enc outputs), starting from ``state`` (None: the SOS step, as the
    oracle starts) -> (GreedyResult with frames of ``ep``, the state to carry)."""
    res = res if res is not None else O.GreedyResult()
    emb = sd["decoder.prediction.embed.weight"]
    W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
    if state is None:
        hp = cfg.pred_hidden
        h, c = O.lstm_step(torch.zeros(hp), torch.zeros(hp), torch.zeros(hp), sd)
        state = DecoderState(h, c, F.linear(h, sd["joint.pred.weight"], sd["joint.pred.bias"]))
    h, c, pp = state.h, state.c, state.pp
    for t in range(t0, t1):
        for _ in range(cfg.max_symbols):
            logits = F.linear(torch.relu(ep[t] + pp), W, b)
            top2 = torch.topk(logits, 2)
            k = int(top2.indices[0])
            res.margins.append(float(top2.values[0] - top2.values[1]))
            res.decisions.append(k)
            if k == cfg.blank:
                break
            res.tokens.append(k); res.frames.append(t)
            h, c = O.lstm_step(emb[k], h, c, sd)
            pp = F.linear(h, sd["joint.pred.weight"], sd["joint.pred.bias"])
    return res, DecoderState(h, c, pp)


def stream_buffers(padded: np.ndarray, frames_cfg) -> List[tuple]:
    """The steps of one stream fed and closed up front: (a, b, dec_begin, dec_end, offset) rows in order."""
    n, D, out = len(padded), 0, []
    while True:
        row = plan_row(n, D, True, frames_cfg)
        if row is None:
            return out
        out.append(row)
        D = row.dec_end + row.offset


def oracle_stream(wave: np.ndarray, sd, cfg, frames_cfg, emulate: bool = False, rows: Optional[Sequence] = None):
    """The oracle's streaming decode of one utterance (``wave`` unpadded, fed and closed up front): every step encodes its buffer
    with the oracle and decodes the step's frames from the carried state -> GreedyResult with GLOBAL frames."""
    padded = np.concatenate([np.zeros(PAD_SAMPLES, np.float32), wave.astype(np.float32), np.zeros(PAD_SAMPLES, np.float32)])
    res, state = O.GreedyResult(), None
    with torch.no_grad():
        for row in rows if rows is not None else stream_buffers(padded, frames_cfg):
            buf = torch.from_numpy(padded[row.a:row.b])
            ep = O.joint_enc_proj(O._q(O.encoder(O.log_mel(buf, cfg), sd, cfg, emulate), emulate), sd)
            part, state = greedy_resume(ep, sd, cfg, row.dec_begin, row.dec_end, state)
            res.tokens += part.tokens
            res.frames += [f + row.offset for f in part.frames]
            res.margins += part.margins
            res.decisions += part.decisions
    return res


def follow_resume(ep: torch.Tensor, sd, cfg, t0: int, t1: int, tokens: Sequence[int], frames: Sequence[int],
                  state: Optional[DecoderState] = None):
    """``greedy_resume`` TEACHER-FORCED along a decode made elsewhere (its tokens and frames of ``ep`` in [t0, t1)): at every joint
    evaluation the oracle's argmax is compared with the given decision and the walk follows the given one -> (gaps, state):
    gaps lists (frame, given, oracle argmax, logit[oracle argmax] - logit[given]) where they differ."""
    emb = sd["decoder.prediction.embed.weight"]
    W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
    if state is None:
        hp = cfg.pred_hidden
        h, c = O.lstm_step(torch.zeros(hp), torch.zeros(hp), torch.zeros(hp), sd)
        state = DecoderState(h, c, F.linear(h, sd["joint.pred.weight"], sd["joint.pred.bias"]))
    h, c, pp = state.h, state.c, state.pp
    gaps, i = [], 0
    for t in range(t0, t1):
        for _ in range(cfg.max_symbols):
            k = int(tokens[i]) if i < len(tokens) and int(frames[i]) == t else cfg.blank
            logits = F.linear(torch.relu(ep[t] + pp), W, b)
            top = int(torch.argmax(logits))
            if top != k:
                gaps.append((t, k, top, float(logits[top] - logits[k])))
            if k == cfg.blank:
                break
            i += 1
            h, c = O.lstm_step(emb[k], h, c, sd)
            pp = F.linear(h, sd["joint.pred.weight"], sd["joint.pred.bias"])
    assert i == len(tokens), "tokens outside [t0, t1)"
    return gaps, DecoderState(h, c, pp)
