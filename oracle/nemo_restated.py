"""CPU oracle: a plain-PyTorch fp32 restatement of the NeMo inference path that
``reazonspeech.nemo.asr.transcribe`` reaches through ``model.transcribe(...)``
(reference call site: pkg/nemo-asr/src/transcribe.py:48-53).

THIS IS TEST INFRASTRUCTURE.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it.  The product
package ``reazonspeech_b200`` never does.

PARITY: PINNED FOR N1-N7 AGAINST TWO THIRD-PARTY PORTS OF NeMo, UNPINNED FOR THE GLOBAL TOKEN AND THE GREEDY LOOP.  The arithmetic
of this path lives in ``nemo_toolkit[asr] >= 2.6.1`` (pkg/nemo-asr/pyproject.toml:13), which is absent
from /root/reference and cannot be imported offline, and the reference ships no tests, golden vectors
or fixtures for it (SURVEY.md section 8c).  What the image does ship is ``transformers.models.parakeet``,
NVIDIA's port of NeMo's FilterbankFeatures + FastConformer encoder: tests/golden/make_parakeet_golden.py
runs it on seeded weights/clips and tests/test_oracle_parakeet.py holds this file to its outputs
(log-mel incl. the get_seq_len = L // hop length convention and the masked final frame, dw_striding
subsampling, xscale, relative positional encoding + rel_shift, MHSA, convolution module, macaron FFN,
LayerNorm order: encoder output relative L2 1e-5).  Parakeet has full relative-position attention only,
so that pin covers the local-attention code path with T <= w + 1 and no global token.  A SECOND third-party
implementation closes the window gap: vLLM's Cohere-ASR model carries a near-verbatim port of NeMo's
ConformerEncoder under NeMo's own parameter names (``vllm.model_executor.models.cohere_asr``);
tests/golden/make_nemo_port_golden.py loads this file's seeded NeMo-named state dict into it with strict=True and runs
it with LIMITED attention context (band mask, symmetric and asymmetric windows) on ragged zero-padded batches whose
utterances are several windows long; tests/test_oracle_nemo_port.py holds this file to those outputs (relative L2
3e-7): windowing, pad masks, the masking between the subsampling convolutions and the key names / tensor layouts of
the checkpoint are therefore verified, not recalled.  The same package also carries a copy of NeMo's
``FilterbankFeatures`` class; a ragged batch goes through it (fp32 buffers, dither 0, pad_to 0) and on into the encoder
port: ``log_mel`` here matches its valid frames to 2.6e-4 and the whole N1-N7 path matches end to end at 1.2e-5.  NOT covered by any implementation in the image, and
still recalled (R) rather than verified: the global-token wiring of
RelPositionMultiHeadAttentionLongformer, and the RNN-T prediction network / joint / greedy loop
(``max_symbols``) -- standard LSTM-transducer arithmetic restated from NeMo's modules/rnnt.py.  For the
latter, tests/test_oracle_cpu.py::test_greedy_matches_stock_module_implementation at least ties the hand-written
LSTM cell, gate order, bias handling and joint to stock torch.nn modules (nn.LSTM is the module NeMo wraps) built
under the checkpoint's parameter names and loaded with strict=True; the loop's control flow stays recalled (R).
The reference-owned ``decode_hypothesis`` is pinned separately by importing the reference's decode.py
(tests/golden/make_decode_golden.py).

Semantics are batch=1, exactly as the reference calls NeMo (transcribe.py:48-50): every
function takes ONE utterance with no padding.  ``emulate`` switches on bf16 rounding of
activations at the points where the sm_90a engine stores bf16 (used only to tighten the
token-identity test; the reference semantics are ``emulate=False``).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from reazonspeech_b200.config import ModelConfig, conv_out_len, xscale
from reazonspeech_b200.weights import hann_window, mel_filterbank, rel_pos_table

StateDict = Dict[str, torch.Tensor]


def _q(x: torch.Tensor, emulate: bool) -> torch.Tensor:
    return x.to(torch.bfloat16).to(torch.float32) if emulate else x


# --------------------------------------------------------------------------------------
# N1  AudioToMelSpectrogramPreprocessor / FilterbankFeatures.forward
#     (nemo/collections/asr/parts/preprocessing/features.py)
# --------------------------------------------------------------------------------------
def log_mel(wave: torch.Tensor, cfg: ModelConfig, independent_fb: bool = False) -> torch.Tensor:
    """float32[L] -> float32[n_mels, F], F = L // hop: the VALID frames (``get_seq_len``).

    The centred STFT yields L // hop + 1 frames; NeMo's length is one less, the final frame is
    masked to zero, stays out of the statistics, and every later stage masks by length -- which at
    batch=1 is the same as dropping it here (pinned against transformers' Parakeet port of NeMo,
    tests/test_oracle_parakeet.py).

    preemph -> torch.stft(center=True, zero pad (R: "constant"; identical to "reflect" on
    transcribe() inputs, whose 0.5 s edges are silence -- audio.py:80-82)) -> |X| -> **2 ->
    mel -> log(x + 2^-24) -> per-feature (mean, unbiased std + 1e-5) normalisation."""
    x = wave.to(torch.float32)
    if cfg.preemph:
        x = torch.cat((x[:1], x[1:] - cfg.preemph * x[:-1]))
    spec = torch.stft(x, n_fft=cfg.n_fft, hop_length=cfg.n_window_stride, win_length=cfg.n_window_size,
                      window=hann_window(cfg), center=True, pad_mode="constant", return_complex=True)
    mag = torch.sqrt(torch.view_as_real(spec).pow(2).sum(-1))
    power = mag.pow(2.0)
    if independent_fb:      # cross-check of weights.mel_filterbank against torchaudio's construction
        import torchaudio
        fb = torchaudio.functional.melscale_fbanks(cfg.n_freq, 0.0, cfg.sample_rate / 2, cfg.n_mels,
                                                   cfg.sample_rate, norm="slaney", mel_scale="slaney").T
    else:
        fb = mel_filterbank(cfg)
    mel = torch.matmul(fb, power)
    mel = torch.log(mel + cfg.log_zero_guard)
    assert mel.shape[1] == cfg.mel_frames(wave.numel())
    mel = mel[:, : cfg.mel_valid(wave.numel())]
    mean = mel.mean(dim=1, keepdim=True)
    std = mel.std(dim=1, keepdim=True) + cfg.norm_eps          # unbiased (N-1)
    return (mel - mean) / std


# --------------------------------------------------------------------------------------
# N2  ConvSubsampling (dw_striding, x8)   (parts/submodules/subsampling.py)
# --------------------------------------------------------------------------------------
def subsample(mel: torch.Tensor, sd: StateDict, cfg: ModelConfig, emulate: bool = False) -> torch.Tensor:
    """float32[n_mels, F] -> float32[T, d_model] (before xscale)."""
    p = "encoder.pre_encode."
    x = mel.T.unsqueeze(0).unsqueeze(0)                                           # [1,1,F,80]
    x = F.relu(F.conv2d(x, sd[p + "conv.0.weight"], sd[p + "conv.0.bias"], stride=2, padding=1))
    for dw, pw in ((2, 3), (5, 6)):
        c = x.shape[1]
        x = F.conv2d(x, sd[p + f"conv.{dw}.weight"], sd[p + f"conv.{dw}.bias"], stride=2, padding=1, groups=c)
        x = _q(x, emulate)
        x = F.relu(F.conv2d(x, sd[p + f"conv.{pw}.weight"], sd[p + f"conv.{pw}.bias"]))
        x = _q(x, emulate)
    b, c, t, f = x.shape
    x = x.transpose(1, 2).reshape(b, t, c * f)                                    # index c*f_out + f
    x = F.linear(x, sd[p + "out.weight"], sd[p + "out.bias"])
    return x[0]


# --------------------------------------------------------------------------------------
# N5  RelPositionMultiHeadAttentionLongformer  (parts/submodules/multi_head_attention.py) (R)
# --------------------------------------------------------------------------------------
def local_attention_core(q, k, v, p, u, vb, cfg: ModelConfig, emulate: bool = False) -> torch.Tensor:
    """q,k,v: [H,T,dk]; p: [H,n_rel,dk] (linear_pos of the table); u,vb: [H,dk] -> [H,T,dk].

    Dense restatement of the sliding-chunk computation:
      local score(i, j) = ((q_i+u).k_j + (q_i+v).p[w_left-(i-j)]) / sqrt(dk),  -w_left <= j-i <= w_right
      keys outside [0,T) or outside the band are excluded (upstream fills them with -inf / -1e4);
      with global_tokens=G: an extra column per global key g with score (q_i/sqrt(dk)).k_g
      (no positional term; the same key ALSO stays in the local band (R)); softmax over the
      concatenation; output = P_glob.v_g + P_local.v.  Rows of the global tokens themselves
      are overwritten with full attention softmax_j((q_g/sqrt(dk)).k_j).v_j over all T keys."""
    H, T, dk = q.shape
    wl, wr, G = cfg.att_left, cfg.att_right, cfg.global_tokens
    scale = 1.0 / math.sqrt(dk)
    qu = _q(q + u[:, None, :], emulate)
    qv = _q(q + vb[:, None, :], emulate)
    ac = torch.matmul(qu, k.transpose(1, 2))                                      # [H,T,T]
    bd_rel = torch.matmul(qv, p.transpose(1, 2))                                  # [H,T,n_rel]
    if emulate:                                                                   # the engine stores this term in IEEE half
        bd_rel = bd_rel.to(torch.float16).to(torch.float32)
    i = torch.arange(T)[:, None]
    j = torch.arange(T)[None, :]
    rel = j - i
    band = (rel >= -wl) & (rel <= wr)
    idx = (rel + wl).clamp(0, cfg.n_rel - 1)
    bd = torch.gather(bd_rel, 2, idx.unsqueeze(0).expand(H, T, T))
    s_local = ((ac + bd) * scale).masked_fill(~band.unsqueeze(0), float("-inf"))
    if G > 0:
        s_glob = torch.matmul(q * scale, k[:, :G].transpose(1, 2))                # [H,T,G]
        probs = torch.softmax(torch.cat((s_glob, s_local), dim=-1), dim=-1)
        probs = _q(probs, emulate)
        out = torch.matmul(probs[..., :G], v[:, :G]) + torch.matmul(probs[..., G:], v)
        sg = torch.matmul(q[:, :G] * scale, k.transpose(1, 2))                    # [H,G,T]
        out[:, :G] = torch.matmul(_q(torch.softmax(sg, dim=-1), emulate), v)
    else:
        out = torch.matmul(_q(torch.softmax(s_local, dim=-1), emulate), v)
    return out


def self_attention(x: torch.Tensor, sd: StateDict, pfx: str, cfg: ModelConfig, emulate: bool = False) -> torch.Tensor:
    """x: [T,d] (already layer-normed) -> [T,d]."""
    T, d = x.shape
    H, dk = cfg.n_heads, cfg.d_head
    a = pfx + "self_attn."
    def heads(t):
        return t.view(T, H, dk).transpose(0, 1)
    q = _q(F.linear(x, sd[a + "linear_q.weight"], sd[a + "linear_q.bias"]), emulate)
    k = _q(F.linear(x, sd[a + "linear_k.weight"], sd[a + "linear_k.bias"]), emulate)
    v = _q(F.linear(x, sd[a + "linear_v.weight"], sd[a + "linear_v.bias"]), emulate)
    pos = F.linear(rel_pos_table(cfg), sd[a + "linear_pos.weight"])               # [n_rel,d], no bias
    p = _q(pos, emulate).view(cfg.n_rel, H, dk).transpose(0, 1)
    o = local_attention_core(heads(q), heads(k), heads(v), p, sd[a + "pos_bias_u"], sd[a + "pos_bias_v"], cfg, emulate)
    o = _q(o.transpose(0, 1).reshape(T, d), emulate)
    return F.linear(o, sd[a + "linear_out.weight"], sd[a + "linear_out.bias"])


# --------------------------------------------------------------------------------------
# N4 / N6 / N7  ConformerLayer  (parts/submodules/conformer_modules.py)
# --------------------------------------------------------------------------------------
def feed_forward(x, sd, pfx, emulate=False):
    h = F.silu(F.linear(x, sd[pfx + "linear1.weight"], sd[pfx + "linear1.bias"]))
    return F.linear(_q(h, emulate), sd[pfx + "linear2.weight"], sd[pfx + "linear2.bias"])


def conv_module(x, sd, pfx, cfg: ModelConfig, emulate=False):
    """pointwise_conv1 -> GLU(channels) -> depthwise k (zero pad) -> BatchNorm1d(eval) -> Swish -> pointwise_conv2."""
    c = pfx + "conv."
    y = F.linear(x, sd[c + "pointwise_conv1.weight"][:, :, 0], sd[c + "pointwise_conv1.bias"])
    y = _q(F.glu(y, dim=-1), emulate)                                             # first half * sigmoid(second half)
    y = y.T.unsqueeze(0)                                                          # [1,d,T]
    pad = (cfg.conv_kernel - 1) // 2
    y = F.conv1d(y, sd[c + "depthwise_conv.weight"], sd[c + "depthwise_conv.bias"], padding=pad, groups=y.shape[1])
    y = F.batch_norm(y, sd[c + "batch_norm.running_mean"], sd[c + "batch_norm.running_var"],
                     sd[c + "batch_norm.weight"], sd[c + "batch_norm.bias"], training=False, eps=cfg.bn_eps)
    y = _q(F.silu(y)[0].T, emulate)
    return F.linear(y, sd[c + "pointwise_conv2.weight"][:, :, 0], sd[c + "pointwise_conv2.bias"])


def conformer_layer(x, sd, i: int, cfg: ModelConfig, emulate=False):
    p = f"encoder.layers.{i}."
    d = (cfg.d_model,)
    def ln(t, name):
        return F.layer_norm(t, d, sd[p + name + ".weight"], sd[p + name + ".bias"], cfg.ln_eps)
    x = x + 0.5 * feed_forward(_q(ln(x, "norm_feed_forward1"), emulate), sd, p + "feed_forward1.", emulate)
    x = x + self_attention(_q(ln(x, "norm_self_att"), emulate), sd, p, cfg, emulate)
    x = x + conv_module(_q(ln(x, "norm_conv"), emulate), sd, p, cfg, emulate)
    x = x + 0.5 * feed_forward(_q(ln(x, "norm_feed_forward2"), emulate), sd, p + "feed_forward2.", emulate)
    return ln(x, "norm_out")


def encoder(mel: torch.Tensor, sd: StateDict, cfg: ModelConfig, emulate: bool = False,
            n_layers: Optional[int] = None) -> torch.Tensor:
    """ConformerEncoder.forward_internal at batch=1: float32[n_mels,F] -> float32[T,d_model]."""
    x = subsample(mel, sd, cfg, emulate) * xscale(cfg)
    for i in range(cfg.n_layers if n_layers is None else n_layers):
        x = conformer_layer(x, sd, i, cfg, emulate)
    return x


# --------------------------------------------------------------------------------------
# N8 / N9  RNNTDecoder.predict, RNNTJoint.joint, GreedyRNNTInfer._greedy_decode
#          (modules/rnnt.py, parts/submodules/rnnt_greedy_decoding.py)
# --------------------------------------------------------------------------------------
@dataclass
class GreedyResult:
    tokens: List[int] = field(default_factory=list)
    frames: List[int] = field(default_factory=list)       # encoder frame index of each emission
    margins: List[float] = field(default_factory=list)    # top1 - top2 logit of EVERY joint evaluation
    decisions: List[int] = field(default_factory=list)    # argmax of every joint evaluation (incl. blanks)


def joint_enc_proj(enc: torch.Tensor, sd: StateDict) -> torch.Tensor:
    return F.linear(enc, sd["joint.enc.weight"], sd["joint.enc.bias"])


def lstm_step(x, h, c, sd):
    l = "decoder.prediction.dec_rnn.lstm."
    gates = (F.linear(x, sd[l + "weight_ih_l0"], sd[l + "bias_ih_l0"]) +
             F.linear(h, sd[l + "weight_hh_l0"], sd[l + "bias_hh_l0"]))
    i, f, g, o = gates.chunk(4)
    c2 = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
    h2 = torch.sigmoid(o) * torch.tanh(c2)
    return h2, c2


def rnnt_greedy(enc: torch.Tensor, sd: StateDict, cfg: ModelConfig, emulate: bool = False) -> GreedyResult:
    """enc: float32[T,d_model] -> greedy hypothesis (tokens, frame of each token).

    For every frame t: up to max_symbols times { g = pred(last_token, state);
    logits = W_out relu(W_enc f_t + W_pred g + b); k = argmax; blank -> next frame;
    else emit k at t and commit the LSTM state }.  The start token is blank, whose
    embedding row is the zero vector (blank_as_pad)."""
    hp = cfg.pred_hidden
    res = GreedyResult()
    ep = joint_enc_proj(_q(enc, emulate), sd)
    n_threads = torch.get_num_threads()
    torch.set_num_threads(1)            # the token loop is matrix-vector work; threads only add sync cost
    try:
        return _greedy_loop(ep, sd, cfg, res)
    finally:
        torch.set_num_threads(n_threads)


def _greedy_loop(ep, sd, cfg, res):
    hp = cfg.pred_hidden
    emb = sd["decoder.prediction.embed.weight"]
    h = torch.zeros(hp); c = torch.zeros(hp)
    h_new, c_new = lstm_step(torch.zeros(hp), h, c, sd)                            # SOS step
    pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
    W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
    for t in range(ep.shape[0]):
        for _ in range(cfg.max_symbols):
            logits = F.linear(torch.relu(ep[t] + pp), W, b)
            top2 = torch.topk(logits, 2)
            k = int(top2.indices[0])
            res.margins.append(float(top2.values[0] - top2.values[1]))
            res.decisions.append(k)
            if k == cfg.blank:
                break
            res.tokens.append(k); res.frames.append(t)
            h, c = h_new, c_new
            h_new, c_new = lstm_step(emb[k], h, c, sd)
            pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
    return res


@dataclass
class FollowResult:
    """Outcome of walking a GIVEN decision sequence through the oracle's predictor + joint."""
    n_decisions: int = 0
    complete: bool = True                                  # the sequence accounts for every frame, no more, no less
    gaps: List[tuple] = field(default_factory=list)        # (decision index, frame, given, oracle argmax, logit gap) where they differ
    min_margin: float = float("inf")                       # smallest oracle top-2 margin met on the way
    margins: List[float] = field(default_factory=list)     # oracle top-2 margin of every decision
    noise: List[float] = field(default_factory=list)       # with enc_ref: change of that top-2 gap when enc_ref replaces enc


def greedy_follow(enc: torch.Tensor, sd: StateDict, cfg: ModelConfig, decisions: List[int], emulate: bool = False,
                  enc_ref: Optional[torch.Tensor] = None) -> FollowResult:
    """Re-synchronising comparison with a greedy decode produced elsewhere (the sm_90a engine).

    Walks ``decisions`` (the argmax of EVERY joint evaluation, blanks included, as rebuilt from tokens + frames) through
    the same control flow as ``rnnt_greedy`` but TEACHER-FORCED: the predictor state always follows the given decision.
    Wherever the oracle's own argmax differs, the entry records ``logit[oracle argmax] - logit[given]`` -- the amount by
    which the given decision loses under the oracle's arithmetic -- and the walk goes on, so one near-tie cannot hide the
    rest of the sequence.  A decode is greedy-identical to the oracle iff ``gaps`` is empty and ``complete`` is true.

    ``enc_ref`` (a second evaluation of the SAME encoder, e.g. the fp32 one next to the bf16-emulated ``enc``) turns the walk
    into a noise measurement as well: at every decision the gap between the oracle's two best classes is re-evaluated with
    ``enc_ref``'s frame and the change is recorded in ``noise`` -- how far storage rounding alone moves a decision gap."""
    res = FollowResult()
    ep = joint_enc_proj(_q(enc, emulate), sd)
    ep_ref = joint_enc_proj(_q(enc_ref, emulate), sd) if enc_ref is not None else None
    n_threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        hp = cfg.pred_hidden
        emb = sd["decoder.prediction.embed.weight"]
        h = torch.zeros(hp); c = torch.zeros(hp)
        h_new, c_new = lstm_step(torch.zeros(hp), h, c, sd)
        pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
        W, b = sd["joint.joint_net.2.weight"], sd["joint.joint_net.2.bias"]
        i = 0
        for t in range(ep.shape[0]):
            for _ in range(cfg.max_symbols):
                if i >= len(decisions):
                    res.complete = False
                    return res
                logits = F.linear(torch.relu(ep[t] + pp), W, b)
                top2 = torch.topk(logits, 2)
                m = float(top2.values[0] - top2.values[1])
                res.min_margin = min(res.min_margin, m)
                res.margins.append(m)
                if ep_ref is not None:
                    alt = F.linear(torch.relu(ep_ref[t] + pp), W, b)
                    res.noise.append(float(alt[top2.indices[0]] - alt[top2.indices[1]]) - m)
                k = int(decisions[i]); i += 1
                if k != int(top2.indices[0]):
                    res.gaps.append((i - 1, t, k, int(top2.indices[0]), float(top2.values[0] - logits[k])))
                if k == cfg.blank:
                    break
                h, c = h_new, c_new
                h_new, c_new = lstm_step(emb[k], h, c, sd)
                pp = F.linear(h_new, sd["joint.pred.weight"], sd["joint.pred.bias"])
        res.n_decisions = i
        res.complete = i == len(decisions)
        return res
    finally:
        torch.set_num_threads(n_threads)


# --------------------------------------------------------------------------------------
# Whole path at the model.transcribe seam
# --------------------------------------------------------------------------------------
def transcribe_tokens(wave: torch.Tensor, sd: StateDict, cfg: ModelConfig, emulate: bool = False) -> GreedyResult:
    """The reference path from the padded waveform tensor (transcribe.py:46) to greedy tokens."""
    with torch.no_grad():
        return rnnt_greedy(encoder(log_mel(wave, cfg), sd, cfg, emulate), sd, cfg, emulate)
