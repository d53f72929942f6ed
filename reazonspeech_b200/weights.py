"""Checkpoint handling: NeMo state-dict naming, seeded synthetic weights, ``.nemo`` reader.

The reference obtains its weights through
``EncDecRNNTBPEModel.from_pretrained('reazon-research/reazonspeech-nemo-v2')``
(pkg/nemo-asr/src/transcribe.py:26-28).  Neither NeMo nor the checkpoint is reachable
offline, so every test and the benchmark run on *seeded random weights of the same
shapes*, keyed by the same state-dict names NeMo uses -- a real ``model_weights.ckpt``
drops in through :func:`load_nemo_archive` without touching anything downstream.

Synthetic weights are rounded to bf16-representable values on purpose: the engine keeps
GEMM weights in bf16, so with representable weights the CPU oracle and the engine
evaluate *the same model* and the only deviation left is activation rounding.
"""
from __future__ import annotations

import io
import math
import tarfile
from typing import Dict, Optional

import numpy as np
import torch

from .config import ModelConfig

StateDict = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------------------
# Fixed (non-learned) tables of the frontend / positional encoding
# --------------------------------------------------------------------------------------
def hann_window(cfg: ModelConfig) -> torch.Tensor:
    """Symmetric Hann (torch.hann_window(periodic=False)), float32, length n_window_size."""
    n = cfg.n_window_size
    k = torch.arange(n, dtype=torch.float64)
    return (0.5 - 0.5 * torch.cos(2.0 * math.pi * k / (n - 1))).to(torch.float32)


def _hz_to_mel_slaney(f: np.ndarray) -> np.ndarray:
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz, min_log_mel = 1000.0, 1000.0 / f_sp
    logstep = math.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, mels)


def _mel_to_hz_slaney(m: np.ndarray) -> np.ndarray:
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel = 1000.0, 1000.0 / f_sp
    logstep = math.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(cfg: ModelConfig) -> torch.Tensor:
    """Slaney-scale, slaney-normalised triangular filterbank, float32 [n_mels, n_freq].

    Restates librosa.filters.mel(sr, n_fft, n_mels, fmin=0, fmax=sr/2, htk=False,
    norm='slaney'), which NeMo's FilterbankFeatures uses for ``self.fb``."""
    sr, n_fft, n_mels = cfg.sample_rate, cfg.n_fft, cfg.n_mels
    fftfreqs = np.linspace(0.0, sr / 2.0, cfg.n_freq)
    mel_pts = np.linspace(_hz_to_mel_slaney(0.0), _hz_to_mel_slaney(sr / 2.0), n_mels + 2)
    hz_pts = _mel_to_hz_slaney(mel_pts)
    fdiff = np.diff(hz_pts)
    ramps = hz_pts[:, None] - fftfreqs[None, :]
    fb = np.zeros((n_mels, cfg.n_freq), dtype=np.float64)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        fb[i] = np.maximum(0.0, np.minimum(lower, upper))
    enorm = 2.0 / (hz_pts[2:n_mels + 2] - hz_pts[:n_mels])
    fb *= enorm[:, None]
    return torch.from_numpy(fb.astype(np.float32))


def rel_pos_table(cfg: ModelConfig) -> torch.Tensor:
    """LocalAttRelPositionalEncoding table, float32 [n_rel, d_model].

    Row c holds the sinusoid of relative position (att_left - c): positions run from
    +left down to -right, interleaved sin/cos with the 10000^(-2i/d) frequencies."""
    pos = torch.arange(cfg.att_left, -cfg.att_right - 1, -1, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, cfg.d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / cfg.d_model))
    pe = torch.zeros(pos.shape[0], cfg.d_model, dtype=torch.float32)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


# --------------------------------------------------------------------------------------
# State-dict schema (NeMo names)
# --------------------------------------------------------------------------------------
def state_dict_shapes(cfg: ModelConfig) -> Dict[str, tuple]:
    d, h, dk, ff, k = cfg.d_model, cfg.n_heads, cfg.d_head, cfg.d_ff, cfg.conv_kernel
    c = cfg.sub_channels
    s: Dict[str, tuple] = {}
    pe = "encoder.pre_encode."
    s[pe + "conv.0.weight"] = (c, 1, 3, 3); s[pe + "conv.0.bias"] = (c,)
    for dw, pw in ((2, 3), (5, 6)):
        s[pe + f"conv.{dw}.weight"] = (c, 1, 3, 3); s[pe + f"conv.{dw}.bias"] = (c,)
        s[pe + f"conv.{pw}.weight"] = (c, c, 1, 1); s[pe + f"conv.{pw}.bias"] = (c,)
    s[pe + "out.weight"] = (d, cfg.sub_out_dim); s[pe + "out.bias"] = (d,)
    for i in range(cfg.n_layers):
        p = f"encoder.layers.{i}."
        for ln in ("norm_feed_forward1", "norm_self_att", "norm_conv", "norm_feed_forward2", "norm_out"):
            s[p + ln + ".weight"] = (d,); s[p + ln + ".bias"] = (d,)
        for f in ("feed_forward1", "feed_forward2"):
            s[p + f + ".linear1.weight"] = (ff, d); s[p + f + ".linear1.bias"] = (ff,)
            s[p + f + ".linear2.weight"] = (d, ff); s[p + f + ".linear2.bias"] = (d,)
        for l in ("linear_q", "linear_k", "linear_v", "linear_out"):
            s[p + f"self_attn.{l}.weight"] = (d, d); s[p + f"self_attn.{l}.bias"] = (d,)
        s[p + "self_attn.linear_pos.weight"] = (d, d)
        s[p + "self_attn.pos_bias_u"] = (h, dk); s[p + "self_attn.pos_bias_v"] = (h, dk)
        s[p + "conv.pointwise_conv1.weight"] = (2 * d, d, 1); s[p + "conv.pointwise_conv1.bias"] = (2 * d,)
        s[p + "conv.depthwise_conv.weight"] = (d, 1, k); s[p + "conv.depthwise_conv.bias"] = (d,)
        for b in ("weight", "bias", "running_mean", "running_var"):
            s[p + "conv.batch_norm." + b] = (d,)
        s[p + "conv.pointwise_conv2.weight"] = (d, d, 1); s[p + "conv.pointwise_conv2.bias"] = (d,)
    hp, hj = cfg.pred_hidden, cfg.joint_hidden
    s["decoder.prediction.embed.weight"] = (cfg.n_classes, hp)
    lstm = "decoder.prediction.dec_rnn.lstm."
    s[lstm + "weight_ih_l0"] = (4 * hp, hp); s[lstm + "weight_hh_l0"] = (4 * hp, hp)
    s[lstm + "bias_ih_l0"] = (4 * hp,); s[lstm + "bias_hh_l0"] = (4 * hp,)
    s["joint.enc.weight"] = (hj, d); s["joint.enc.bias"] = (hj,)
    s["joint.pred.weight"] = (hj, hp); s["joint.pred.bias"] = (hj,)
    s["joint.joint_net.2.weight"] = (cfg.n_classes, hj); s["joint.joint_net.2.bias"] = (cfg.n_classes,)
    return s


def _bf16_round(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float32)


def _cfg_key(cfg: ModelConfig) -> str:
    return f"{cfg.n_layers}x{cfg.d_model}_v{cfg.vocab_size}_p{cfg.pred_hidden}_j{cfg.joint_hidden}"


def calibration_path(cfg: ModelConfig, seed: int) -> str:
    import os
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", f"synth_calib_{_cfg_key(cfg)}_seed{seed}.json")


def apply_calibration(sd: StateDict, cfg: ModelConfig, calib: dict) -> None:
    """In-place: joint.enc gain (a power of two, so weights stay bf16-exact) and bias, blank shift."""
    sd["joint.enc.weight"] = sd["joint.enc.weight"] * float(2.0 ** int(calib.get("joint_enc_gain_log2", 0)))
    if calib.get("joint_enc_bias") is not None:
        sd["joint.enc.bias"] = _bf16_round(torch.tensor(calib["joint_enc_bias"], dtype=torch.float32))
    b = sd["joint.joint_net.2.bias"].clone()
    b[cfg.blank] += float(calib.get("blank_shift", 0.0))
    sd["joint.joint_net.2.bias"] = _bf16_round(b)


def _structure_predictor(sd: StateDict, cfg: ModelConfig, suppress: float = 16.0, decay_logit: float = 2.2) -> None:
    """Give the synthetic prediction network the one behaviour greedy RNN-T decoding relies on in a trained
    model: having emitted a token, stop preferring it.  An untrained LSTM instead has states in which some
    token keeps winning on every frame (decoding then emits max_symbols tokens per frame for the rest of the
    clip).  Construction (still an ordinary embedding + LSTM + linear, only the values are chosen):
      embed[k] = -suppress * W_out[k];  LSTM: input gate ~1, output gate ~1, forget gate sigmoid(2.2) ~ 0.9,
      candidate g = tanh(embed + small noise);  joint.pred ~ identity (+ small noise).
    so pred_proj ~ -suppress * sum_i 0.9^i W_out[k_{-i}]: the logits of the most recently emitted tokens are
    pushed down, everything else is perturbed only by the small random terms.

    The RECURRENT random term is kept small enough (row norm 0.1) for the state map to be a contraction.  With row norm 0.5
    (round 1) the predictor was weakly chaotic: the fp32 and fp64 evaluations of the SAME token sequence drifted apart
    exponentially (1e-7 after one step, 2.5e-3 after 800), so on a
    clip that bursts to a thousand tokens not even the oracle agreed with itself across precisions, let alone with the
    engine.  A trained prediction network forgets its distant past; this one now does too."""
    hp, hj = cfg.pred_hidden, cfg.joint_hidden
    # The blank row of the output layer is the constant vector 0.1875 / sqrt(hj).  A random blank row makes the blank logit
    # swing from frame to frame like any token's while the SPREAD of the 3000 token logits follows the frame's activation norm:
    # a frame then emits either nothing or -- where its norm is large -- max_symbols tokens at once, and a clip's token count
    # is decided by a handful of such frames (one clip of the bench set decoded 50 to 3800 tokens depending on the last bit
    # of the blank bias).  A constant positive row makes the blank logit proportional to the l1 norm of the (ReLU) activation,
    # i.e. it sits a fixed number of standard deviations (about 3.3 at 0.1875) above the token logits of EVERY frame: the
    # tokens that beat it are few and spread over the frames, like speech.  Values only; bf16-exact.
    w_all = sd["joint.joint_net.2.weight"].clone()
    w_all[cfg.blank] = _bf16_round(torch.full((hj,), 0.1875 / math.sqrt(hj)))
    sd["joint.joint_net.2.weight"] = w_all
    if hp != hj:
        return                                           # construction needs the two widths to agree (640 == 640)
    l = "decoder.prediction.dec_rnn.lstm."
    w_out = sd["joint.joint_net.2.weight"]
    emb = -suppress * w_out.clone()
    emb[cfg.blank] = 0.0
    sd["decoder.prediction.embed.weight"] = _bf16_round(emb)
    w_ih = 0.02 * sd[l + "weight_ih_l0"] * math.sqrt(hp)            # small noise everywhere ...
    w_ih[2 * hp:3 * hp] += torch.eye(hp)                             # ... identity on the candidate (g) block
    sd[l + "weight_ih_l0"] = _bf16_round(w_ih)
    sd[l + "weight_hh_l0"] = _bf16_round(0.004 * sd[l + "weight_hh_l0"] * math.sqrt(hp))
    b = torch.zeros(4 * hp)
    b[0 * hp:1 * hp] = 3.0                                           # input gate open
    b[1 * hp:2 * hp] = decay_logit                                   # forget gate: memory of recent tokens decays
    b[3 * hp:4 * hp] = 3.0                                           # output gate open
    sd[l + "bias_ih_l0"] = _bf16_round(b)
    sd["joint.pred.weight"] = _bf16_round(torch.eye(hj, hp) + 0.02 * sd["joint.pred.weight"] * math.sqrt(hp))


def random_state_dict(cfg: ModelConfig, seed: int = 0, calibrate: bool = True) -> StateDict:
    """Seeded synthetic checkpoint with NeMo's names and shapes (float32, bf16-representable).

    Linear / conv weights ~ N(0, gain/fan_in) (variance preserving; gain 2 ahead of a ReLU), small
    biases, LayerNorm gains near 1, BatchNorm running stats near (0, 1).

    An untrained network of this depth has two properties a trained model does not: its encoder
    output is dominated by a time-constant component (every ReLU/Swish turns zero-mean input into
    a DC offset), and its joint puts blank at 1/3001, so greedy decoding would emit ``max_symbols``
    tokens on every frame.  With ``calibrate`` the stored calibration for this (config, seed)
    (``data/synth_calib_*.json``, produced by scripts/calibrate_synthetic.py from the seeded weights)
    is applied: joint.enc's bias cancels the DC component of the encoder output and its gain is a
    power of two bringing the time-varying part to a fixed scale, and the blank bias is shifted so the
    greedy emission rate is about one token per three frames -- the decode LOAD of speech
    (SURVEY.md section 8d).  The prediction network is structured (see _structure_predictor) so that
    an emitted token is suppressed afterwards, as in a trained model.  All of this shapes the workload
    only; oracle and engine see identical tensors."""
    sd: StateDict = {}
    for idx, (name, shape) in enumerate(state_dict_shapes(cfg).items()):
        rng = np.random.default_rng([seed, idx])
        randn = lambda: torch.from_numpy(rng.standard_normal(shape, dtype=np.float32))
        leaf = name.rsplit(".", 1)[-1]
        if "norm" in name and leaf == "weight":
            t = 1.0 + 0.1 * randn()
        elif "norm" in name and leaf == "bias":
            t = 0.1 * randn()
        elif leaf == "running_mean":
            t = 0.1 * randn()
        elif leaf == "running_var":
            t = 0.5 + torch.from_numpy(rng.random(shape, dtype=np.float32))
        elif leaf in ("pos_bias_u", "pos_bias_v"):
            t = 0.1 * randn()
        elif name == "decoder.prediction.embed.weight":
            t = randn()
            t[cfg.blank] = 0.0                      # padding_idx == blank (blank_as_pad)
        elif len(shape) == 1:                       # a bias
            t = 0.02 * randn()
        else:
            fan_in = int(np.prod(shape[1:]))
            gain = 2.0 if "pre_encode.conv" in name else 1.0
            t = randn() * math.sqrt(gain / fan_in)
        sd[name] = _bf16_round(t.to(torch.float32))
    _structure_predictor(sd, cfg)
    if calibrate:
        import json
        import os
        path = calibration_path(cfg, seed)
        if os.path.exists(path):
            apply_calibration(sd, cfg, json.load(open(path)))
    return sd


# --------------------------------------------------------------------------------------
# .nemo archive reader
# --------------------------------------------------------------------------------------
def load_nemo_archive(path: str):
    """Read a ``.nemo`` archive: returns (ModelConfig, state_dict, tokenizer_model_bytes | None).

    A ``.nemo`` file is a (possibly gzipped) tar holding ``model_config.yaml``,
    ``model_weights.ckpt`` (a torch state dict) and ``*_tokenizer.model`` (SentencePiece)."""
    import yaml
    cfg_d, sd, tok = None, None, None
    with tarfile.open(path, "r:*") as tar:
        for m in tar.getmembers():
            base = m.name.rsplit("/", 1)[-1]
            if base == "model_config.yaml":
                cfg_d = yaml.safe_load(tar.extractfile(m).read())
            elif base == "model_weights.ckpt":
                sd = torch.load(io.BytesIO(tar.extractfile(m).read()), map_location="cpu", weights_only=True)
            elif base.endswith("tokenizer.model"):
                tok = tar.extractfile(m).read()
    if cfg_d is None or sd is None:
        raise ValueError(f"{path}: not a .nemo archive (model_config.yaml / model_weights.ckpt missing)")
    cfg = ModelConfig.from_nemo_yaml(cfg_d)
    want = state_dict_shapes(cfg)
    sd = {k: v.to(torch.float32) for k, v in sd.items() if k in want}
    missing = [k for k in want if k not in sd]
    if missing:
        raise ValueError(f"{path}: checkpoint lacks {len(missing)} tensors, e.g. {missing[:3]}")
    for k, shp in want.items():
        if tuple(sd[k].shape) != tuple(shp):
            raise ValueError(f"{path}: {k} has shape {tuple(sd[k].shape)}, expected {shp}")
    return cfg, sd, tok
