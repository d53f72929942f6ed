"""ctypes binding of librs_engine.so (include/rs_engine.h) + weight packing.

PyTorch is used for device memory, streams and the one-time weight repack only; every
operation on the inference path is a hand-written sm_90a kernel behind the C ABI.  There
is deliberately no CPU or eager-PyTorch fallback: if the library or an H100 is missing the
constructors raise.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .config import ModelConfig, conv_out_len, xscale
from .logmel_tables import logmel_tables
from .weights import StateDict, rel_pos_table

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "librs_engine.so")

EPI_BIAS_BF16, EPI_BIAS_RELU_BF16, EPI_BIAS_SWISH_BF16, EPI_BIAS_GLU_BF16, EPI_RESID_F32, EPI_BIAS_F32, EPI_BIAS_F16, EPI_QKV_VT = range(8)


class RsModelConfig(C.Structure):
    _fields_ = [
        ("sample_rate", C.c_int32), ("n_window_size", C.c_int32), ("n_window_stride", C.c_int32),
        ("n_fft", C.c_int32), ("n_mels", C.c_int32),
        ("preemph", C.c_float), ("log_zero_guard", C.c_float), ("norm_eps", C.c_float),
        ("n_layers", C.c_int32), ("d_model", C.c_int32), ("n_heads", C.c_int32), ("d_ff", C.c_int32),
        ("conv_kernel", C.c_int32), ("sub_channels", C.c_int32),
        ("att_left", C.c_int32), ("att_right", C.c_int32), ("global_tokens", C.c_int32),
        ("xscale", C.c_float), ("ln_eps", C.c_float),
        ("vocab_size", C.c_int32), ("pred_hidden", C.c_int32), ("joint_hidden", C.c_int32), ("max_symbols", C.c_int32),
    ]


class RsTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dev_ptr", C.c_void_p), ("dtype", C.c_int32), ("numel", C.c_int64)]


_DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.int32: 2}
_lib = None

EXPORTS = [
    "rs_engine_create", "rs_engine_destroy", "rs_last_error", "rs_workspace_bytes", "rs_set_workspace",
    "rs_mel_frames", "rs_enc_frames", "rs_mel_valid", "rs_enc_valid", "rs_logmel", "rs_encode", "rs_rnnt_greedy", "rs_transcribe_device",
    "rs_transcribe_batch", "rs_transcribe_device_pcm16", "rs_transcribe_batch_pcm16", "rs_resample_mono", "rs_rnnt_alsd", "rs_gemm_bf16", "rs_layernorm", "rs_launch_count", "rs_enable_stage_timing",
    "rs_stage_times_ms", "rs_enable_gemm_timing", "rs_gemm_timing", "rs_debug_decode_cycles",
    "rs_enable_kernel_timing", "rs_kernel_timing", "rs_stage_rows",
    "rs_rnnt_greedy_confidence", "rs_transcribe_device_confidence", "rs_transcribe_batch_confidence",
    "rs_attention", "rs_conv_dw", "rs_sub_conv0_dw1", "rs_sub_dw", "rs_set_phrase_boosting",
    "rs_set_ngram_lm", "rs_ngram_lm_eval", "rs_rnnt_align", "rs_rnnt_align_lattice", "rs_rnnt_alsd_trace",
    "rs_stream_state_bytes", "rs_rnnt_greedy_resume", "rs_stream_step", "rs_set_boost_roots", "rs_rnnt_alsd_nbest", "rs_rnnt_maes", "rs_maes_last_rows",
    "rs_rnnt_align_segment", "rs_rnnt_spot", "rs_rnnt_spot_lattice", "rs_rnnt_align_banded", "rs_rnnt_align_banded_lattice",
    "rs_set_spot_keywords", "rs_spot_state_bytes", "rs_spot_max_hits", "rs_rnnt_spot_resume", "rs_stream_step_spot",
]

MAX_NBEST = 64                          # include/rs_engine.h RS_MAX_NBEST


# per-step buffers of rs_alsd_trace: (name, dtype, trailing shape); then the back-pointer tree, [B, node_pitch] each
ALSD_TRACE_STEP = [("n_hyp", torch.int32, ()), ("beam_score", torch.float64, ("beam",)), ("beam_u", torch.int32, ("beam",)),
                   ("beam_node", torch.int32, ("beam",)), ("row_t", torch.int32, ("beam",)), ("cand_logp", torch.float32, ("beam", 9)),
                   ("cand_tok", torch.int32, ("beam", 8)), ("has_final", torch.int32, ()), ("final_key", torch.float64, ()),
                   ("final_score", torch.float64, ())]
ALSD_TRACE_FIELDS = [n for n, _, _ in ALSD_TRACE_STEP] + ["node_parent", "node_tok", "node_step"]


class RsNgramLM(C.Structure):
    """include/rs_engine.h rs_ngram_lm"""
    _fields_ = [("order", C.c_int), ("n_states", C.c_int), ("n_arcs", C.c_int), ("pitch", C.c_int), ("start_state", C.c_int),
                ("cb", C.c_void_p), ("chain", C.c_void_p), ("arc_begin", C.c_void_p), ("arc_tok", C.c_void_p),
                ("arc_to", C.c_void_p), ("arc_w", C.c_void_p), ("uni_w", C.c_void_p), ("uni_to", C.c_void_p)]


class RsMaesParams(C.Structure):
    _fields_ = [("beam", C.c_int32), ("num_steps", C.c_int32), ("prefix_alpha", C.c_int32), ("expansion_beta", C.c_int32),
                ("expansion_gamma", C.c_float), ("score_norm", C.c_int32), ("recombine_returns_input", C.c_int32)]


class RsAlsdTrace(C.Structure):
    """include/rs_engine.h rs_alsd_trace"""
    _fields_ = [("max_steps", C.c_int32), ("node_pitch", C.c_int32)] + [(n, C.c_void_p) for n in ALSD_TRACE_FIELDS]


def load_library(build_if_missing: bool = True) -> C.CDLL:
    """dlopen librs_engine.so (building it with nvcc first if it is absent and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _LIB_PATH
    if not os.path.exists(_LIB_PATH):
        if not build_if_missing:
            raise FileNotFoundError(_LIB_PATH)
        from .build import build
        build()
    lib = C.CDLL(path)
    vp, ip, i32p, f32p = C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float)
    lib.rs_engine_create.argtypes = [C.POINTER(RsModelConfig), C.POINTER(RsTensor), ip, ip, C.POINTER(vp)]
    lib.rs_engine_create.restype = ip
    lib.rs_engine_destroy.argtypes = [vp]
    lib.rs_engine_destroy.restype = None
    lib.rs_last_error.argtypes = [vp]
    lib.rs_last_error.restype = C.c_char_p
    lib.rs_workspace_bytes.argtypes = [vp, ip, ip, C.POINTER(C.c_size_t)]
    lib.rs_set_workspace.argtypes = [vp, vp, C.c_size_t]
    lib.rs_mel_frames.argtypes = [vp, ip]
    lib.rs_enc_frames.argtypes = [vp, ip]
    lib.rs_mel_valid.argtypes = [vp, ip]
    lib.rs_enc_valid.argtypes = [vp, ip]
    lib.rs_logmel.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp]
    lib.rs_encode.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, vp]
    lib.rs_rnnt_greedy.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp, ip, vp]
    lib.rs_transcribe_device.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp, ip, vp]
    lib.rs_transcribe_batch.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp, ip, vp]
    lib.rs_transcribe_device_pcm16.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp, ip, vp]
    lib.rs_transcribe_batch_pcm16.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp, ip, vp]
    lib.rs_rnnt_greedy_confidence.argtypes = [vp, vp, vp, ip, ip, vp, vp, vp, ip, C.c_float, vp, vp]
    lib.rs_transcribe_device_confidence.argtypes = [vp, vp, ip, vp, ip, ip, vp, vp, vp, ip, C.c_float, vp, vp]
    lib.rs_transcribe_batch_confidence.argtypes = [vp, vp, ip, vp, ip, ip, vp, vp, vp, ip, C.c_float, vp, vp]
    lib.rs_set_phrase_boosting.argtypes = [vp, vp, vp, ip, ip]
    lib.rs_set_boost_roots.argtypes = [vp, vp, ip]
    lib.rs_set_ngram_lm.argtypes = [vp, C.POINTER(RsNgramLM)]
    lib.rs_ngram_lm_eval.argtypes = [vp, vp, vp, ip, vp, vp, vp]
    lib.rs_rnnt_alsd.argtypes = [vp, vp, vp, ip, ip, ip, C.c_double, ip, ip, vp, vp, vp, vp, ip, vp]
    lib.rs_rnnt_alsd.restype = ip
    lib.rs_rnnt_alsd_trace.argtypes = [vp, vp, vp, ip, ip, ip, C.c_double, ip, ip, vp, vp, vp, vp, ip, C.POINTER(RsAlsdTrace), vp]
    lib.rs_rnnt_alsd_trace.restype = ip
    lib.rs_rnnt_alsd_nbest.argtypes = [vp, vp, vp, ip, ip, ip, C.c_double, ip, ip, ip, vp, vp, vp, vp, vp, vp, vp, ip, vp]
    lib.rs_rnnt_alsd_nbest.restype = ip
    lib.rs_rnnt_maes.argtypes = [vp, vp, vp, ip, ip, C.POINTER(RsMaesParams), ip, vp, vp, vp, vp, vp, ip, vp]
    lib.rs_rnnt_maes.restype = ip
    lib.rs_maes_last_rows.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.rs_maes_last_rows.restype = ip
    lib.rs_rnnt_align.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, vp, vp, vp, vp, vp]
    lib.rs_rnnt_align.restype = ip
    lib.rs_rnnt_align_lattice.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, vp, vp, vp]
    lib.rs_rnnt_align_lattice.restype = ip
    lib.rs_rnnt_align_segment.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, vp, vp, vp, vp, vp, vp, vp]
    lib.rs_rnnt_align_segment.restype = ip
    lib.rs_rnnt_align_banded.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.rs_rnnt_align_banded.restype = ip
    lib.rs_rnnt_align_banded_lattice.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, vp, vp, vp, vp, vp]
    lib.rs_rnnt_align_banded_lattice.restype = ip
    lib.rs_rnnt_spot.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, ip, C.c_float, ip, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.rs_rnnt_spot.restype = ip
    lib.rs_rnnt_spot_lattice.argtypes = [vp, vp, vp, ip, ip, vp, vp, ip, ip, vp, vp, vp]
    lib.rs_rnnt_spot_lattice.restype = ip
    lib.rs_set_spot_keywords.argtypes = [vp, vp, vp, ip, ip, C.c_float, ip, ip, vp]
    lib.rs_spot_state_bytes.argtypes = [vp]
    lib.rs_spot_state_bytes.restype = C.c_size_t
    lib.rs_spot_max_hits.argtypes = [vp, ip]
    lib.rs_rnnt_spot_resume.argtypes = [vp, vp, vp, vp, vp, vp, vp, ip, ip, ip, ip, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.rs_stream_step_spot.argtypes = [vp, vp, ip, vp, vp, vp, vp, vp, ip, ip, vp, vp, vp, ip, C.c_float, vp, vp, vp, ip, ip,
                                        vp, vp, vp, vp, vp, vp]
    lib.rs_stream_state_bytes.argtypes = [vp]
    lib.rs_stream_state_bytes.restype = C.c_size_t
    lib.rs_rnnt_greedy_resume.argtypes = [vp, vp, vp, vp, vp, vp, ip, ip, vp, vp, vp, ip, C.c_float, vp, vp]
    lib.rs_rnnt_greedy_resume.restype = ip
    lib.rs_stream_step.argtypes = [vp, vp, ip, vp, vp, vp, vp, vp, ip, ip, vp, vp, vp, ip, C.c_float, vp, vp]
    lib.rs_stream_step.restype = ip
    lib.rs_resample_mono.argtypes = [vp, vp, ip, vp, ip, ip, ip, vp, ip, ip, ip, ip, ip, vp, ip, vp, vp]
    lib.rs_resample_mono.restype = ip
    lib.rs_gemm_bf16.argtypes = [vp, vp, vp, vp, vp, vp, ip, ip, ip, ip, C.c_float, vp, ip, ip, vp]
    lib.rs_layernorm.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, ip, ip, vp]
    lib.rs_attention.argtypes = [vp, vp, vp, ip, vp, vp, ip, vp, vp, vp, ip, ip, ip, ip, ip, ip, vp]
    lib.rs_conv_dw.argtypes = [vp, vp, vp, vp, vp, vp, ip, ip, ip, ip, vp]
    lib.rs_sub_conv0_dw1.argtypes = [vp, vp, vp, vp, ip, ip, ip, ip, vp, vp, vp, vp, vp, vp]
    lib.rs_sub_dw.argtypes = [vp, vp, vp, vp, vp, vp, ip, ip, ip, ip, ip, ip, ip, vp]
    lib.rs_launch_count.argtypes = [vp]
    lib.rs_launch_count.restype = C.c_int64
    lib.rs_enable_stage_timing.argtypes = [vp, ip]
    lib.rs_stage_times_ms.argtypes = [vp, f32p]
    lib.rs_debug_decode_cycles.argtypes = [vp, ip, ip, ip, C.POINTER(C.c_int64)]
    lib.rs_debug_decode_cycles.restype = ip
    lib.rs_stage_rows.argtypes = [vp, C.c_int64, C.POINTER(vp), C.POINTER(C.c_int64), i32p, ip, ip, C.c_int64, ip]
    lib.rs_stage_rows.restype = ip
    lib.rs_enable_kernel_timing.argtypes = [vp, ip]
    lib.rs_enable_kernel_timing.restype = ip
    lib.rs_kernel_timing.argtypes = [vp, C.c_char_p, ip]
    lib.rs_kernel_timing.restype = ip
    lib.rs_enable_gemm_timing.argtypes = [vp, ip]
    lib.rs_gemm_timing.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    for fn in ("rs_workspace_bytes", "rs_set_workspace", "rs_mel_frames", "rs_enc_frames", "rs_mel_valid", "rs_enc_valid", "rs_logmel", "rs_encode",
               "rs_rnnt_greedy", "rs_transcribe_device", "rs_transcribe_batch", "rs_transcribe_device_pcm16", "rs_transcribe_batch_pcm16",
               "rs_rnnt_greedy_confidence", "rs_transcribe_device_confidence", "rs_transcribe_batch_confidence",
               "rs_set_phrase_boosting", "rs_set_boost_roots", "rs_set_ngram_lm", "rs_ngram_lm_eval", "rs_gemm_bf16", "rs_layernorm", "rs_attention", "rs_conv_dw", "rs_sub_conv0_dw1", "rs_sub_dw",
               "rs_enable_stage_timing", "rs_stage_times_ms", "rs_enable_gemm_timing", "rs_gemm_timing"):
        getattr(lib, fn).restype = ip
    _lib = lib
    return lib


# --------------------------------------------------------------------------------------
# Weight packing (NeMo state dict -> the engine's named device tensors)
# --------------------------------------------------------------------------------------
def glu_interleave_index(d: int) -> torch.Tensor:
    """Row permutation of pointwise_conv1 so that each 32-column GEMM chunk holds 16 value rows
    followed by their 16 gate rows (RS_EPI_BIAS_GLU_BF16)."""
    blk = torch.arange(d // 16).repeat_interleave(32)
    within = torch.arange(32).repeat(d // 16)
    return torch.where(within < 16, blk * 16 + within, d + blk * 16 + within - 16)


def pack_weights(sd: StateDict, cfg: ModelConfig) -> Dict[str, torch.Tensor]:
    """NeMo-named fp32 state dict -> packed host tensors (bf16 GEMM weights, folded BN, ...)."""
    bf = lambda t: t.to(torch.bfloat16).contiguous()
    f32 = lambda t: t.to(torch.float32).contiguous()
    out: Dict[str, torch.Tensor] = dict(logmel_tables(cfg))
    d, H, dk, Cc = cfg.d_model, cfg.n_heads, cfg.d_head, cfg.sub_channels
    pe = "encoder.pre_encode."
    out["sub.conv0.w"] = f32(sd[pe + "conv.0.weight"].reshape(Cc, 9)); out["sub.conv0.b"] = f32(sd[pe + "conv.0.bias"])
    out["sub.dw1.w"] = f32(sd[pe + "conv.2.weight"].reshape(Cc, 9)); out["sub.dw1.b"] = f32(sd[pe + "conv.2.bias"])
    out["sub.pw1.w"] = bf(sd[pe + "conv.3.weight"].reshape(Cc, Cc)); out["sub.pw1.b"] = f32(sd[pe + "conv.3.bias"])
    out["sub.dw2.w"] = f32(sd[pe + "conv.5.weight"].reshape(Cc, 9)); out["sub.dw2.b"] = f32(sd[pe + "conv.5.bias"])
    out["sub.pw2.w"] = bf(sd[pe + "conv.6.weight"].reshape(Cc, Cc)); out["sub.pw2.b"] = f32(sd[pe + "conv.6.bias"])
    F3 = cfg.sub_freq
    # NeMo flattens [C, F3] channel-major (index c*F3+f); the engine's activations are [F3, C]
    out["sub.out.w"] = bf(sd[pe + "out.weight"].view(d, Cc, F3).permute(0, 2, 1).reshape(d, F3 * Cc))
    out["sub.out.b"] = f32(sd[pe + "out.bias"])
    table = rel_pos_table(cfg)
    glu_idx = glu_interleave_index(d)
    for i in range(cfg.n_layers):
        p, o = f"encoder.layers.{i}.", f"L{i}."
        for src, dst in (("norm_feed_forward1", "ln_ff1"), ("norm_self_att", "ln_att"), ("norm_conv", "ln_conv"),
                         ("norm_feed_forward2", "ln_ff2"), ("norm_out", "ln_out")):
            out[o + dst + ".g"] = f32(sd[p + src + ".weight"]); out[o + dst + ".b"] = f32(sd[p + src + ".bias"])
        for src, dst in (("feed_forward1", "ff1"), ("feed_forward2", "ff2")):
            out[o + dst + ".w1"] = bf(sd[p + src + ".linear1.weight"]); out[o + dst + ".b1"] = f32(sd[p + src + ".linear1.bias"])
            out[o + dst + ".w2"] = bf(sd[p + src + ".linear2.weight"]); out[o + dst + ".b2"] = f32(sd[p + src + ".linear2.bias"])
        a = p + "self_attn."
        out[o + "att.wqkv"] = bf(torch.cat([sd[a + "linear_q.weight"], sd[a + "linear_k.weight"], sd[a + "linear_v.weight"]], 0))
        # the q columns of the projection carry q + pos_bias_u (the content term (q+u).k is then a plain Q'K^T for the
        # tensor cores); the positional term and the global token, which want q + pos_bias_v resp. q, get u taken out again
        # through their own bias / in their own kernel
        u_flat = sd[a + "pos_bias_u"].reshape(-1)
        out[o + "att.bqkv"] = f32(torch.cat([sd[a + "linear_q.bias"] + u_flat, sd[a + "linear_k.bias"], sd[a + "linear_v.bias"]], 0))
        pos = torch.nn.functional.linear(table, sd[a + "linear_pos.weight"])          # input independent: once at load
        n_rel_pad = (cfg.n_rel + 31) // 32 * 32
        pos_h = torch.zeros(H, n_rel_pad, dk)
        pos_h[:, : cfg.n_rel] = pos.view(cfg.n_rel, H, dk).permute(1, 0, 2)
        out[o + "att.pos"] = bf(pos_h)                                                 # B operand of the batched BD GEMM
        # (q + v).p = (q + u).p + (v - u).p: the second term is input independent -> the GEMM's bias
        out[o + "att.bdbias"] = f32((out[o + "att.pos"].float() * (sd[a + "pos_bias_v"] - sd[a + "pos_bias_u"])[:, None, :]).sum(-1).reshape(-1))
        out[o + "att.u"] = f32(sd[a + "pos_bias_u"].reshape(-1))
        out[o + "att.wo"] = bf(sd[a + "linear_out.weight"]); out[o + "att.bo"] = f32(sd[a + "linear_out.bias"])
        c = p + "conv."
        out[o + "conv.pw1.w"] = bf(sd[c + "pointwise_conv1.weight"][:, :, 0][glu_idx])
        out[o + "conv.pw1.b"] = f32(sd[c + "pointwise_conv1.bias"][glu_idx])
        s = sd[c + "batch_norm.weight"] / torch.sqrt(sd[c + "batch_norm.running_var"] + cfg.bn_eps)
        out[o + "conv.dw.w"] = f32((sd[c + "depthwise_conv.weight"][:, 0, :] * s[:, None]).T)
        out[o + "conv.dw.shift"] = f32((sd[c + "depthwise_conv.bias"] - sd[c + "batch_norm.running_mean"]) * s + sd[c + "batch_norm.bias"])
        out[o + "conv.pw2.w"] = bf(sd[c + "pointwise_conv2.weight"][:, :, 0]); out[o + "conv.pw2.b"] = f32(sd[c + "pointwise_conv2.bias"])
    l = "decoder.prediction.dec_rnn.lstm."
    out["joint.enc.w"] = bf(sd["joint.enc.weight"]); out["joint.enc.b"] = f32(sd["joint.enc.bias"])
    out["joint.out.w"] = bf(sd["joint.joint_net.2.weight"]); out["joint.out.b"] = f32(sd["joint.joint_net.2.bias"])
    out["pred.embed"] = f32(sd["decoder.prediction.embed.weight"])
    out["pred.lstm.w"] = bf(torch.cat([sd[l + "weight_ih_l0"], sd[l + "weight_hh_l0"]], 1))
    out["pred.lstm.b"] = f32(sd[l + "bias_ih_l0"] + sd[l + "bias_hh_l0"])
    # the input half of the LSTM gates is a function of the token alone: one row per token (decode_spec.cu), from the same
    # bf16-rounded W_ih the kernels multiply with, accumulated in fp32
    w_ih = sd[l + "weight_ih_l0"].to(torch.bfloat16).to(torch.float32)
    out["pred.gate_tab"] = f32(out["pred.embed"] @ w_ih.T + out["pred.lstm.b"])
    out["joint.pred.w"] = bf(sd["joint.pred.weight"]); out["joint.pred.b"] = f32(sd["joint.pred.bias"])
    return out


def alsd_tensors(packed: Dict[str, torch.Tensor], cfg: ModelConfig) -> Dict[str, torch.Tensor]:
    """Weights of the ALSD beam search (csrc/decode_alsd.cu): the predictor / joint matrices repeated three times along K, so
    that activations split into three bf16 terms (24 mantissa bits) meet bf16-exact weights -- fp32-accurate log-probabilities
    out of the bf16 tensor-core GEMM.  The output layer is padded to a multiple of 64 rows (zero rows, never read)."""
    nc, hj = cfg.vocab_size + 1, cfg.joint_hidden
    n_pad = (nc + 63) // 64 * 64
    w = torch.zeros(n_pad, hj, dtype=torch.bfloat16)
    w[:nc] = packed["joint.out.w"]
    b = torch.zeros(n_pad, dtype=torch.float32)
    b[:nc] = packed["joint.out.b"]
    return {"alsd.out.w3": torch.cat([w] * 3, dim=1).contiguous(), "alsd.out.b": b,
            "alsd.lstm.w3": torch.cat([packed["pred.lstm.w"]] * 3, dim=1).contiguous(),
            "alsd.pred.w3": torch.cat([packed["joint.pred.w"]] * 3, dim=1).contiguous()}


def resample_taps(orig_sr: int, target_sr: int):
    """The polyphase FIR of ``scipy.signal.resample_poly(x, up, down)`` (its default Kaiser-5 window design, restated here
    step by step) in the layout rs_resample_mono wants: (taps float32 [up, taps_per_phase], up, down, n_pre_remove).
    out[m] = sum_j taps[phase][j] * x[n_hi - j] with t = (m + n_pre_remove) * down, n_hi = t // up, phase = t % up."""
    from math import gcd
    from scipy.signal import firwin
    g = gcd(int(orig_sr), int(target_sr))
    up, down = int(target_sr) // g, int(orig_sr) // g
    if up == down == 1:                                  # already at the target rate: the identity filter (down-mix / padding only)
        return torch.ones(1, 1, dtype=torch.float32), 1, 1, 0
    max_rate = max(up, down)
    half_len = 10 * max_rate
    h = (firwin(2 * half_len + 1, 1.0 / max_rate, window=("kaiser", 5.0)) * up).astype(np.float32)
    n_pre_pad = down - half_len % down
    n_pre_remove = (half_len + n_pre_pad) // down
    hp = np.concatenate((np.zeros(n_pre_pad, np.float32), h))
    per = (len(hp) + up - 1) // up
    taps = np.zeros((up, per), np.float32)
    for p in range(up):
        col = hp[p::up]
        taps[p, : len(col)] = col
    return torch.from_numpy(taps), up, down, n_pre_remove


def to_rs_config(cfg: ModelConfig) -> RsModelConfig:
    return RsModelConfig(
        cfg.sample_rate, cfg.n_window_size, cfg.n_window_stride, cfg.n_fft, cfg.n_mels,
        cfg.preemph, cfg.log_zero_guard, cfg.norm_eps,
        cfg.n_layers, cfg.d_model, cfg.n_heads, cfg.d_ff, cfg.conv_kernel, cfg.sub_channels,
        cfg.att_left, cfg.att_right, cfg.global_tokens, xscale(cfg), cfg.ln_eps,
        cfg.vocab_size, cfg.pred_hidden, cfg.joint_hidden, cfg.max_symbols)


# --------------------------------------------------------------------------------------
# Engine
# --------------------------------------------------------------------------------------
class Engine:
    """One engine per device: packed weights + workspace + the C-ABI handle."""

    def __init__(self, cfg: ModelConfig, state_dict: Optional[StateDict], device: str = "cuda", packed: Optional[Dict[str, torch.Tensor]] = None,
                 alsd: bool = False):
        """``packed``: the result of ``pack_weights(state_dict, cfg)`` when several engines share one checkpoint (one replica
        per device): the repack is done once, every engine uploads its own copy."""
        if not torch.cuda.is_available():
            raise RuntimeError("reazonspeech_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = load_library()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"device {device!r}: the engine has no CPU path")
        self.dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", self.dev_index)
        if packed is None:
            packed = pack_weights(state_dict, cfg)
        if alsd and "alsd.out.w3" not in packed:             # beam search wanted: +34 MB of tripled predictor / joint weights
            packed = dict(packed, **alsd_tensors(packed, cfg))
        self.weights = {k: v.to(self.device) for k, v in packed.items()}
        self._names = [k.encode() for k in self.weights]
        arr = (RsTensor * len(self.weights))()
        for i, (k, v) in enumerate(self.weights.items()):
            arr[i] = RsTensor(self._names[i], v.data_ptr(), _DTYPES[v.dtype], v.numel())
        self._rs_cfg = to_rs_config(cfg)
        h = C.c_void_p()
        rc = self.lib.rs_engine_create(C.byref(self._rs_cfg), arr, len(self.weights), self.dev_index, C.byref(h))
        if rc != 0:
            raise RuntimeError(f"rs_engine_create failed ({rc}): {self.lib.rs_last_error(None).decode()}")
        self.h = h
        self._ws: Optional[torch.Tensor] = None
        self._ws_key: Tuple[int, int] = (0, 0)
        self._boost: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
        self._lm: Optional[Dict[str, torch.Tensor]] = None

    def __del__(self):
        h = getattr(self, "h", None)
        if h:
            self.lib.rs_engine_destroy(h)
            self.h = None

    # -- helpers
    def _check(self, rc: int, what: str):
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.lib.rs_last_error(self.h).decode()}")

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def ensure_workspace(self, B: int, L_max: int):
        if self._ws is not None and B <= self._ws_key[0] and L_max <= self._ws_key[1]:
            return
        B2, L2 = max(B, self._ws_key[0]), max(L_max, self._ws_key[1])
        n = C.c_size_t()
        self._check(self.lib.rs_workspace_bytes(self.h, B2, L2, C.byref(n)), "rs_workspace_bytes")
        self._ws = None
        self._ws = torch.empty(n.value + 256, dtype=torch.uint8, device=self.device)
        ptr = (self._ws.data_ptr() + 255) // 256 * 256
        self._check(self.lib.rs_set_workspace(self.h, ptr, n.value), "rs_set_workspace")
        self._ws_key = (B2, L2)

    def set_phrase_boosting(self, bonus, next_state=None):
        """Phrase boosting of every greedy decode (rs_set_phrase_boosting): ``bonus`` float32 / ``next_state`` int32, both
        [n_states, pitch] (``boosting.PhraseBoostingTables`` fields; host or device tensors / arrays), or ``None`` to clear.
        The engine keeps its device copies alive while they are set; replacing or clearing a table first waits for the work
        queued on this device's current stream, which may still read the old one."""
        if bonus is None:
            new = None
        else:
            bonus_d = torch.as_tensor(bonus).to(self.device, torch.float32).contiguous()
            next_d = torch.as_tensor(next_state).to(self.device, torch.int32).contiguous()
            if bonus_d.dim() != 2 or bonus_d.shape != next_d.shape:
                raise ValueError(f"bonus and next must be [n_states, pitch] tensors of one shape, got {tuple(bonus_d.shape)} and {tuple(next_d.shape)}")
            new = (bonus_d, next_d)
        if self._boost is not None:
            torch.cuda.current_stream(self.device).synchronize()
        if new is None:
            self._check(self.lib.rs_set_phrase_boosting(self.h, None, None, 0, 0), "rs_set_phrase_boosting")
        else:
            self._check(self.lib.rs_set_phrase_boosting(self.h, new[0].data_ptr(), new[1].data_ptr(), new[0].shape[0], new[0].shape[1]),
                        "rs_set_phrase_boosting")
        self._boost = new

    def set_boost_roots(self, roots) -> None:
        """Per-row roots of the phrase-boosting table (rs_set_boost_roots): row b of every following greedy call starts at
        ``roots[b]`` (a table from ``boosting.combine_tables``), or ``None`` / empty to clear.  A host-side setting: the roots are
        copied to the device on each decode's stream."""
        r = np.ascontiguousarray(np.asarray([] if roots is None else roots, dtype=np.int32).reshape(-1))
        self._check(self.lib.rs_set_boost_roots(self.h, r.ctypes.data if r.size else None, int(r.size)), "rs_set_boost_roots")

    def set_ngram_lm(self, tables) -> None:
        """n-gram LM shallow fusion of every greedy decode and ``maes`` search (rs_set_ngram_lm): ``tables`` an ``ngram_lm.NgramLMTables``, or
        ``None`` to clear.  The engine keeps its device copies alive while they are set; replacing or clearing a table first
        waits for the work queued on this device's current stream, which may still read the old one."""
        new = None
        if tables is not None:
            dtypes = {"cb": torch.float32, "arc_w": torch.float32, "uni_w": torch.float32}
            new = {k: torch.as_tensor(v).to(self.device, dtypes.get(k, torch.int32)).contiguous()
                   for k, v in tables.device_arrays().items()}
            lm = RsNgramLM(int(tables.order), int(tables.n_states), int(tables.n_arcs), int(tables.pitch), int(tables.start_state),
                           *[new[k].data_ptr() for k in ("cb", "chain", "arc_begin", "arc_tok", "arc_to", "arc_w", "uni_w", "uni_to")])
        if self._lm is not None:
            torch.cuda.current_stream(self.device).synchronize()
        self._check(self.lib.rs_set_ngram_lm(self.h, None if new is None else C.byref(lm)), "rs_set_ngram_lm")
        self._lm = new

    def ngram_lm_eval(self, states: torch.Tensor, tokens: torch.Tensor):
        """The decode kernel's LM lookup on (state, token) pairs (rs_ngram_lm_eval) -> (score f32, next i32) device tensors."""
        states = states.to(self.device, torch.int32).contiguous()
        tokens = tokens.to(self.device, torch.int32).contiguous()
        score = torch.empty(states.shape, dtype=torch.float32, device=self.device)
        nxt = torch.empty(states.shape, dtype=torch.int32, device=self.device)
        self._check(self.lib.rs_ngram_lm_eval(self.h, states.data_ptr(), tokens.data_ptr(), states.numel(), score.data_ptr(),
                                              nxt.data_ptr(), self._stream()), "rs_ngram_lm_eval")
        return score, nxt

    def mel_frames(self, n: int) -> int:
        return self.lib.rs_mel_frames(self.h, n)

    def enc_frames(self, n: int) -> int:
        return self.lib.rs_enc_frames(self.h, n)

    def u_max(self, L_max: int) -> int:
        return self.enc_frames(L_max) * self.cfg.max_symbols

    @property
    def launch_count(self) -> int:
        return int(self.lib.rs_launch_count(self.h))

    # -- stages (device tensors in, device tensors out)
    def log_mel(self, wav: torch.Tensor, lens: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        B, L = wav.shape
        assert wav.dtype == torch.float32 and wav.is_contiguous() and lens.dtype == torch.int32
        self.ensure_workspace(B, L)                  # the per-feature statistics are reduced in the workspace
        F = self.mel_frames(L)
        mel = torch.empty(B, F, self.cfg.n_mels, dtype=torch.float32, device=self.device)
        mel_len = torch.empty(B, dtype=torch.int32, device=self.device)
        self._check(self.lib.rs_logmel(self.h, wav.data_ptr(), lens.data_ptr(), B, L, mel.data_ptr(), mel_len.data_ptr(),
                                       self._stream()), "rs_logmel")
        return mel, mel_len

    def encode(self, mel: torch.Tensor, mel_len: torch.Tensor, n_layers: int = -1) -> Tuple[torch.Tensor, torch.Tensor]:
        B, F, _ = mel.shape
        L = (F - 1) * self.cfg.n_window_stride
        self.ensure_workspace(B, L)
        T = self.enc_frames(L)                       # capacity of the padded encoder tensors (a multiple of 8)
        enc = torch.empty(B, T, self.cfg.d_model, dtype=torch.float32, device=self.device)
        enc_len = torch.empty(B, dtype=torch.int32, device=self.device)
        self._check(self.lib.rs_encode(self.h, mel.data_ptr(), mel_len.data_ptr(), B, F, enc.data_ptr(), enc_len.data_ptr(),
                                       n_layers, self._stream()), "rs_encode")
        return enc, enc_len

    def greedy(self, enc: torch.Tensor, enc_len: torch.Tensor, U_max: Optional[int] = None, alpha: Optional[float] = None):
        """-> (tokens, frames, n_tok), plus stats f32 [B, U, 4] = (lp, H1, A_alpha, G_alpha) per stored token when ``alpha`` is
        given (rs_rnnt_greedy_confidence; the tokens are the same either way)."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous()
        self.ensure_workspace(B, (T * 8 + 8) * self.cfg.n_window_stride)
        U = U_max or T * self.cfg.max_symbols
        tokens = torch.zeros(B, U, dtype=torch.int32, device=self.device)
        frames = torch.zeros(B, U, dtype=torch.int32, device=self.device)
        ntok = torch.zeros(B, dtype=torch.int32, device=self.device)
        if alpha is None:
            self._check(self.lib.rs_rnnt_greedy(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, tokens.data_ptr(),
                                                frames.data_ptr(), ntok.data_ptr(), U, self._stream()), "rs_rnnt_greedy")
            return tokens, frames, ntok
        stats = torch.zeros(B, U, 4, dtype=torch.float32, device=self.device)
        self._check(self.lib.rs_rnnt_greedy_confidence(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, tokens.data_ptr(), frames.data_ptr(),
                                                       ntok.data_ptr(), U, float(alpha), stats.data_ptr(), self._stream()), "rs_rnnt_greedy_confidence")
        return tokens, frames, ntok, stats

    @property
    def stream_state_bytes(self) -> int:
        """Bytes of one stream's decoder-state record (rs_stream_state_bytes; streaming.py)."""
        return int(self.lib.rs_stream_state_bytes(self.h))

    def greedy_resume(self, enc: torch.Tensor, dec_begin: torch.Tensor, dec_end: torch.Tensor, slot: torch.Tensor, states: torch.Tensor,
                      U_max: Optional[int] = None, alpha: Optional[float] = None):
        """The resumed greedy decode (rs_rnnt_greedy_resume): row b decodes frames [dec_begin[b], dec_end[b]) of ``enc`` from record
        ``states[slot[b]]`` (device uint8 [n_records, stream_state_bytes]) and stores its state there -> (tokens, frames, n_tok),
        plus stats [B, U, 4] with ``alpha``.  Slots must be distinct."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous()
        assert states.dtype == torch.uint8 and states.is_contiguous() and states.shape[-1] == self.stream_state_bytes
        args = [a.to(self.device, torch.int32).contiguous() for a in (dec_begin, dec_end, slot)]
        self.ensure_workspace(B, (T * 8 + 8) * self.cfg.n_window_stride)
        U = U_max or T * self.cfg.max_symbols
        tokens = torch.zeros(B, U, dtype=torch.int32, device=self.device)
        frames = torch.zeros(B, U, dtype=torch.int32, device=self.device)
        ntok = torch.zeros(B, dtype=torch.int32, device=self.device)
        stats = torch.zeros(B, U, 4, dtype=torch.float32, device=self.device) if alpha is not None else None
        self._check(self.lib.rs_rnnt_greedy_resume(self.h, enc.data_ptr(), args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(),
                                                   states.data_ptr(), B, T, tokens.data_ptr(), frames.data_ptr(), ntok.data_ptr(), U,
                                                   float(alpha or 0.0), None if stats is None else stats.data_ptr(), self._stream()),
                    "rs_rnnt_greedy_resume")
        return (tokens, frames, ntok) if stats is None else (tokens, frames, ntok, stats)

    def stream_step(self, wav: torch.Tensor, lens: torch.Tensor, dec_begin: torch.Tensor, dec_end: torch.Tensor, slot: torch.Tensor,
                    states: torch.Tensor, U_max: int, out, alpha: Optional[float] = None):
        """One streaming step over host buffers (rs_stream_step): ``wav`` host float32 or int16 [B, L] (the rows' buffers), ``lens``,
        ``dec_begin``, ``dec_end``, ``slot`` host int32 [B], ``states`` the device records -> ``out`` (host tokens [B, U],
        frames [B, U], n_tok [B], and stats [B, U, 4] with ``alpha``) filled; synchronises."""
        B, L = wav.shape
        assert wav.device.type == "cpu" and wav.dtype in (torch.float32, torch.int16) and wav.is_contiguous()
        assert states.dtype == torch.uint8 and states.is_contiguous() and states.shape[-1] == self.stream_state_bytes
        host = [a.to(torch.int32).contiguous() for a in (lens, dec_begin, dec_end, slot)]
        assert all(a.device.type == "cpu" for a in host)
        self.ensure_workspace(B, L)
        tokens, frames, ntok = out[:3]
        self._check(self.lib.rs_stream_step(self.h, wav.data_ptr(), int(wav.dtype == torch.int16), host[0].data_ptr(), host[1].data_ptr(),
                                            host[2].data_ptr(), host[3].data_ptr(), states.data_ptr(), B, L, tokens.data_ptr(),
                                            frames.data_ptr(), ntok.data_ptr(), U_max, float(alpha or 0.0),
                                            out[3].data_ptr() if alpha is not None else None, self._stream()), "rs_stream_step")
        return out

    # -- streaming keyword spotting (keywords.py, "Streaming")
    def set_spot_keywords(self, keywords: Sequence[Sequence[int]], threshold: float, delay_frames: int, chunk_frames: int) -> None:
        """Install the keyword set of the streaming spot (rs_set_spot_keywords): token-id lists of 1..32 ids, the threshold, the
        delay D and the chunk C in frames; the keywords' predictor rows are computed once, here.  An empty list clears the set."""
        self._spot_owner = None                  # whoever installs a set claims it afterwards (StreamingTranscriber)
        if not keywords:
            self._check(self.lib.rs_set_spot_keywords(self.h, None, None, 0, 1, 0.0, 0, 1, self._stream()), "rs_set_spot_keywords")
            self._spot_U = self._spot_kw = 0
            return
        U = max(len(k) for k in keywords)
        labels = np.zeros((len(keywords), max(U, 1)), dtype=np.int32)
        for i, k in enumerate(keywords):
            labels[i, : len(k)] = k
        lens = np.array([len(k) for k in keywords], dtype=np.int32)
        self._check(self.lib.rs_set_spot_keywords(self.h, labels.ctypes.data, lens.ctypes.data, len(keywords), max(U, 1), float(threshold),
                                                  int(delay_frames), int(chunk_frames), self._stream()), "rs_set_spot_keywords")
        self._spot_U, self._spot_kw = max(U, 1), len(keywords)

    def _check_records(self, records: torch.Tensor) -> None:
        """The spot records must be uint8 [n_slots, n_kw of the installed set, spot_state_bytes] on this device: the kernels
        index them as [slot][keyword]."""
        n_kw = getattr(self, "_spot_kw", 0)
        if not (records.dtype == torch.uint8 and records.is_contiguous() and records.dim() == 3 and records.device == self.device
                and records.shape[1] == n_kw and records.shape[2] == self.spot_state_bytes and n_kw > 0):
            raise ValueError(f"spot records must be contiguous uint8 [n_slots, {n_kw}, {self.spot_state_bytes}] on {self.device} "
                             f"(the installed keyword set), got {records.dtype} {tuple(records.shape)} on {records.device}")

    @property
    def spot_state_bytes(self) -> int:
        """Bytes of one (stream, keyword) record of the installed set (rs_spot_state_bytes; 0 without a set)."""
        return int(self.lib.rs_spot_state_bytes(self.h))

    def _spot_outputs(self, B: int):
        n = int(self.lib.rs_spot_max_hits(self.h, B))
        U = getattr(self, "_spot_U", 0) or 1
        cached = getattr(self, "_spot_out", None)
        if cached is None or cached[0].shape[0] < n or cached[2].shape[1] != U:
            cached = (np.empty((max(n, 1), 5), np.int32), np.empty((max(n, 1), 2), np.float32), np.empty((max(n, 1), U), np.int32),
                      np.empty((max(n, 1), U), np.float32), np.zeros(1, np.int32))
            self._spot_out = cached
        return cached

    @staticmethod
    def _spot_hits(out):
        n = int(out[4][0])
        return tuple(a[:n].copy() for a in out[:4])

    def spot_resume(self, enc: torch.Tensor, dec_begin: torch.Tensor, dec_end: torch.Tensor, slot: torch.Tensor, last: torch.Tensor,
                    records: torch.Tensor, scores: bool = False):
        """The resumed keyword spot (rs_rnnt_spot_resume): row b continues its stream from records[slot[b]] (device uint8
        [n_slots, n_kw, spot_state_bytes]) over frames [dec_begin[b], dec_end[b]) of ``enc`` -> the decided hits as host arrays
        (meta i32 [n, 5] = (row, keyword, s, e, forced), val f32 [n, 2] = (score, confidence), frames i32 [n, U], token_lp
        f32 [n, U]) sorted by (row, keyword, e); with ``scores`` also E f32 / S i32 [B, n_kw, T] (NaN / -1 outside the ranges)
        and sigma i32 [B, n_kw] device tensors."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous()
        self._check_records(records)
        n_kw = records.shape[1]
        args = [a.to(self.device, torch.int32).contiguous() for a in (dec_begin, dec_end, slot, last)]
        out = self._spot_outputs(B)
        E = torch.full((B, n_kw, T), float("nan"), device=self.device) if scores else None
        S = torch.full((B, n_kw, T), -1, dtype=torch.int32, device=self.device) if scores else None
        sigma = torch.full((B, n_kw), -2, dtype=torch.int32, device=self.device) if scores else None
        ptr = lambda x: None if x is None else x.data_ptr()
        self._check(self.lib.rs_rnnt_spot_resume(self.h, enc.data_ptr(), *[a.data_ptr() for a in args], records.data_ptr(), records.shape[0],
                                                 B, T, out[0].shape[0], *[a.ctypes.data for a in out], ptr(E), ptr(S), ptr(sigma),
                                                 self._stream()), "rs_rnnt_spot_resume")
        hits = self._spot_hits(out)
        return hits + (E, S, sigma) if scores else hits

    def stream_step_spot(self, wav: torch.Tensor, lens: torch.Tensor, dec_begin: torch.Tensor, dec_end: torch.Tensor, slot: torch.Tensor,
                         states: torch.Tensor, U_max: int, out, last: torch.Tensor, records: torch.Tensor, alpha: Optional[float] = None):
        """``stream_step`` plus the resumed keyword spot on the same joint.enc rows (rs_stream_step_spot): ``last`` host int32 [B]
        (row b decodes its stream's last frame), ``records`` the spot records -> the decided hits as ``spot_resume`` returns them;
        ``out`` is filled as ``stream_step`` fills it."""
        B, L = wav.shape
        assert wav.device.type == "cpu" and wav.dtype in (torch.float32, torch.int16) and wav.is_contiguous()
        assert states.dtype == torch.uint8 and states.is_contiguous() and states.shape[-1] == self.stream_state_bytes
        self._check_records(records)
        host = [a.to(torch.int32).contiguous() for a in (lens, dec_begin, dec_end, slot, last)]
        assert all(a.device.type == "cpu" for a in host)
        self.ensure_workspace(B, L)
        tokens, frames, ntok = out[:3]
        hits = self._spot_outputs(B)
        self._check(self.lib.rs_stream_step_spot(self.h, wav.data_ptr(), int(wav.dtype == torch.int16), host[0].data_ptr(), host[1].data_ptr(),
                                                 host[2].data_ptr(), host[3].data_ptr(), states.data_ptr(), B, L, tokens.data_ptr(),
                                                 frames.data_ptr(), ntok.data_ptr(), U_max, float(alpha or 0.0),
                                                 out[3].data_ptr() if alpha is not None else None, host[4].data_ptr(), records.data_ptr(),
                                                 records.shape[0], hits[0].shape[0], *[a.ctypes.data for a in hits], self._stream()),
                    "rs_stream_step_spot")
        return self._spot_hits(hits)

    def transcribe_device(self, wav: torch.Tensor, lens: torch.Tensor, U_max: Optional[int] = None, out=None, alpha: Optional[float] = None):
        """With ``alpha``: also the confidence statistics (``greedy``), ``out`` then holds four tensors."""
        B, L = wav.shape
        self.ensure_workspace(B, L)
        U = U_max or self.u_max(L)
        if out is None:
            out = (torch.zeros(B, U, dtype=torch.int32, device=self.device),
                   torch.zeros(B, U, dtype=torch.int32, device=self.device),
                   torch.zeros(B, dtype=torch.int32, device=self.device))
            if alpha is not None:
                out += (torch.zeros(B, U, 4, dtype=torch.float32, device=self.device),)
        tokens, frames, ntok = out[:3]
        assert wav.dtype in (torch.float32, torch.int16) and wav.is_contiguous()
        if alpha is not None:
            self._check(self.lib.rs_transcribe_device_confidence(self.h, wav.data_ptr(), int(wav.dtype == torch.int16), lens.data_ptr(), B, L,
                                                                 tokens.data_ptr(), frames.data_ptr(), ntok.data_ptr(), U, float(alpha),
                                                                 out[3].data_ptr(), self._stream()), "rs_transcribe_device_confidence")
            return tokens, frames, ntok, out[3]
        fn, name = ((self.lib.rs_transcribe_device_pcm16, "rs_transcribe_device_pcm16") if wav.dtype == torch.int16
                    else (self.lib.rs_transcribe_device, "rs_transcribe_device"))        # int16: PCM, scaled by 2^-15 on the device
        self._check(fn(self.h, wav.data_ptr(), lens.data_ptr(), B, L, tokens.data_ptr(), frames.data_ptr(), ntok.data_ptr(), U, self._stream()), name)
        return tokens, frames, ntok

    def transcribe_host(self, wav: torch.Tensor, lens: torch.Tensor, U_max: Optional[int] = None, out=None, alpha: Optional[float] = None):
        """wav: host float32 or int16 (PCM) [B, L] (pinned for speed), lens: host int32 [B] -> host tokens/frames/n_tok, plus
        the confidence statistics [B, U, 4] when ``alpha`` is given (``out`` then holds four tensors)."""
        B, L = wav.shape
        assert wav.device.type == "cpu" and wav.dtype in (torch.float32, torch.int16) and wav.is_contiguous()
        self.ensure_workspace(B, L)
        U = U_max or self.u_max(L)
        if out is None:
            out = (torch.zeros(B, U, dtype=torch.int32).pin_memory(), torch.zeros(B, U, dtype=torch.int32).pin_memory(),
                   torch.zeros(B, dtype=torch.int32).pin_memory())
            if alpha is not None:
                out += (torch.zeros(B, U, 4, dtype=torch.float32).pin_memory(),)
        tokens, frames, ntok = out[:3]
        if alpha is not None:
            self._check(self.lib.rs_transcribe_batch_confidence(self.h, wav.data_ptr(), int(wav.dtype == torch.int16), lens.data_ptr(), B, L,
                                                                tokens.data_ptr(), frames.data_ptr(), ntok.data_ptr(), U, float(alpha),
                                                                out[3].data_ptr(), self._stream()), "rs_transcribe_batch_confidence")
            return tokens, frames, ntok, out[3]
        fn, name = ((self.lib.rs_transcribe_batch_pcm16, "rs_transcribe_batch_pcm16") if wav.dtype == torch.int16
                    else (self.lib.rs_transcribe_batch, "rs_transcribe_batch"))
        self._check(fn(self.h, wav.data_ptr(), lens.data_ptr(), B, L, tokens.data_ptr(), frames.data_ptr(), ntok.data_ptr(), U, self._stream()), name)
        return tokens, frames, ntok

    def alsd(self, enc: torch.Tensor, enc_len: torch.Tensor, beam: int = 4, u_max_ratio: float = 2.0, score_norm: bool = True,
             recombine_returns_input: bool = True, U_cap: Optional[int] = None):
        """ALSD beam search over encoder outputs -> (y [B, U_cap + 1] with the leading blank, steps [B, U_cap], n [B], score [B])."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous() and enc_len.dtype == torch.int32
        U = U_cap or (T + int(u_max_ratio * T) + 1)
        y = torch.zeros(B, U + 1, dtype=torch.int32, device=self.device)
        steps = torch.zeros(B, U, dtype=torch.int32, device=self.device)
        n = torch.zeros(B, dtype=torch.int32, device=self.device)
        score = torch.zeros(B, dtype=torch.float64, device=self.device)
        self._check(self.lib.rs_rnnt_alsd(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, int(beam), float(u_max_ratio), int(score_norm),
                                          int(recombine_returns_input), y.data_ptr(), steps.data_ptr(), n.data_ptr(), score.data_ptr(), U,
                                          self._stream()), "rs_rnnt_alsd")
        return y, steps, n, score

    def alsd_nbest(self, enc: torch.Tensor, enc_len: torch.Tensor, n_best: int, beam: int = 4, u_max_ratio: float = 2.0,
                   score_norm: bool = True, recombine_returns_input: bool = True, U_cap: Optional[int] = None):
        """The N-best list of the ALSD search (rs_rnnt_alsd_nbest), best first -> (y [B, N, U_cap + 1] with the leading blank,
        steps [B, N, U_cap], n [B, N], score [B, N], count [B], pool [B], from_final [B]) device tensors; entries at or past
        count[b] stay zero.  Entry 0 is what ``alsd`` returns."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous() and enc_len.dtype == torch.int32
        N = int(n_best)
        U = U_cap or (T + int(u_max_ratio * T) + 1)
        y, steps, n, count, pool, from_final = [torch.zeros(*shape, dtype=torch.int32, device=self.device)
                                                for shape in ((B, N, U + 1), (B, N, U), (B, N), (B,), (B,), (B,))]
        score = torch.zeros(B, N, dtype=torch.float64, device=self.device)
        self._check(self.lib.rs_rnnt_alsd_nbest(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, int(beam), float(u_max_ratio), int(score_norm),
                                                int(recombine_returns_input), N, y.data_ptr(), steps.data_ptr(), n.data_ptr(), score.data_ptr(),
                                                count.data_ptr(), pool.data_ptr(), from_final.data_ptr(), U, self._stream()), "rs_rnnt_alsd_nbest")
        return y, steps, n, score, count, pool, from_final

    def maes(self, enc: torch.Tensor, enc_len: torch.Tensor, beam: int = 4, n_best: int = 1, num_steps: int = 2, prefix_alpha: int = 1,
             expansion_beta: int = 2, expansion_gamma: float = 2.3, score_norm: bool = True, recombine_returns_input: bool = True,
             U_cap: Optional[int] = None):
        """MAES beam search over encoder outputs (rs_rnnt_maes), fused with the n-gram LM while one is set -> NeMo's sort_nbest
        list, best first: (y [B, N, U_cap + 1] with the leading blank, frames [B, N, U_cap], n [B, N], score [B, N], count [B])
        device tensors; entries at or past count[b] stay zero."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous() and enc_len.dtype == torch.int32
        N = int(n_best)
        U = U_cap or (T * int(num_steps) + 1)
        y, frames, n, count = [torch.zeros(*shape, dtype=torch.int32, device=self.device) for shape in ((B, N, U + 1), (B, N, U), (B, N), (B,))]
        score = torch.zeros(B, N, dtype=torch.float64, device=self.device)
        p = RsMaesParams(int(beam), int(num_steps), int(prefix_alpha), int(expansion_beta), float(expansion_gamma), int(score_norm),
                         int(recombine_returns_input))
        self._check(self.lib.rs_rnnt_maes(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, C.byref(p), N, y.data_ptr(), frames.data_ptr(),
                                          n.data_ptr(), score.data_ptr(), count.data_ptr(), U, self._stream()), "rs_rnnt_maes")
        return y, frames, n, score, count

    def maes_last_rows(self) -> Tuple[int, int]:
        """(expansion rows run through the predictor, frames searched) of the last ``maes`` call (rs_maes_last_rows)."""
        rows, frames = C.c_int64(), C.c_int64()
        self._check(self.lib.rs_maes_last_rows(self.h, C.byref(rows), C.byref(frames)), "rs_maes_last_rows")
        return rows.value, frames.value

    def alsd_trace(self, enc: torch.Tensor, enc_len: torch.Tensor, beam: int = 4, u_max_ratio: float = 2.0, score_norm: bool = True,
                   recombine_returns_input: bool = True, U_cap: Optional[int] = None, max_steps: Optional[int] = None):
        """``alsd`` through the trace seam (rs_rnnt_alsd_trace) -> dict of CPU tensors: y, steps, n, score as ``alsd`` returns
        them; per recorded step i: n_hyp [S, B], beam_score / beam_u / beam_node / row_t [S, B, beam], cand_logp [S, B, beam, 9], cand_tok
        [S, B, beam, 8], has_final / final_key / final_score [S, B]; the back-pointer tree node_parent / node_tok / node_step
        [B, node_pitch].  S = the steps the search ran (at most ``max_steps``, default all it may run)."""
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous() and enc_len.dtype == torch.int32
        total_steps = T + int(u_max_ratio * T)
        S = total_steps + 1 if max_steps is None else int(max_steps)
        U = U_cap or (total_steps + 1)
        node_pitch = 1 + beam * (total_steps + 1)
        dims = {"beam": beam}
        buf = {n: torch.full((max(S, 1), B) + tuple(dims.get(d, d) for d in shape), -1, dtype=dt, device=self.device)
               for n, dt, shape in ALSD_TRACE_STEP}
        for n in ("node_parent", "node_tok", "node_step"):
            buf[n] = torch.full((B, node_pitch), -1, dtype=torch.int32, device=self.device)
        tr = RsAlsdTrace(S, node_pitch, *[buf[n].data_ptr() for n in ALSD_TRACE_FIELDS])
        y = torch.zeros(B, U + 1, dtype=torch.int32, device=self.device)
        steps = torch.zeros(B, U, dtype=torch.int32, device=self.device)
        n = torch.zeros(B, dtype=torch.int32, device=self.device)
        score = torch.zeros(B, dtype=torch.float64, device=self.device)
        self._check(self.lib.rs_rnnt_alsd_trace(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, int(beam), float(u_max_ratio), int(score_norm),
                                                int(recombine_returns_input), y.data_ptr(), steps.data_ptr(), n.data_ptr(), score.data_ptr(), U,
                                                C.byref(tr), self._stream()), "rs_rnnt_alsd_trace")
        out = {k: v.cpu() for k, v in buf.items()}
        ran = int((out["n_hyp"][:, 0] >= 0).sum())               # steps never run keep the -1 fill
        for k, _, _ in ALSD_TRACE_STEP:
            out[k] = out[k][:ran]
        out.update(y=y.cpu(), steps=steps.cpu(), n=n.cpu(), score=score.cpu())
        return out

    def _align_inputs(self, enc, enc_len, labels, label_len):
        B, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous() and enc_len.dtype == torch.int32
        assert labels.dtype == torch.int32 and labels.dim() == 2 and labels.shape[0] == B and label_len.dtype == torch.int32
        labels = labels.contiguous()
        if labels.shape[1] == 0:                                 # every utterance has no label: one unused column
            labels = torch.zeros(B, 1, dtype=torch.int32, device=self.device)
        return B, T, labels, labels.shape[1]

    def align(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor):
        """Forced alignment of the label sequences labels[b, :label_len[b]] (rs_rnnt_align; semantics: alignment.py) ->
        (frames i32 [B, U], token_lp f32 [B, U], viterbi f32 [B], loglik f32 [B]) device tensors."""
        B, T, labels, U = self._align_inputs(enc, enc_len, labels, label_len)
        frames = torch.empty(B, U, dtype=torch.int32, device=self.device)
        token_lp = torch.empty(B, U, dtype=torch.float32, device=self.device)
        viterbi = torch.empty(B, dtype=torch.float32, device=self.device)
        loglik = torch.empty(B, dtype=torch.float32, device=self.device)
        self._check(self.lib.rs_rnnt_align(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, labels.data_ptr(), label_len.data_ptr(), U,
                                           frames.data_ptr(), token_lp.data_ptr(), viterbi.data_ptr(), loglik.data_ptr(),
                                           self._stream()), "rs_rnnt_align")
        return frames, token_lp, viterbi, loglik

    def align_segment(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor):
        """Segment alignment of labels[b, :label_len[b]] inside each row's frames (rs_rnnt_align_segment; semantics:
        alignment.py) -> (seg i32 [B, 2], frames i32 [B, U], token_lp f32 [B, U], frame_lp f32 [B, T], viterbi f32 [B],
        loglik f32 [B]) device tensors."""
        B, T, labels, U = self._align_inputs(enc, enc_len, labels, label_len)
        seg = torch.empty(B, 2, dtype=torch.int32, device=self.device)
        frames = torch.empty(B, U, dtype=torch.int32, device=self.device)
        token_lp = torch.empty(B, U, dtype=torch.float32, device=self.device)
        frame_lp = torch.empty(B, T, dtype=torch.float32, device=self.device)
        viterbi = torch.empty(B, dtype=torch.float32, device=self.device)
        loglik = torch.empty(B, dtype=torch.float32, device=self.device)
        self._check(self.lib.rs_rnnt_align_segment(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, labels.data_ptr(), label_len.data_ptr(), U,
                                                   seg.data_ptr(), frames.data_ptr(), token_lp.data_ptr(), frame_lp.data_ptr(),
                                                   viterbi.data_ptr(), loglik.data_ptr(), self._stream()), "rs_rnnt_align_segment")
        return seg, frames, token_lp, frame_lp, viterbi, loglik

    def align_lattice(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor, out=None):
        """The lattice alone (rs_rnnt_align_lattice) -> (lp_blank, lp_emit) f32 [B, T, U + 1]; cells outside an utterance keep
        what ``out`` held (NaN for fresh buffers)."""
        B, T, labels, U = self._align_inputs(enc, enc_len, labels, label_len)
        if out is None:
            out = (torch.full((B, T, U + 1), float("nan"), device=self.device), torch.full((B, T, U + 1), float("nan"), device=self.device))
        lp_blank, lp_emit = out
        self._check(self.lib.rs_rnnt_align_lattice(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, labels.data_ptr(), label_len.data_ptr(), U,
                                                   lp_blank.data_ptr(), lp_emit.data_ptr(), self._stream()), "rs_rnnt_align_lattice")
        return lp_blank, lp_emit

    @staticmethod
    def _band_rows(band, B: int, U: int) -> np.ndarray:
        """A host band [B, <= U + 1] as the int32 [B, U + 1] the C call reads (the padding rows are never read)."""
        band = np.asarray(band, dtype=np.int32)
        assert band.ndim == 2 and band.shape[0] == B and band.shape[1] <= U + 1
        out = np.zeros((B, U + 1), dtype=np.int32)
        out[:, : band.shape[1]] = band
        return out

    def align_banded(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor, band_lo, band_hi):
        """Banded alignment of labels[b, :label_len[b]] inside the band band_lo[b][u] <= t < band_hi[b][u] (host int32 arrays
        [B, >= label_len + 1]; rs_rnnt_align_banded; semantics: alignment.py) -> (frames i32 [B, U], token_lp f32 [B, U],
        viterbi f32 [B], loglik f32 [B], edge i32 [B]) device tensors."""
        B, T, labels, U = self._align_inputs(enc, enc_len, labels, label_len)
        lo, hi = self._band_rows(band_lo, B, U), self._band_rows(band_hi, B, U)
        frames = torch.empty(B, U, dtype=torch.int32, device=self.device)
        token_lp = torch.empty(B, U, dtype=torch.float32, device=self.device)
        viterbi = torch.empty(B, dtype=torch.float32, device=self.device)
        loglik = torch.empty(B, dtype=torch.float32, device=self.device)
        edge = torch.empty(B, dtype=torch.int32, device=self.device)
        self._check(self.lib.rs_rnnt_align_banded(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, labels.data_ptr(), label_len.data_ptr(), U,
                                                  lo.ctypes.data, hi.ctypes.data, frames.data_ptr(), token_lp.data_ptr(), viterbi.data_ptr(),
                                                  loglik.data_ptr(), edge.data_ptr(), self._stream()), "rs_rnnt_align_banded")
        return frames, token_lp, viterbi, loglik, edge

    def align_banded_lattice(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor, band_lo,
                             band_hi, cells: int):
        """The banded lattice alone (rs_rnnt_align_banded_lattice) -> (lp_blank, lp_emit) f32 [cells] in banded storage
        (longform.band_offsets gives each row's offset; ``cells`` is their total)."""
        B, T, labels, U = self._align_inputs(enc, enc_len, labels, label_len)
        lo, hi = self._band_rows(band_lo, B, U), self._band_rows(band_hi, B, U)
        lp_blank = torch.full((max(cells, 1),), float("nan"), device=self.device)
        lp_emit = torch.full((max(cells, 1),), float("nan"), device=self.device)
        self._check(self.lib.rs_rnnt_align_banded_lattice(self.h, enc.data_ptr(), enc_len.data_ptr(), B, T, labels.data_ptr(),
                                                          label_len.data_ptr(), U, lo.ctypes.data, hi.ctypes.data, lp_blank.data_ptr(),
                                                          lp_emit.data_ptr(), self._stream()), "rs_rnnt_align_banded_lattice")
        return lp_blank[:cells], lp_emit[:cells]

    def spot(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor, threshold: float = -1.0,
             max_hits: int = 64, scores: bool = False):
        """Keyword spotting (rs_rnnt_spot; semantics: keywords.py): every hit of each keyword labels[k, :label_len[k]] in each
        recording enc[r, :enc_len[r]], pair p = r * n_kw + k -> (span i32 [P, H, 2], score f32 [P, H], confidence f32 [P, H],
        frames i32 [P, H, U], token_lp f32 [P, H, U], count i32 [P]) device tensors, H = max_hits, hits in pick order; with
        ``scores`` also E f32 [P, T] and S i32 [P, T], the best segment ending at every frame."""
        R, T, _ = enc.shape
        assert enc.dtype == torch.float32 and enc.is_contiguous() and enc_len.dtype == torch.int32
        assert labels.dtype == torch.int32 and labels.dim() == 2 and label_len.dtype == torch.int32
        labels = labels.contiguous()
        K, U = labels.shape
        P, H, dev = R * K, int(max_hits), self.device
        span = torch.empty(P, H, 2, dtype=torch.int32, device=dev)
        score = torch.empty(P, H, dtype=torch.float32, device=dev)
        conf = torch.empty(P, H, dtype=torch.float32, device=dev)
        frames = torch.empty(P, H, U, dtype=torch.int32, device=dev)
        token_lp = torch.empty(P, H, U, dtype=torch.float32, device=dev)
        count = torch.empty(P, dtype=torch.int32, device=dev)
        E = torch.empty(P, T, dtype=torch.float32, device=dev) if scores else None
        S = torch.empty(P, T, dtype=torch.int32, device=dev) if scores else None
        self._check(self.lib.rs_rnnt_spot(self.h, enc.data_ptr(), enc_len.data_ptr(), R, T, labels.data_ptr(), label_len.data_ptr(), K, U,
                                          float(threshold), H, span.data_ptr(), score.data_ptr(), conf.data_ptr(), frames.data_ptr(),
                                          token_lp.data_ptr(), count.data_ptr(), E.data_ptr() if scores else None,
                                          S.data_ptr() if scores else None, self._stream()), "rs_rnnt_spot")
        out = (span, score, conf, frames, token_lp, count)
        return out + (E, S) if scores else out

    def spot_lattice(self, enc: torch.Tensor, enc_len: torch.Tensor, labels: torch.Tensor, label_len: torch.Tensor):
        """The pairs' lattice alone (rs_rnnt_spot_lattice) -> (lp_blank, lp_emit) f32 [R * K, T, U + 1], pair p = r * K + k;
        cells outside a pair are NaN."""
        R, T, _ = enc.shape
        K, U = labels.shape
        lp_blank = torch.full((R * K, T, U + 1), float("nan"), device=self.device)
        lp_emit = torch.full((R * K, T, U + 1), float("nan"), device=self.device)
        self._check(self.lib.rs_rnnt_spot_lattice(self.h, enc.data_ptr(), enc_len.data_ptr(), R, T, labels.contiguous().data_ptr(),
                                                  label_len.data_ptr(), K, U, lp_blank.data_ptr(), lp_emit.data_ptr(), self._stream()),
                    "rs_rnnt_spot_lattice")
        return lp_blank, lp_emit

    def resample_mono(self, raw: torch.Tensor, lens: torch.Tensor, samplerate: int, pad: int = 0):
        """norm_audio on the device (pkg/nemo-asr/src/audio.py:54-68) + transcribe()'s padding: ``raw`` [B, C, L] float32 or
        int16 (PCM) on this device at ``samplerate``, ``lens`` int32 [B] valid samples -> (wav float32 [B, L16] at 16 kHz mono
        with ``pad`` zeros on both sides of every utterance, lens int32 [B]); feed both to ``transcribe_device``."""
        assert raw.dim() == 3 and raw.is_contiguous() and raw.dtype in (torch.float32, torch.int16) and lens.dtype == torch.int32
        key = int(samplerate)
        if not hasattr(self, "_rs_taps"):
            self._rs_taps = {}
        if key not in self._rs_taps:
            taps, up, down, pre = resample_taps(key, self.cfg.sample_rate)
            self._rs_taps[key] = (taps.to(self.device), up, down, pre)
        taps, up, down, pre = self._rs_taps[key]
        B, Cn, L = raw.shape
        n_out = (L * up + down - 1) // down
        L16 = (n_out + 2 * pad + 3) & ~3
        out = torch.empty(B, L16, dtype=torch.float32, device=self.device)
        out_len = torch.empty(B, dtype=torch.int32, device=self.device)
        self._check(self.lib.rs_resample_mono(self.h, raw.data_ptr(), int(raw.dtype == torch.int16), lens.data_ptr(), B, Cn, L,
                                              taps.data_ptr(), taps.shape[1], up, down, pre, pad, out.data_ptr(), L16, out_len.data_ptr(),
                                              self._stream()), "rs_resample_mono")
        return out, out_len

    # -- kernel seams
    def gemm(self, a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], epilogue: int,
             resid: Optional[torch.Tensor] = None, alpha: float = 1.0, out: Optional[torch.Tensor] = None,
             out2: Optional[torch.Tensor] = None, split: int = 0) -> torch.Tensor:
        """``out2`` / ``split``: EPI_QKV_VT only -- columns >= split go transposed into out2 (bf16 [N - split, ld2], its row
        pitch ld2 = out2.stride(0)); ``out`` keeps the row pitch N and its columns >= split are not written."""
        M, K = a.shape
        N = w.shape[0]
        assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.is_contiguous() and w.is_contiguous()
        if out is None:
            if epilogue in (EPI_RESID_F32, EPI_BIAS_F32):
                out = torch.empty(M, N, dtype=torch.float32, device=self.device)
            elif epilogue == EPI_BIAS_F16:
                out = torch.empty(M, N, dtype=torch.float16, device=self.device)
            elif epilogue == EPI_BIAS_GLU_BF16:
                out = torch.empty(M, N // 2, dtype=torch.bfloat16, device=self.device)
            else:
                out = torch.empty(M, N, dtype=torch.bfloat16, device=self.device)
        ld2 = 0
        if out2 is not None:
            assert out2.dtype == torch.bfloat16 and out2.dim() == 2 and out2.stride(1) == 1
            ld2 = out2.stride(0)
        self._check(self.lib.rs_gemm_bf16(self.h, a.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                          resid.data_ptr() if resid is not None else None, out.data_ptr(), M, N, K,
                                          epilogue, alpha, out2.data_ptr() if out2 is not None else None, split, ld2,
                                          self._stream()), "rs_gemm_bf16")
        return out

    def layernorm(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, bf16_out: bool = True) -> torch.Tensor:
        rows, d = x.shape
        out = torch.empty(rows, d, dtype=torch.bfloat16 if bf16_out else torch.float32, device=self.device)
        self._check(self.lib.rs_layernorm(self.h, x.data_ptr(), g.data_ptr(), b.data_ptr(),
                                          None if bf16_out else out.data_ptr(), out.data_ptr() if bf16_out else None,
                                          None, None, rows, d, self._stream()), "rs_layernorm")
        return out

    def layernorm_chained(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, g2: torch.Tensor, b2: torch.Tensor,
                          out_f32: torch.Tensor, out_bf16: torch.Tensor) -> None:
        """out_f32 = LN1(x) (``out_f32`` may be ``x``: in place, as the encoder runs it), out_bf16 = LN2(LN1(x))."""
        rows, d = x.shape
        assert x.dtype == out_f32.dtype == torch.float32 and out_bf16.dtype == torch.bfloat16
        self._check(self.lib.rs_layernorm(self.h, x.data_ptr(), g.data_ptr(), b.data_ptr(), out_f32.data_ptr(), out_bf16.data_ptr(),
                                          g2.data_ptr(), b2.data_ptr(), rows, d, self._stream()), "rs_layernorm")

    def attention(self, qkv: torch.Tensor, vt: torch.Tensor, pos: torch.Tensor, bd_bias: torch.Tensor, bias_u: torch.Tensor,
                  enc_len: torch.Tensor, B: int, T_max: int, w_left: int, w_right: int, n_global: int,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The local-attention kernels alone: qkv bf16 [B*T_max, 3*H*128] (q + pos_bias_u | k | unused), vt bf16 [H*128, ld_vt]
        (row pitch vt.stride(0)), pos bf16 [H, n_rel_pad, 128], bd_bias f32 [H, n_rel_pad], bias_u f32 [H, 128] ->
        bf16 [B*T_max, H*128]."""
        H, n_rel_pad, _ = pos.shape
        assert qkv.dtype == vt.dtype == pos.dtype == torch.bfloat16 and vt.stride(1) == 1 and enc_len.dtype == torch.int32
        if out is None:
            out = torch.empty(B * T_max, H * 128, dtype=torch.bfloat16, device=self.device)
        self._check(self.lib.rs_attention(self.h, qkv.data_ptr(), vt.data_ptr(), vt.stride(0), pos.data_ptr(), bd_bias.data_ptr(),
                                          n_rel_pad, bias_u.data_ptr(), out.data_ptr(), enc_len.data_ptr(), B, T_max, H,
                                          w_left, w_right, n_global, self._stream()), "rs_attention")
        return out

    def conv_dw(self, u: torch.Tensor, w: torch.Tensor, shift: torch.Tensor, enc_len: torch.Tensor, T_max: int) -> torch.Tensor:
        """u bf16 [B*T_max, d], w f32 [k, d] (BatchNorm folded), shift f32 [d] -> swish(depthwise conv + shift) bf16."""
        rows, d = u.shape
        assert u.dtype == torch.bfloat16 and u.is_contiguous() and enc_len.dtype == torch.int32
        out = torch.empty_like(u)
        self._check(self.lib.rs_conv_dw(self.h, u.data_ptr(), out.data_ptr(), w.data_ptr(), shift.data_ptr(), enc_len.data_ptr(),
                                        rows // T_max, T_max, d, w.shape[0], self._stream()), "rs_conv_dw")
        return out

    def sub_conv0_dw1(self, mel: torch.Tensor, mel_len: torch.Tensor, mel_stats: Optional[torch.Tensor], w0: torch.Tensor,
                      b0: torch.Tensor, wd: torch.Tensor, bd: torch.Tensor) -> torch.Tensor:
        """mel f32 [B, F_max, n_mels] (+ (mean, 1 / (std + eps)) [B, n_mels, 2]) -> conv.0 + ReLU + conv.2, bf16 [B, T2, F2, C]."""
        B, F_max, n_mels = mel.shape
        C = w0.shape[0]
        T2, F2 = conv_out_len(conv_out_len(F_max)), conv_out_len(conv_out_len(n_mels))
        assert mel.dtype == torch.float32 and mel.is_contiguous() and mel_len.dtype == torch.int32
        out = torch.empty(B, T2, F2, C, dtype=torch.bfloat16, device=self.device)
        self._check(self.lib.rs_sub_conv0_dw1(self.h, mel.data_ptr(), mel_len.data_ptr(), mel_stats.data_ptr() if mel_stats is not None else None,
                                              B, F_max, n_mels, C, w0.data_ptr(), b0.data_ptr(), wd.data_ptr(), bd.data_ptr(),
                                              out.data_ptr(), self._stream()), "rs_sub_conv0_dw1")
        return out

    def sub_dw(self, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, mel_len: torch.Tensor, len_shift: int) -> torch.Tensor:
        """Depthwise 3x3 s2 on channels-last bf16 [B, Tin, Fin, C] -> [B, conv_len(Tin), conv_len(Fin), C]."""
        B, Tin, Fin, C = x.shape
        Tout, Fout = conv_out_len(Tin), conv_out_len(Fin)
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and mel_len.dtype == torch.int32
        out = torch.empty(B, Tout, Fout, C, dtype=torch.bfloat16, device=self.device)
        self._check(self.lib.rs_sub_dw(self.h, x.data_ptr(), out.data_ptr(), w.data_ptr(), b.data_ptr(), mel_len.data_ptr(), len_shift,
                                       B, Tin, Fin, Tout, Fout, C, self._stream()), "rs_sub_dw")
        return out

    def enable_stage_timing(self, on: bool = True):
        self._check(self.lib.rs_enable_stage_timing(self.h, int(on)), "rs_enable_stage_timing")

    def kernel_timing(self, enable: Optional[bool] = None):
        """enable=True/False switches per-launch event timing; with None returns {name: (launches, total_ms)} and resets."""
        if enable is not None:
            self._check(self.lib.rs_enable_kernel_timing(self.h, int(enable)), "rs_enable_kernel_timing")
            return None
        buf = C.create_string_buffer(1 << 16)
        self._check(self.lib.rs_kernel_timing(self.h, buf, len(buf)), "rs_kernel_timing")
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms = line.split("\t")
            out[name] = (int(n), float(ms))
        return out

    def attention_cycles(self):
        """Cycle stamps of the attention kernel: the kernel records none, so both are zero."""
        return {"start": 0, "end": 0}

    def decode_cycles(self, B: int, L_max: int, U_max: int):
        out = (C.c_int64 * 12)()
        self._check(self.lib.rs_debug_decode_cycles(self.h, B, L_max, U_max, out), "rs_debug_decode_cycles")
        return dict(zip(("phase_j", "barrier_a", "reduce", "phase_l", "barrier_b", "phase_p", "barrier_c", "iterations", "j_loads", "j_rows", "j_misc", "_"), [int(v) for v in out]))

    def enable_gemm_timing(self, on: bool = True):
        self._check(self.lib.rs_enable_gemm_timing(self.h, int(on)), "rs_enable_gemm_timing")

    def gemm_timing(self):
        """(summed device ms, summed algorithmic FLOPs, launches) of the wgmma GEMM since enabled / last read."""
        ms, fl, n = C.c_double(), C.c_double(), C.c_int64()
        self._check(self.lib.rs_gemm_timing(self.h, C.byref(ms), C.byref(fl), C.byref(n)), "rs_gemm_timing")
        return ms.value, fl.value, n.value

    def stage_times_ms(self) -> Dict[str, float]:
        ms = (C.c_float * 8)()
        self._check(self.lib.rs_stage_times_ms(self.h, ms), "rs_stage_times_ms")
        return dict(zip(("logmel", "subsample", "layers", "enc_proj", "decode"), [float(v) for v in ms[:5]]))
