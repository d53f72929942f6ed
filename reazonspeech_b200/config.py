"""Model configuration for the FastConformer-RNNT path.

Mirrors the fields of the ``model_config.yaml`` inside the ``.nemo`` archive that
``reazonspeech.nemo.asr.load_model`` fetches (reference call site:
pkg/nemo-asr/src/transcribe.py:26-28).  Field names follow NeMo's yaml so a real
config can be mapped one-to-one (see ``ModelConfig.from_nemo_yaml``).  Defaults are
the values SURVEY.md App. A.1 expects for ``reazon-research/reazonspeech-nemo-v2``
(all tagged (R) there: NeMo and the checkpoint are not available offline).
"""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass
from typing import Optional


@dataclass(frozen=True)
class ModelConfig:
    # --- preprocessor (AudioToMelSpectrogramPreprocessor) ---
    sample_rate: int = 16000
    n_window_size: int = 400          # window_size 0.025 s
    n_window_stride: int = 160        # window_stride 0.01 s
    n_fft: int = 512
    n_mels: int = 80
    preemph: float = 0.97
    log_zero_guard: float = 2.0 ** -24
    norm_eps: float = 1e-5            # CONSTANT added to per-feature std
    # --- encoder (ConformerEncoder, dw_striding x8) ---
    n_layers: int = 24
    d_model: int = 1024
    n_heads: int = 8
    ff_expansion: int = 4
    conv_kernel: int = 9
    sub_channels: int = 256
    sub_factor: int = 8
    att_left: int = 128               # att_context_size[0]
    att_right: int = 128              # att_context_size[1]
    global_tokens: int = 1
    xscaling: bool = True
    ln_eps: float = 1e-5
    bn_eps: float = 1e-5
    # --- decoder / joint ---
    vocab_size: int = 3000            # blank index == vocab_size
    pred_hidden: int = 640
    joint_hidden: int = 640
    max_symbols: int = 10
    checkpoint_maes: Optional["MaesConfig"] = dataclasses.field(default=None, compare=False)   # decoding.beam.maes_* of model_config.yaml
    checkpoint_decoding: str = dataclasses.field(default="greedy", compare=False)   # the strategy model_config.yaml asks for (informational: load_model decides what runs)

    # ---- derived ----
    @property
    def d_head(self) -> int:
        return self.d_model // self.n_heads

    @property
    def d_ff(self) -> int:
        return self.d_model * self.ff_expansion

    @property
    def n_freq(self) -> int:
        return self.n_fft // 2 + 1

    @property
    def blank(self) -> int:
        return self.vocab_size

    @property
    def n_classes(self) -> int:
        return self.vocab_size + 1

    @property
    def sub_freq(self) -> int:
        """Frequency bins left after the three stride-2 convs (80 -> 40 -> 20 -> 10)."""
        f = self.n_mels
        for _ in range(3):
            f = conv_out_len(f)
        return f

    @property
    def sub_out_dim(self) -> int:
        return self.sub_channels * self.sub_freq

    @property
    def n_rel(self) -> int:
        """Number of relative positions held by the local-attention table (2w+1)."""
        return self.att_left + self.att_right + 1

    def mel_frames(self, n_samples: int) -> int:
        """Frames the centred STFT produces (the feature TENSOR's time size): L // hop + 1."""
        return n_samples // self.n_window_stride + 1

    def mel_valid(self, n_samples: int) -> int:
        """FilterbankFeatures.get_seq_len (NeMo 2.x): floor((L + 2*(n_fft//2) - n_fft) / hop) = L // hop.

        One less than the STFT's frame count: the final frame is masked to zero and excluded from
        the normalisation statistics.  Pinned by transformers' Parakeet port of NeMo
        (feature_extraction_parakeet.py ``features_lengths``; tests/golden/make_parakeet_golden.py)."""
        return (n_samples + 2 * (self.n_fft // 2) - self.n_fft) // self.n_window_stride

    def enc_frames(self, n_samples: int) -> int:
        """Valid encoder frames: ConvSubsampling.calc_length applied three times to ``mel_valid``."""
        t = self.mel_valid(n_samples)
        for _ in range(3):
            t = conv_out_len(t)
        return t

    def replace(self, **kw) -> "ModelConfig":
        return dataclasses.replace(self, **kw)

    @staticmethod
    def tiny() -> "ModelConfig":
        """Small shape-compatible config for CPU-side tests (same code paths, tiny dims).

        d_model/d_ff/heads keep the alignment constraints of the kernels
        (d_head == 128, every GEMM K and N a multiple of 128 / 64)."""
        return ModelConfig(n_layers=2, d_model=256, n_heads=2, sub_channels=64,
                           att_left=16, att_right=16, vocab_size=127,
                           pred_hidden=128, joint_hidden=128)

    @staticmethod
    def decoding_strategy(cfg: dict) -> str:
        """The checkpoint's configured decoding strategy ("greedy", "greedy_batch", "beam", "alsd", ...); the reference never
        overrides it (pkg/nemo-asr/src/transcribe.py:26-28), reazonspeech-nemo-v2 ships ALSD (decode.py:29)."""
        dec = cfg.get("decoding", {}) or {}
        strategy = str(dec.get("strategy", "greedy_batch"))
        if strategy == "beam" or "beam" in strategy:
            return str((dec.get("beam", {}) or {}).get("search_type", strategy))
        return strategy

    @staticmethod
    def from_nemo_yaml(cfg: dict) -> "ModelConfig":
        """Map a parsed ``model_config.yaml`` (dict) onto ModelConfig.

        Every setting that changes the arithmetic and that the kernels do not implement raises ValueError: a
        checkpoint trained with another frontend normalisation, attention type, norm layer or prediction network must
        not load and quietly transcribe garbage.  Training-only keys (dither, pad_to, dropout, spec-augment, optimiser)
        are ignored, as ``model.transcribe`` ignores or zeroes them (SURVEY.md App. A.1)."""
        pre, enc = cfg["preprocessor"], cfg["encoder"]
        dec, joint = cfg["decoder"], cfg["joint"]
        sr = int(pre.get("sample_rate", 16000))

        def require(block: str, d: dict, key: str, allowed, default):
            v = d.get(key, default)
            ok = any((v is None and a is None) or (v is not None and a is not None and (
                (isinstance(a, float) and abs(float(v) - a) <= 1e-9 * max(1.0, abs(a))) or (not isinstance(a, float) and v == a))) for a in allowed)
            if not ok:
                raise ValueError(f"model_config.yaml: {block}.{key}={v!r} is not implemented by the engine (supported: {list(allowed)})")
            return v

        require("preprocessor", pre, "window", ("hann",), "hann")
        require("preprocessor", pre, "normalize", ("per_feature",), "per_feature")
        require("preprocessor", pre, "log", (True,), True)
        require("preprocessor", pre, "log_zero_guard_type", ("add",), "add")
        require("preprocessor", pre, "mag_power", (2.0,), 2.0)
        require("preprocessor", pre, "lowfreq", (0, 0.0), 0)
        require("preprocessor", pre, "highfreq", (None, sr / 2.0, sr // 2), None)
        require("preprocessor", pre, "mel_norm", ("slaney",), "slaney")
        require("preprocessor", pre, "frame_splicing", (1,), 1)
        require("preprocessor", pre, "exact_pad", (False,), False)          # exact_pad changes the STFT padding and the frame count
        guard = pre.get("log_zero_guard_value", 2.0 ** -24)
        if isinstance(guard, str):                                   # NeMo also accepts "tiny" / "eps" of float32
            import numpy as np
            guard = {"tiny": float(np.finfo(np.float32).tiny), "eps": float(np.finfo(np.float32).eps)}.get(guard)
            if guard is None:
                raise ValueError(f"model_config.yaml: preprocessor.log_zero_guard_value={pre['log_zero_guard_value']!r} not understood")
        ctx = enc.get("att_context_size", [128, 128]) or [128, 128]
        if ctx and isinstance(ctx[0], (list, tuple)):               # multi-lookahead configs list several contexts: the first is the default
            ctx = ctx[0]
        require("encoder", enc, "self_attention_model", ("rel_pos_local_attn",), "rel_pos_local_attn")
        require("encoder", enc, "subsampling", ("dw_striding",), "dw_striding")
        require("encoder", enc, "subsampling_factor", (8,), 8)
        require("encoder", enc, "conv_norm_type", ("batch_norm",), "batch_norm")
        require("encoder", enc, "untie_biases", (True,), True)
        require("encoder", enc, "global_tokens_spacing", (1,), 1)
        require("encoder", enc, "global_attn_separate", (False,), False)
        require("encoder", enc, "conv_context_size", (None,), None)
        require("encoder", enc, "causal_downsampling", (False,), False)
        require("encoder", enc, "att_context_style", ("regular",), "regular")  # "chunked_limited" masks by chunk, not by band
        require("encoder", enc, "reduction", (None,), None)
        if not jointnet_probe(cfg).get("dropout"):                            # without dropout NeMo builds joint_net as [act, Linear]: the
            raise ValueError("model_config.yaml: joint.jointnet.dropout is absent or 0: NeMo then builds the output layer as joint_net.1, "
                             "the engine binds joint.joint_net.2 (the layout with dropout, as reazonspeech-nemo-v2 ships)")
        n_mels = int(pre.get("features", 80))
        if int(enc.get("feat_in", n_mels)) != n_mels:
            raise ValueError(f"model_config.yaml: encoder.feat_in={enc.get('feat_in')} != preprocessor.features={n_mels}")
        if int(ctx[0]) < 0 or int(ctx[1]) < 0:
            raise ValueError(f"model_config.yaml: encoder.att_context_size={ctx} (unlimited context) is not implemented")
        prednet, jointnet = dec["prednet"], joint["jointnet"]
        require("decoder.prednet", prednet, "pred_rnn_layers", (1,), 1)
        require("decoder", dec, "blank_as_pad", (True,), True)
        require("joint.jointnet", jointnet, "activation", ("relu",), "relu")
        vocab = int(dec.get("vocab_size", joint.get("num_classes", 3000)))
        if "num_classes" in joint and int(joint["num_classes"]) != vocab:
            raise ValueError(f"model_config.yaml: joint.num_classes={joint['num_classes']} != decoder.vocab_size={vocab}")
        pred_hidden, d_model = int(prednet["pred_hidden"]), int(enc["d_model"])
        if int(jointnet.get("pred_hidden", pred_hidden)) != pred_hidden or int(jointnet.get("encoder_hidden", d_model)) != d_model:
            raise ValueError("model_config.yaml: joint.jointnet.{pred_hidden, encoder_hidden} disagree with decoder / encoder")
        return ModelConfig(
            sample_rate=sr,
            n_window_size=int(round(float(pre.get("window_size", 0.025)) * sr)),
            n_window_stride=int(round(float(pre.get("window_stride", 0.01)) * sr)),
            n_fft=int(pre.get("n_fft") or 512),
            n_mels=n_mels,
            preemph=float(pre.get("preemph", 0.97) or 0.0),
            log_zero_guard=float(guard),
            n_layers=int(enc["n_layers"]),
            d_model=d_model,
            n_heads=int(enc.get("n_heads", 8)),
            ff_expansion=int(enc.get("ff_expansion_factor", 4)),
            conv_kernel=int(enc.get("conv_kernel_size", 9)),
            sub_channels=int(enc.get("subsampling_conv_channels", 256)),
            sub_factor=int(enc.get("subsampling_factor", 8)),
            att_left=int(ctx[0]), att_right=int(ctx[1]),
            global_tokens=int(enc.get("global_tokens", 1)),
            xscaling=bool(enc.get("xscaling", True)),
            vocab_size=vocab,
            pred_hidden=pred_hidden,
            joint_hidden=int(jointnet["joint_hidden"]),
            max_symbols=int(cfg.get("decoding", {}).get("greedy", {}).get("max_symbols", 10) or 10),
            checkpoint_decoding=ModelConfig.decoding_strategy(cfg),
            checkpoint_maes=MaesConfig.from_beam_block((cfg.get("decoding", {}) or {}).get("beam", {}) or {}),
        )


@dataclass(frozen=True)
class MaesConfig:
    """Parameters of the MAES beam search (NeMo's maes_* keys of decoding.beam, with NeMo's defaults): ``num_steps``
    expansion rounds per frame (>= 2), ``prefix_alpha`` the longest prefix-search gap (>= 0), ``expansion_beta`` extra candidates
    per hypothesis beyond the beam (>= 0), ``expansion_gamma`` the score window of the candidates kept (> 0).  The engine runs
    num_steps <= 4 and prefix_alpha, expansion_beta <= 4, and at most 1024 expansion rows per utterance
    (beam * (beam + expansion_beta)^num_steps)."""
    num_steps: int = 2
    prefix_alpha: int = 1
    expansion_beta: int = 2
    expansion_gamma: float = 2.3

    def validate(self) -> "MaesConfig":
        if int(self.num_steps) != self.num_steps or not 2 <= int(self.num_steps) <= 4:
            raise ValueError(f"maes num_steps must be an integer in 2..4, got {self.num_steps!r}")
        for name in ("prefix_alpha", "expansion_beta"):
            v = getattr(self, name)
            if int(v) != v or not 0 <= int(v) <= 4:
                raise ValueError(f"maes {name} must be an integer in 0..4, got {v!r}")
        g = float(self.expansion_gamma)
        if not (math.isfinite(g) and g > 0.0):
            raise ValueError(f"maes expansion_gamma must be finite and > 0, got {self.expansion_gamma!r}")
        return self

    def check_beam(self, beam: int, vocab_size: int) -> "MaesConfig":
        """The limits that depend on the beam: 1..8, beam + expansion_beta <= vocab_size, at most 1024 expansion rows."""
        self.validate()
        if int(beam) != beam or not 1 <= int(beam) <= 8:
            raise ValueError(f"beam_size must be an integer in 1..8 for MAES, got {beam!r}")
        k = min(int(beam), int(vocab_size))
        if k + self.expansion_beta > vocab_size:
            raise ValueError(f"beam_size + expansion_beta = {k + self.expansion_beta} exceeds the vocabulary ({vocab_size})")
        w = k * (k + self.expansion_beta) ** self.num_steps
        if w > 1024:
            raise ValueError(f"beam_size * (beam_size + expansion_beta)^num_steps = {w} expansion rows exceed the engine's 1024")
        return self

    @staticmethod
    def from_beam_block(beam: dict) -> Optional["MaesConfig"]:
        """NeMo's decoding.beam block -> the MaesConfig its maes_* keys give (None: it has none)."""
        keys = {"maes_num_steps": "num_steps", "maes_prefix_alpha": "prefix_alpha", "maes_expansion_beta": "expansion_beta",
                "maes_expansion_gamma": "expansion_gamma"}
        kw = {f: beam[k] for k, f in keys.items() if beam.get(k) is not None}
        if not kw:
            return None
        kw = {f: float(v) if f == "expansion_gamma" else int(v) for f, v in kw.items()}
        return MaesConfig(**kw)


def jointnet_probe(cfg: dict) -> dict:
    return (cfg.get("joint", {}) or {}).get("jointnet", {}) or {}


def conv_out_len(n: int) -> int:
    """ConvSubsampling.calc_length for k=3, s=2, p=1: floor((n + 2 - 3) / 2) + 1."""
    return (n - 1) // 2 + 1


def xscale(cfg: ModelConfig) -> float:
    return math.sqrt(cfg.d_model) if cfg.xscaling else 1.0
