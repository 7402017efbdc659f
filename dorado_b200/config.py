"""Model description for the B200 basecalling engine.

Mirrors the fields of the reference's ``BasecallModelConfig`` that the hot path reads
(dorado/config/include/config/BasecallModelConfig.h, parsing rules from
dorado/config/BasecallModelConfig.cpp:214-323 for Conv->LSTM->CRF models and :422-470 for
Conv->Transformer->CRF models, conv parsing from dorado/config/common.cpp:53-93).

Inside dorado the C++ adapter (include/B200ModelRunner.h) fills ``b200_model_desc`` straight from
``BasecallModelConfig``; this module does the same from a ``config.toml`` for the tests and bench.
"""
from __future__ import annotations

import dataclasses
import pathlib
import tomllib
from typing import List, Optional, Tuple

ACT_SWISH, ACT_SWISH_CLAMP, ACT_TANH = 0, 1, 2
_ACT = {"swish": ACT_SWISH, "tanh": ACT_TANH}


@dataclasses.dataclass
class ConvParams:
    insize: int
    size: int
    winlen: int
    stride: int
    activation: int


@dataclasses.dataclass
class TxParams:
    d_model: int
    nhead: int
    dim_feedforward: int
    depth: int
    deepnorm_alpha: float
    attn_window: Tuple[int, int]
    theta: float = 10000.0
    max_seq_len: int = 2048
    upsample_scale: int = 2
    crf_scale: float = 5.0


@dataclasses.dataclass
class BasecallModelConfig:
    name: str
    path: pathlib.Path
    convs: List[ConvParams]
    stride: int
    state_len: int
    outsize: int
    num_features: int = 1
    lstm_size: int = -1
    lstm_layers: int = 0
    lstm_inner_dim: "int | None" = None   # FLSTM models: rank of the factorised gate matrices (is_flstm_model)
    clamp: bool = False
    bias: bool = False
    out_features: Optional[int] = None
    scale: float = 1.0
    blank_score: float = 2.0
    qscale: float = 1.0
    qbias: float = 0.0
    tx: Optional[TxParams] = None

    @property
    def is_tx_model(self) -> bool:
        return self.tx is not None

    @property
    def is_flstm_model(self) -> bool:
        """BasecallModelConfig::is_flstm_model (BasecallModelConfig.h:145)."""
        return self.tx is None and self.lstm_inner_dim is not None

    @property
    def num_states(self) -> int:
        return self.outsize // 4

    def stride_inner(self) -> int:
        """Stride of the conv stack alone (BasecallModelConfig.h: stride_inner)."""
        return self.stride * (self.tx.upsample_scale if self.tx else 1)

    def chunk_size_granularity(self) -> int:
        """BasecallModelConfig.h:159 -- LSTM: stride; tx: stride_inner * 16."""
        return self.stride_inner() * 16 if self.tx else self.stride

    def normalise_chunk_size(self, chunk_size: int) -> int:
        """BatchParams::normalise (dorado/config/BatchParams.cpp:89-105): round down."""
        g = self.chunk_size_granularity()
        return (chunk_size // g) * g

    def out_len(self, chunk_size: int) -> int:
        return chunk_size // self.stride


def _parse_conv(seg: dict, clamp_next: bool) -> ConvParams:
    act = seg["activation"]
    if act not in _ACT:
        raise ValueError(f"Unknown activation: `{act}` in model config, expected `swish` or `tanh`")
    a = _ACT[act]
    if a == ACT_SWISH and clamp_next:
        a = ACT_SWISH_CLAMP
    return ConvParams(seg["insize"], seg["size"], seg["winlen"], seg["stride"], a)


def load_model_config(path) -> BasecallModelConfig:
    path = pathlib.Path(path)
    with open(path / "config.toml", "rb") as f:
        toml = tomllib.load(f)
    q = toml.get("qscore", {})
    qscale, qbias = float(q.get("scale", 1.0)), float(q.get("bias", 0.0))
    model = toml.get("model", {})
    if "encoder" in model and "transformer_encoder" in model["encoder"]:
        enc = model["encoder"]
        layer = enc["transformer_encoder"]["layer"]
        crf = enc["crf"]
        ups = enc["upsample"]
        convs = [_parse_conv(s, False) for s in enc["conv"]["sublayers"] if s["type"] == "convolution"]
        stride = 1
        for c in convs:
            stride *= c.stride
        stride //= ups["scale_factor"]
        theta = float(layer.get("theta", layer.get("rotary_base", 10000.0)))
        tx = TxParams(
            d_model=layer["d_model"], nhead=layer["nhead"], dim_feedforward=layer["dim_feedforward"],
            depth=enc["transformer_encoder"]["depth"], deepnorm_alpha=float(layer["deepnorm_alpha"]),
            attn_window=(int(layer["attn_window"][0]), int(layer["attn_window"][1])), theta=theta,
            max_seq_len=int(layer.get("max_seq_len", 2048)), upsample_scale=ups["scale_factor"],
            crf_scale=float(crf["scale"]))
        state_len = crf["state_len"]
        return BasecallModelConfig(
            name=path.name, path=path, convs=convs, stride=stride, state_len=state_len,
            outsize=4 ** (state_len + 1), num_features=convs[0].insize, clamp=False,
            blank_score=float(crf["blank_score"]), qscale=qscale, qbias=qbias, tx=tx)

    enc = toml["encoder"]
    if "type" not in enc:
        # pre-v4 layout (BasecallModelConfig.cpp:280-295): a fixed swish conv stack described by [encoder] alone; the
        # defaults of BasecallModelConfig.h apply (5 LSTM layers, a biased CRF linear)
        stride, C = int(enc["stride"]), int(enc["features"])
        first = int(enc.get("first_conv_size", 4))
        features = int(toml["input"]["features"])
        state_len = toml["global_norm"]["state_len"]
        convs = [ConvParams(features, first, 5, 1, ACT_SWISH), ConvParams(first, 16, 5, 1, ACT_SWISH),
                 ConvParams(16, C, 19, stride, ACT_SWISH)]
        return BasecallModelConfig(
            name=path.name, path=path, convs=convs, stride=stride, state_len=state_len,
            outsize=4 ** (state_len + 1), num_features=features, lstm_size=C, lstm_layers=5, bias=True,
            scale=float(enc["scale"]), blank_score=float(enc["blank_score"]), qscale=qscale, qbias=qbias)
    subs = enc["sublayers"]
    convs = []
    for i, s in enumerate(subs):
        if s["type"] == "convolution":
            clamp_next = i + 1 < len(subs) and subs[i + 1]["type"] == "clamp"
            convs.append(_parse_conv(s, clamp_next))
    if len(convs) != 3:
        raise ValueError(f"Expected 3 convolution layers but found: {len(convs)}")
    stride = 1
    for c in convs:
        stride *= c.stride
    cfg = BasecallModelConfig(
        name=path.name, path=path, convs=convs, stride=stride,
        state_len=toml["global_norm"]["state_len"], outsize=0,
        num_features=toml["input"]["features"], lstm_size=convs[-1].size,
        clamp=any(s["type"] == "clamp" for s in subs), qscale=qscale, qbias=qbias)
    flstm_layers = 0
    for s in subs:
        if s["type"] == "linear":
            cfg.out_features = s["out_features"]
            cfg.bias = bool(s.get("bias", cfg.lstm_size > 128))
        elif s["type"] == "linearcrfencoder":
            cfg.blank_score = float(s["blank_score"])
            cfg.scale = float(s.get("scale", 1.0))
        elif s["type"] == "lstm":
            cfg.lstm_layers += 1
        elif s["type"] == "flstm":
            # factorised LSTM (BasecallModelConfig.cpp:257-279): all layers share one inner dimension, no mixing with LSTM
            inner = int(s["inner_dim"])
            if cfg.lstm_inner_dim is not None and cfg.lstm_inner_dim != inner:
                raise ValueError(f"Mismatch in inner dimension of FLSTM, found  {cfg.lstm_inner_dim} and {inner}")
            cfg.lstm_inner_dim = inner
            flstm_layers += 1
    if flstm_layers > 0:
        if cfg.lstm_layers > 0:
            raise ValueError(f"Cannot mix LSTM and FLSTM layers, found {cfg.lstm_layers} and {flstm_layers}")
        cfg.lstm_layers = flstm_layers
    cfg.outsize = 4 ** (cfg.state_len + 1)
    return cfg


# ---- modified-base models ----------------------------------------------------------------------------------------------
# ModBaseModelConfig (dorado/config/include/config/ModBaseModelConfig.h, parsing in dorado/config/ModBaseModelConfig.cpp).
# Only conv_lstm_v3 runs on the engine: the older types run through plain libtorch even on the reference's CUDA path
# (dorado/modbase/nn/ModBaseModel.cpp:622-645).
MODBASE_TYPES = {"conv_lstm": "conv_lstm", "conv_lstm_v2": "conv_lstm_v2", "conv_lstm_v3": "conv_lstm_v3",
                 "conv_only": "conv_v1", "conv_v1": "conv_v1"}


@dataclasses.dataclass
class ModBaseModules:
    signal_convs: List[ConvParams]
    sequence_convs: List[ConvParams]
    merge_conv: ConvParams
    lstms: List[Tuple[int, bool]]          # (size, reverse) per layer
    linear: Tuple[int, int]                # (in_features, out_features)
    upsample: Optional[Tuple[int, int]]    # (size, scale_factor)

    def signal_stride(self) -> int:
        s = 1
        for c in self.signal_convs:
            s *= c.stride
        return s

    def sequence_stride(self) -> int:
        s = 1
        for c in self.sequence_convs:
            s *= c.stride
        return s

    def stride_ratio(self) -> int:
        sig, seq = self.signal_stride(), self.sequence_stride()
        if sig < seq:
            raise ValueError("modbase sequence stride must be less than or equal to signal stride")
        if sig % seq != 0:
            raise ValueError("modbase signal stride must be evenly divisible by sequence stride")
        return sig // seq


@dataclasses.dataclass
class ModBaseModelConfig:
    name: str
    path: pathlib.Path
    model_type: str
    size: int
    kmer_len: int
    num_out: int
    stride: int
    sequence_stride: int
    modules: ModBaseModules
    mod_codes: List[str]
    mod_long_names: List[str]
    motif: str
    motif_offset: int
    samples_before: int
    samples_after: int
    chunk_size: int
    bases_before: int
    bases_after: int
    reverse_signal: bool
    base_start_justify: bool
    refine_do_rough_rescale: bool
    refine_center_idx: int

    @property
    def lstm_size(self) -> int:
        return self.modules.lstms[0][0]

    @property
    def upsample_scale(self) -> int:
        return self.modules.upsample[1] if self.modules.upsample else 0

    def chunked_sequence_input_TC(self) -> Tuple[int, int]:
        """ModBaseModelConfig::chunked_sequence_input_TC (ModBaseModelConfig.cpp:514-519)."""
        return self.chunk_size // self.modules.stride_ratio(), self.kmer_len * 4

    def chunked_signal_input_TC(self) -> Tuple[int, int]:
        return self.chunk_size, 1

    def chunked_output_TC(self) -> Tuple[int, int]:
        """The reference's nominal output shape; the forward itself returns out_steps() steps (ModsConv pads winlen // 2)."""
        return self.chunk_size // self.stride, self.num_out

    def encoder_steps(self) -> int:
        t = self.chunk_size
        for c in self.modules.signal_convs:
            t = conv_out_len(t, c)
        return t

    def lstm_steps(self) -> int:
        return conv_out_len(self.encoder_steps(), self.modules.merge_conv)

    def out_steps(self) -> int:
        """Steps per chunk of ModBaseConvLSTMV3Model::forward's output."""
        return self.lstm_steps() * max(1, self.upsample_scale)


def conv_out_len(length: int, c: ConvParams) -> int:
    """torch Conv1d length with ModsConv's padding of winlen // 2 (ModBaseModel.cpp:91-97)."""
    return (length + 2 * (c.winlen // 2) - c.winlen) // c.stride + 1


def _int_in_range(seg: dict, key: str, lo: int, hi: int, default=None) -> int:
    """get_int_in_range (ModBaseModelConfig.cpp:30-47)."""
    if key not in seg and default is None:
        raise ValueError(f"modbase model config is missing '{key}'")
    v = int(seg.get(key, default))
    if v < lo or v > hi:
        raise ValueError(f"Invalid modbase model value for '{key}' found: '{v}' which is not in range [{lo} <= x <= {hi}]")
    return v


def _parse_convs(subs: list) -> List[ConvParams]:
    """config::parse_convs (dorado/config/common.cpp:80-94)."""
    out = []
    for i, s in enumerate(subs):
        if s["type"] == "convolution":
            out.append(_parse_conv(s, i + 1 < len(subs) and subs[i + 1]["type"] == "clamp"))
    return out


def load_modbase_config(path) -> ModBaseModelConfig:
    """load_modbase_model_config (ModBaseModelConfig.cpp:527-533) for conv_lstm_v3 models, with the reference's checks."""
    path = pathlib.Path(path)
    with open(path / "config.toml", "rb") as f:
        toml = tomllib.load(f)
    model = toml.get("general", {}).get("model")
    kind = MODBASE_TYPES.get(model)
    if kind is None:
        raise ValueError(f"Unknown modbase model type in config file: {model!r}")
    if kind != "conv_lstm_v3":
        raise ValueError(f"modbase model type {kind!r} is not supported: only conv_lstm_v3 runs on this engine "
                         "(the older types run through plain libtorch in the reference)")
    # parse_modules_params (:155-180)
    layers = toml["encoder"]["sublayers"]
    if not layers:
        raise ValueError("Modbase model config missing enoder sublayers")
    if layers[0]["type"] != "convolution":
        raise ValueError("Modbase model config missing enconder merge convolution")
    merge = _parse_conv(layers[0], False)
    lstms = [(int(s["size"]), bool(int(s["reverse"]))) for s in layers if s["type"] == "lstm"]
    if not lstms:
        raise ValueError("Modbase model config has no lstm layers")
    if lstms[0][1]:
        raise ValueError("Modbase model config first lstm layer must be forward")
    for a, b in zip(lstms, lstms[1:]):
        if a[0] != b[0]:
            raise ValueError("Modbase model config lstm layers unequal sizes")
        if a[1] == b[1]:
            raise ValueError("Modbase model config lstm layers must alternate direction")
    linear = upsample = None
    for s in layers:
        if s["type"] == "linear":
            linear = (int(s["in_features"]), int(s["out_features"]))
        if s["type"] == "upsample":
            upsample = (int(s["size"]), int(s["scale_factor"]))
    if linear is None:
        raise ValueError("Modbase model config has no linear layer")
    if lstms[-1][0] != linear[0]:
        raise ValueError("Modbase model config lstm and linear size mismatch")
    modules = ModBaseModules(_parse_convs(toml["signal_encoder"]["sublayers"]),
                             _parse_convs(toml["sequence_encoder"]["sublayers"]), merge, lstms, linear, upsample)
    # parse_general_params (:255-277) and ModelGeneralParams' checks (:220-245)
    mp = toml["model_params"]
    size = _int_in_range(mp, "size", 1, 4096)
    kmer_len = _int_in_range(mp, "kmer_len", 1, 19)
    num_out = _int_in_range(mp, "num_out", 1, 10)
    stride = _int_in_range(mp, "stride", 1, 6, 3)
    sequence_stride = _int_in_range(mp, "sequence_stride", 1, 6, stride)
    if kmer_len % 2 != 1:
        raise ValueError("Invalid modbase model parameter in general params: 'kmer_length is not odd'.")
    if size != lstms[0][0] or lstms[0][0] != lstms[-1][0]:
        raise ValueError("Modbase model config lstm size mismatch")
    if stride != modules.signal_stride():
        raise ValueError("Modbase model config signal convolution stride mismatch")
    if sequence_stride != modules.sequence_stride():
        raise ValueError("Modbase model config sequence convolution stride mismatch")
    if num_out != linear[1]:
        raise ValueError("Modbase model config linear and num_out mismatch")
    # parse_modification_params (:305-335)
    mb = toml["modbases"]
    codes = list(mb["mod_bases"]) if isinstance(mb["mod_bases"], str) else [str(c) for c in mb["mod_bases"]]
    if not codes:
        raise ValueError("Invalid modbase model parameter in mods params: 'empty modifications.")
    long_names = [str(mb[f"mod_long_names_{i}"]) for i in range(len(codes))]
    motif = str(mb["motif"])
    motif_offset = _int_in_range(mb, "motif_offset", 0, len(motif))
    if motif[motif_offset:motif_offset + 1] not in ("A", "C", "G", "T"):
        raise ValueError(f"Invalid modbase model parameter in mods params: 'invalid motif base {motif[motif_offset:motif_offset + 1]}'.")
    # parse_context_params (:376-397) and ContextParams' checks (:337-360)
    before = _int_in_range(mb, "chunk_context_0", 0, 4096)
    after = _int_in_range(mb, "chunk_context_1", 1, 4096)
    chunk_size = _int_in_range(mb, "chunk_size", before + after, 102400, before + after)
    bases_before = _int_in_range(mb, "kmer_context_bases_0", 0, 9)
    bases_after = _int_in_range(mb, "kmer_context_bases_1", 0, 9)
    if bases_before < 1 or bases_after < 1:
        raise ValueError("Invalid modbase model parameter in context params: 'negative or zero context bases'.")
    if bases_before + bases_after + 1 != kmer_len:
        raise ValueError(f"Invalid modbase model parameter in config: 'inconsistent kmer_len: {kmer_len} != "
                         f"{bases_before + bases_after + 1}'.")
    # parse_refinement_params (:410-425)
    ref = toml.get("refinement", {})
    rough = bool(ref) and int(ref.get("refine_do_rough_rescale", 0)) == 1
    center = _int_in_range(ref, "refine_kmer_center_idx", 0, 19) if rough else 0
    return ModBaseModelConfig(
        name=path.name, path=path, model_type=kind, size=size, kmer_len=kmer_len, num_out=num_out, stride=stride,
        sequence_stride=sequence_stride, modules=modules, mod_codes=codes, mod_long_names=long_names, motif=motif,
        motif_offset=motif_offset, samples_before=before, samples_after=after, chunk_size=chunk_size,
        bases_before=bases_before, bases_after=bases_after, reverse_signal=bool(mb.get("reverse_signal", False)),
        base_start_justify=bool(mb.get("base_start_justify", False)), refine_do_rough_rescale=rough,
        refine_center_idx=center)
