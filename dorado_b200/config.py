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
