"""Weights for the B200 basecalling engine: names, order, synthetic generation and the B2W1 container.

Tensor names and their order are the reference's ``*.tensor`` file list
(dorado/basecall/crf_utils.cpp:26-95 for LSTM models, :97-150 for transformer models), which is also
the order of ``module.parameters()`` that ``utils::load_state_dict`` relies on
(dorado/torch_utils/include/torch_utils/module_utils.h:16-36).  Shapes are torch's:
conv ``[C_out, C_in, W]``, LSTM ``weight_ih/hh [4C, C]`` (gate order i,f,g,o), linear ``[out, in]``.

No model weights ship with the reference tree (they come from ONT's CDN), so parity and the bench
use seeded synthetic weights of the right shapes; ``bias_hh`` is zero because the reference's CUDA
path only ever reads ``bias_ih`` (dorado/nn/LSTMStack.cpp:108,163,224).

B2W1 container (little endian): ``"B2W1"  u32 n  { u32 name_len, name, u32 ndim, u32 dims[], f32 data }*``.
"""
from __future__ import annotations

import struct
from collections import OrderedDict
from typing import Dict

import numpy as np

from .config import BasecallModelConfig


def tensor_specs(cfg: BasecallModelConfig) -> "OrderedDict[str, tuple]":
    specs: "OrderedDict[str, tuple]" = OrderedDict()
    if cfg.is_tx_model:
        tx = cfg.tx
        for i, c in enumerate(cfg.convs):
            specs[f"conv.{i}.conv.weight.tensor"] = (c.size, c.insize, c.winlen)
            specs[f"conv.{i}.conv.bias.tensor"] = (c.size,)
        d, ff = tx.d_model, tx.dim_feedforward
        for l in range(tx.depth):
            p = f"transformer_encoder.{l}."
            specs[p + "self_attn.Wqkv.weight.tensor"] = (3 * d, d)
            specs[p + "self_attn.out_proj.weight.tensor"] = (d, d)
            specs[p + "self_attn.out_proj.bias.tensor"] = (d,)
            specs[p + "ff.fc1.weight.tensor"] = (2 * ff, d)
            specs[p + "ff.fc2.weight.tensor"] = (d, ff)
            specs[p + "norm1.weight.tensor"] = (d,)
            specs[p + "norm2.weight.tensor"] = (d,)
        specs["upsample.linear.weight.tensor"] = (tx.upsample_scale * d, d)
        specs["upsample.linear.bias.tensor"] = (tx.upsample_scale * d,)
        specs["crf.linear.weight.tensor"] = (cfg.outsize, d)
        return specs
    for i, c in enumerate(cfg.convs):
        specs[f"{i}.conv.weight.tensor"] = (c.size, c.insize, c.winlen)
        specs[f"{i}.conv.bias.tensor"] = (c.size,)
    C = cfg.lstm_size
    for l in range(cfg.lstm_layers):
        layer = len(cfg.convs) + l + 1  # the reference skips one index for the fused permute layer
        if cfg.is_flstm_model:  # crf_utils.cpp:36-41, shapes of FLSTMLayerImpl (nn/FLSTMStack.cpp:18-25)
            K = cfg.lstm_inner_dim
            specs[f"{layer}.rnn.dn_weight_ih.tensor"] = (K, C)
            specs[f"{layer}.rnn.dn_weight_hh.tensor"] = (K, C)
            specs[f"{layer}.rnn.up_weight_ih.tensor"] = (4 * C, K)
            specs[f"{layer}.rnn.up_weight_hh.tensor"] = (4 * C, K)
            specs[f"{layer}.rnn.up_bias_ih.tensor"] = (4 * C,)
            specs[f"{layer}.rnn.up_bias_hh.tensor"] = (4 * C,)
            continue
        specs[f"{layer}.rnn.weight_ih_l0.tensor"] = (4 * C, C)
        specs[f"{layer}.rnn.weight_hh_l0.tensor"] = (4 * C, C)
        specs[f"{layer}.rnn.bias_ih_l0.tensor"] = (4 * C,)
        specs[f"{layer}.rnn.bias_hh_l0.tensor"] = (4 * C,)
    layer = len(cfg.convs) + cfg.lstm_layers + 1
    if cfg.out_features is not None:
        specs[f"{layer}.linear.weight.tensor"] = (cfg.out_features, C)
        if cfg.bias:
            specs[f"{layer}.linear.bias.tensor"] = (cfg.out_features,)
        specs[f"{layer + 1}.linear.weight.tensor"] = (cfg.outsize, cfg.out_features)
    else:
        specs[f"{layer}.linear.weight.tensor"] = (cfg.outsize, C)
        if cfg.bias:   # pre-v4 models (crf_utils.cpp:82-86: the bias follows the weight whenever the config has one)
            specs[f"{layer}.linear.bias.tensor"] = (cfg.outsize,)
    return specs


def synthetic_weights(cfg: BasecallModelConfig, seed: int = 42, crf_gain: float | None = None
                      ) -> "OrderedDict[str, np.ndarray]":
    """Seeded fan-in-uniform weights; the CRF linear gets a gain so scores span the clamp range
    (with torch's default init the LSTM models emit |score| < 0.1 and every call is one base long)."""
    rng = np.random.default_rng(seed)
    out: "OrderedDict[str, np.ndarray]" = OrderedDict()
    for name, shape in tensor_specs(cfg).items():
        if "norm" in name:
            w = np.ones(shape, np.float32) + 0.05 * rng.standard_normal(shape).astype(np.float32)
        elif name.endswith("bias_hh_l0.tensor") or name.endswith("up_bias_hh.tensor"):
            w = np.zeros(shape, np.float32)
        elif len(shape) == 1:
            w = (0.1 * rng.uniform(-1, 1, shape)).astype(np.float32)
        else:
            fan_in = int(np.prod(shape[1:]))
            bound = 1.0 / np.sqrt(fan_in)
            gain = 1.0
            if "conv.weight" in name and not cfg.is_tx_model:
                gain = 2.5
            if "rnn.weight_ih" in name:
                gain = 6.0  # lively gates ...
            if "rnn.weight_hh" in name:
                gain = 1.5  # ... but a contractive recurrence: a chaotic LSTM would amplify fp16 rounding
            if "rnn.dn_weight" in name:
                gain = 2.0
            if "rnn.up_weight_ih" in name:
                gain = 3.0  # up @ dn then has about the spread of weight_ih above
            if "rnn.up_weight_hh" in name:
                gain = 0.75
            if name.endswith("linear.weight.tensor") and not cfg.is_tx_model and "upsample" not in name:
                gain = crf_gain if crf_gain is not None else 12.0
            if name == "crf.linear.weight.tensor" and crf_gain is not None:
                gain = crf_gain
            w = (gain * bound * rng.uniform(-1, 1, shape)).astype(np.float32)
        out[name] = np.ascontiguousarray(w)
    return out


def save_b2w(path, tensors: Dict[str, np.ndarray]) -> None:
    with open(path, "wb") as f:
        f.write(b"B2W1")
        f.write(struct.pack("<I", len(tensors)))
        for name, arr in tensors.items():
            nb = name.encode()
            arr = np.ascontiguousarray(arr, dtype=np.float32)
            f.write(struct.pack("<I", len(nb)))
            f.write(nb)
            f.write(struct.pack("<I", arr.ndim))
            f.write(struct.pack(f"<{arr.ndim}I", *arr.shape))
            f.write(arr.tobytes())


def load_b2w(path) -> "OrderedDict[str, np.ndarray]":
    out: "OrderedDict[str, np.ndarray]" = OrderedDict()
    with open(path, "rb") as f:
        if f.read(4) != b"B2W1":
            raise ValueError(f"{path}: not a B2W1 weight file")
        (n,) = struct.unpack("<I", f.read(4))
        for _ in range(n):
            (ln,) = struct.unpack("<I", f.read(4))
            name = f.read(ln).decode()
            (nd,) = struct.unpack("<I", f.read(4))
            dims = struct.unpack(f"<{nd}I", f.read(4 * nd))
            cnt = int(np.prod(dims)) if nd else 1
            out[name] = np.frombuffer(f.read(4 * cnt), dtype=np.float32).reshape(dims).copy()
    return out


def fold_flstm_weights(cfg: BasecallModelConfig, tensors: Dict[str, np.ndarray]) -> "OrderedDict[str, np.ndarray]":
    """The LSTM tensors an FLSTM model is equivalent to: gates = up_ih (dn_ih x_t) + up_hh (dn_hh h_{t-1}) + bias
    (nn/FLSTMStack.cpp:108-124) = (up_ih dn_ih) x_t + (up_hh dn_hh) h_{t-1} + bias.  The engine folds the same way (fp32
    products, lstm_model.cu), so an FLSTM model and its folded LSTM model produce identical scores."""
    out: "OrderedDict[str, np.ndarray]" = OrderedDict()
    for name, w in tensors.items():
        if ".rnn.dn_weight_ih." in name:
            p = name[: name.index("dn_weight_ih")]
            f32 = lambda k: np.asarray(tensors[p + k + ".tensor"], np.float32)
            out[p + "weight_ih_l0.tensor"] = (f32("up_weight_ih").astype(np.float64) @ f32("dn_weight_ih").astype(np.float64)).astype(np.float32)
            out[p + "weight_hh_l0.tensor"] = (f32("up_weight_hh").astype(np.float64) @ f32("dn_weight_hh").astype(np.float64)).astype(np.float32)
            out[p + "bias_ih_l0.tensor"] = f32("up_bias_ih")
            out[p + "bias_hh_l0.tensor"] = f32("up_bias_hh")
        elif ".rnn.dn_weight_hh." in name or ".rnn.up_" in name:
            continue
        else:
            out[name] = w
    return out


def modbase_tensor_specs(cfg) -> "OrderedDict[str, tuple]":
    """Tensors of a conv_lstm_v3 modified-base model in the order load_modbase_conv_lstm_weights reads them
    (dorado/modbase/nn/ModBaseModel.cpp:49-75), which is also the order of the module's parameters."""
    m = cfg.modules
    specs: "OrderedDict[str, tuple]" = OrderedDict()
    convs = [(f"sig_conv{i + 1}", c) for i, c in enumerate(m.signal_convs)]
    convs += [(f"seq_conv{i + 1}", c) for i, c in enumerate(m.sequence_convs)]
    convs.append(("merge_conv1", m.merge_conv))
    for name, c in convs:
        specs[f"{name}.weight.tensor"] = (c.size, c.insize, c.winlen)
        specs[f"{name}.bias.tensor"] = (c.size,)
    for l, (C, _) in enumerate(m.lstms):
        p = f"lstm{l + 1}."
        specs[p + "weight_ih_l0.tensor"] = (4 * C, C)
        specs[p + "weight_hh_l0.tensor"] = (4 * C, C)
        specs[p + "bias_ih_l0.tensor"] = (4 * C,)
        specs[p + "bias_hh_l0.tensor"] = (4 * C,)
    specs["fc.weight.tensor"] = (m.linear[1], m.linear[0])
    specs["fc.bias.tensor"] = (m.linear[1],)
    if m.upsample is not None:
        size, sf = m.upsample
        specs["linear_up.linear.weight.tensor"] = (sf * size, size)
        specs["linear_up.linear.bias.tensor"] = (sf * size,)
    return specs


def synthetic_modbase_weights(cfg, seed: int = 42) -> "OrderedDict[str, np.ndarray]":
    """Seeded fan-in-uniform weights with gains that keep the encoders' tanh units out of saturation, the LSTM gates
    lively but contractive (as synthetic_weights does for the basecaller), and the classes' logits a few units apart,
    so that the softmax is not flat."""
    rng = np.random.default_rng(seed)
    out: "OrderedDict[str, np.ndarray]" = OrderedDict()
    for name, shape in modbase_tensor_specs(cfg).items():
        if len(shape) == 1:
            w = (0.1 * rng.uniform(-1, 1, shape)).astype(np.float32)
        else:
            bound = 1.0 / np.sqrt(int(np.prod(shape[1:])))
            gain = 2.0
            if "weight_ih" in name:
                gain = 6.0
            elif "weight_hh" in name:
                gain = 1.5
            elif name == "fc.weight.tensor":
                gain = 16.0
            elif name.startswith("linear_up"):
                gain = 1.5
            w = (gain * bound * rng.uniform(-1, 1, shape)).astype(np.float32)
        out[name] = np.ascontiguousarray(w)
    return out
