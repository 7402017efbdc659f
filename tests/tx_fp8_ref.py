"""TEST INFRASTRUCTURE ONLY: numpy restatement of the transformer forward in the engine's fp8_ffn precision
(include/b200call.h, b200_model_desc.tx_precision), with the rounding points of dorado_b200/csrc/tx_model.cu:

  weights   fp16(w) for every matrix (the reference holds the model in fp16, CudaCaller.cpp:167); remove_bits = 4 on the
            QKV and out_proj weights and both RMSNorm gains (TxModules.cpp:104-111, 443-453), before the norm2 gain is
            folded into the next QKV's (and the upsample's) columns and rounded to fp16 again; fc1 / fc2 weights are
            E4M3 casts of the fp16 values (TxModules.cpp:560-575, torch.float8_e4m3fn); the out_proj bias stays fp32
  norm1     an explicit pass: fp16(RMSNorm(u) * gain), and its E4M3 cast (from the fp16 value) is fc1's A
  fc1       E4M3 x E4M3, fp32 accumulation; y * silu(gate) in fp32, cast to E4M3 saturating at +-448
  fc2       E4M3 x E4M3, fp32 accumulation, + alpha * the fp16 norm1 output, stored fp16; norm2 stays folded as in fp16
Everything else is oracle/nn_oracle.py's emulate_fp16 path (the engine's folded RMSNorm layout)."""
from __future__ import annotations

import numpy as np
import torch

from oracle.nn_oracle import _q16, _sigmoid, conv1d, rope, windowed_attention

E4M3_MAX = 448.0


def remove_bits(a, bits=4):
    """fp16(a) with the reference's apply_rounding: (int16 bits + 2^(bits-1)) & ~(2^bits - 1), wrapping; returns fp16."""
    h = np.ascontiguousarray(a, np.float16).view(np.uint16).astype(np.uint32)
    return (((h + (1 << (bits - 1))) & (0xFFFF & ~((1 << bits) - 1))).astype(np.uint16)).view(np.float16)


def e4m3(a):
    """torch's float8_e4m3fn cast (round to nearest even, NaN beyond the range), as float32 values."""
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.float8_e4m3fn).to(torch.float32).numpy()


def e4m3_bytes(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def e4m3_sat(a):
    """The device's cvt.rn.satfinite.e4m3x2.f32: as the torch cast, but +-448 beyond the range."""
    return e4m3(np.clip(a, -E4M3_MAX, E4M3_MAX))


def decode_e4m3(b):
    return torch.from_numpy(np.ascontiguousarray(b, np.uint8)).view(torch.float8_e4m3fn).to(torch.float32).numpy()


def prepare_weights(cfg, w):
    """The per-layer weights of the fp8_ffn precision before any gain folding: float32 values."""
    out = {}
    for l in range(cfg.tx.depth):
        p = f"transformer_encoder.{l}."
        for k in ("self_attn.Wqkv.weight", "self_attn.out_proj.weight", "norm1.weight", "norm2.weight"):
            out[p + k] = remove_bits(w[p + k + ".tensor"]).astype(np.float32)
        out[p + "self_attn.out_proj.bias"] = np.asarray(w[p + "self_attn.out_proj.bias.tensor"], np.float32)
        for k in ("ff.fc1.weight", "ff.fc2.weight"):
            out[p + k] = e4m3(np.asarray(w[p + k + ".tensor"], np.float16).astype(np.float32))
    return out


def forward(cfg, w, signal):
    """signal [N, T] -> scores [N, T_out, C] float32, emulating the fp8_ffn engine's storage precision."""
    tx = cfg.tx
    x = np.ascontiguousarray(signal, np.float32).reshape(signal.shape[0], 1, -1)
    for i, c in enumerate(cfg.convs):
        cw = w[f"conv.{i}.conv.weight.tensor"]
        x = _q16(conv1d(x, cw if i == 0 else _q16(cw), w[f"conv.{i}.conv.bias.tensor"], c.stride, c.activation))
    x = x.transpose(0, 2, 1)
    N, T, d = x.shape
    H, D, ff = tx.nhead, d // tx.nhead, tx.dim_feedforward
    alpha = np.float32(tx.deepnorm_alpha)
    pw = prepare_weights(cfg, w)
    inv_rms = lambda u_: (1.0 / np.sqrt(np.mean(u_ * u_, axis=-1, keepdims=True) + 1e-5)).astype(np.float32)
    u_prev, r_prev, g_prev = x, None, None
    for l in range(tx.depth):
        p = f"transformer_encoder.{l}."
        wq = pw[p + "self_attn.Wqkv.weight"]
        wq = _q16(wq * g_prev[None, :]) if g_prev is not None else wq
        acc = u_prev @ wq.T
        if r_prev is not None:
            acc = acc * r_prev
        qkv = acc.reshape(N, T, 3, H, D)
        qq, k, v = _q16(rope(qkv[:, :, 0], tx.theta)), _q16(rope(qkv[:, :, 1], tx.theta)), _q16(qkv[:, :, 2])
        a = _q16(windowed_attention(qq, k, v, tx.attn_window).reshape(N, T, d))
        xn = u_prev * r_prev * g_prev if r_prev is not None else u_prev
        u_mid = _q16(a @ pw[p + "self_attn.out_proj.weight"].T + pw[p + "self_attn.out_proj.bias"] + xn * alpha)
        nrm = _q16(u_mid * inv_rms(u_mid) * pw[p + "norm1.weight"])
        t = e4m3(nrm) @ pw[p + "ff.fc1.weight"].T
        y, gate = t[..., :ff], t[..., ff:]
        hid = e4m3_sat((gate * _sigmoid(gate)) * y)
        u_prev = _q16(hid @ pw[p + "ff.fc2.weight"].T + nrm * alpha)
        r_prev, g_prev = inv_rms(u_prev), pw[p + "norm2.weight"]
    wu = w["upsample.linear.weight.tensor"]
    wu = _q16(wu * g_prev[None, :]) if g_prev is not None else _q16(wu)
    acc = u_prev @ wu.T
    if r_prev is not None:
        acc = acc * r_prev
    u = _q16(acc + w["upsample.linear.bias.tensor"]).reshape(N, tx.upsample_scale * T, d)
    wc = _q16(w["crf.linear.weight.tensor"] * np.float32(tx.crf_scale))
    return _q16(u @ wc.T).astype(np.float32)
