"""TEST INFRASTRUCTURE ONLY: numpy restatement of the int8_lstm precision of the LSTM models (include/b200call.h,
b200_model_desc.lstm_precision), with the rounding points of dorado_b200/csrc/lstm_model.cu and gemm.cu (DESIGN.md §2):

  weights       per LSTM layer fp16(W_ih) | fp16(W_hh) as one [4C, 2C] matrix, per row: scale = fp16(128 / absmax),
                q = clip(round_half_even(fp16(w * scale)), -127, 127) -- utils::quantize_tensor(w, 1) evaluated on an fp16
                tensor (every operation computes in fp32 and rounds to fp16).  The first CRF linear likewise per output row.
                inv[row] = 1 / (127 * scale[row]) in fp32; an all-zero row has q = 0 and inv = 0.
  activations   int8 round_half_even(127 * v) (ACT_SCALE) of conv3's tanh output and of every h_t
  x-projection  gx = fp16(float(acc) * inv[row] + (b_ih + b_hh)), acc the exact integer product
  recurrence    pre = fp32(float(acc) * inv[row]) + gx; gates, fp32 cell state; h_t quantised once
  CRF linear    scores = fp16(float(acc) * inv[row] (+ bias)); a second linear stays fp16 x fp16

The engine's tanh is an approximation (tanh.approx.f32, 2^-11), here it is exact: model scores are compared within a
bound, the integer GEMMs bit for bit.  check_layer holds one engine layer to the teacher-forced float64 reference of
tests/lstm_layer_ref.py, run on the dequantised weights and activations.
"""
from __future__ import annotations

import numpy as np

import lstm_layer_ref as R

ACT_SCALE = np.float32(127.0)


def quantize_rows(w):
    """fp16 values [rows, cols] -> (int8 [rows, cols], fp16 scale [rows], fp32 inv [rows])."""
    w16 = np.asarray(w, np.float16)
    absmax = np.abs(w16).max(axis=1).astype(np.float32)
    zero = absmax == 0
    with np.errstate(divide="ignore", over="ignore"):   # 128 / absmax beyond fp16's range is inf, as in torch
        scale = (np.float32(128.0) / absmax).astype(np.float16)
    prod = (w16.astype(np.float32) * np.where(zero, 0, scale).astype(np.float32)[:, None]).astype(np.float16)
    q = np.clip(np.rint(prod.astype(np.float32)), -127, 127).astype(np.int8)
    with np.errstate(divide="ignore"):
        inv = np.where(zero, np.float32(0), np.float32(1.0) / (ACT_SCALE * scale.astype(np.float32))).astype(np.float32)
    return q, scale, inv


def quant_act(v):
    """int8 of an activation in [-1, 1]: cvt.rni.sat.s8(127 * v) with the product in fp32."""
    return np.clip(np.rint(ACT_SCALE * np.asarray(v, np.float32)), -128, 127).astype(np.int8)


def layer_params(cfg, w, l):
    """(q_ih [4C, C], q_hh [4C, C], inv [4C], bias [4C] fp32) of LSTM layer l."""
    p = f"{len(cfg.convs) + l + 1}.rnn."
    both = np.concatenate([w[p + "weight_ih_l0.tensor"], w[p + "weight_hh_l0.tensor"]], axis=1).astype(np.float16)
    q, _, inv = quantize_rows(both)
    C = cfg.lstm_size
    bias = np.asarray(w[p + "bias_ih_l0.tensor"], np.float32) + np.asarray(w[p + "bias_hh_l0.tensor"], np.float32)
    return q[:, :C], q[:, C:], inv, bias


def linear_params(cfg, w):
    layer = len(cfg.convs) + cfg.lstm_layers + 1
    q, _, inv = quantize_rows(np.asarray(w[f"{layer}.linear.weight.tensor"], np.float16))
    return q, inv, w.get(f"{layer}.linear.bias.tensor")


def _imatmul(a8, q):
    """Exact integer a8 [M, K] x q [N, K]^T as float32 (every partial sum is an integer below 2^24)."""
    return a8.astype(np.float32) @ q.astype(np.float32).T


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def conv3_tanh(cfg, w, signal):
    """conv3's fp32 tanh output [N, T_out, C] with the engine's fp16 storage points before it."""
    from oracle import nn_oracle
    x = np.ascontiguousarray(signal, np.float32).reshape(signal.shape[0], 1, -1)
    q16 = lambda a: a.astype(np.float16).astype(np.float32)
    conv2_tc = cfg.convs[0].size == 16 and cfg.convs[1].winlen == 5
    for i, c in enumerate(cfg.convs):
        wt = w[f"{i}.conv.weight.tensor"]
        if i == 2 or (i == 1 and conv2_tc):
            wt = q16(wt)
        x = nn_oracle.conv1d(x, wt, w[f"{i}.conv.bias.tensor"], c.stride, c.activation)
        if i == 1 or (i == 0 and conv2_tc):
            x = q16(x)
    return np.ascontiguousarray(x.transpose(0, 2, 1))


def lstm_layer(x8, q_ih, q_hh, inv, bias, reverse):
    """x8 int8 [N, T, C] -> int8 [N, T, C]."""
    N, T, C = x8.shape
    if reverse:
        x8 = x8[:, ::-1]
    gx = (_imatmul(x8.reshape(N * T, C), q_ih) * inv + bias).astype(np.float16).astype(np.float32).reshape(N, T, 4 * C)
    h8 = np.zeros((N, C), np.int8)
    c = np.zeros((N, C), np.float32)
    out = np.empty((N, T, C), np.int8)
    for t in range(T):
        g = _imatmul(h8, q_hh) * inv + gx[:, t]
        i, f, gg, o = g[:, :C], g[:, C:2 * C], g[:, 2 * C:3 * C], g[:, 3 * C:]
        c = (_sigmoid(f) * c + _sigmoid(i) * np.tanh(gg)).astype(np.float32)
        h8 = quant_act(_sigmoid(o) * np.tanh(c))
        out[:, t] = h8
    return out[:, ::-1] if reverse else out


def forward(cfg, w, signal, return_intermediates=False):
    """signal [N, T] -> scores [N, T_out, outsize] fp32 (clamped when cfg.clamp), in the int8_lstm precision."""
    inter = {}
    x8 = quant_act(conv3_tanh(cfg, w, signal))
    inter["conv2"] = x8
    for l in range(cfg.lstm_layers):
        x8 = lstm_layer(x8, *layer_params(cfg, w, l), reverse=(l % 2 == 0))
        inter[f"lstm{l}"] = x8
    N, T, C = x8.shape
    q, inv, bias = linear_params(cfg, w)
    scores = _imatmul(x8.reshape(N * T, C), q) * inv
    if bias is not None:
        scores = scores + np.asarray(bias, np.float32)
    layer = len(cfg.convs) + cfg.lstm_layers + 1
    if cfg.out_features is not None:
        w2 = np.asarray(w[f"{layer + 1}.linear.weight.tensor"], np.float16).astype(np.float32)
        scores = scores.astype(np.float16).astype(np.float32) @ w2.T
    if cfg.scale == 5.0:
        scores = np.tanh(scores) * np.float32(5.0)
    scores = scores.astype(np.float16).astype(np.float32).reshape(N, T, -1)
    if cfg.clamp:
        scores = np.clip(scores, -5.0, 5.0)
    return (scores, inter) if return_intermediates else scores


# ---- one engine layer against the teacher-forced float64 reference ------------------------------------------------------
def dequantised_layer_weights(cfg, w, l):
    """The layer as lstm_layer_ref sees it: activations v = level / 127 and W = q * (127 inv), so that W v is the engine's
    float(acc) * inv exactly."""
    q_ih, q_hh, inv, bias = layer_params(cfg, w, l)
    s = (inv.astype(np.float64) * 127.0)[:, None]
    return R.LayerWeights(q_ih.astype(np.float64) * s, q_hh.astype(np.float64) * s, bias.astype(np.float64))


def check_layer(X8, H8, lw, reverse, steps=None, kappa=R.KAPPA):
    """X8, H8 int8 [T, N, C]: the engine's layer input and output.  From the engine's own h_{t-1} and the float64 gx, the
    reference's h_t must quantise to the engine's level e, or lie within its error budget of the tie next to e:
    |127 h - e| <= 0.5 + 127 kappa dh.  Returns (ratio [T, N, C] of the excess over 0.5 to the budget, 0 where not compared;
    fraction of compared elements whose level differs from round(127 h); tidx)."""
    X = X8.astype(np.float64) / 127.0
    H = H8.astype(np.float64) / 127.0
    h, dh, tidx = R.reference_layer(X, lw, reverse, steps, H=H)
    got = R._gather(H8, tidx)
    valid = (tidx >= 0)[..., None]
    excess = np.abs(127.0 * h - got) - 0.5
    ratio = np.where(valid, np.maximum(excess, 0.0) / (127.0 * kappa * dh + 1e-12), 0.0)
    differs = np.where(valid, np.rint(127.0 * h) != got, False)
    return ratio, float(differs.sum() / max(1, np.broadcast_to(valid, differs.shape).sum())), tidx
