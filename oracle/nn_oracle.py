"""TEST INFRASTRUCTURE ONLY: numpy fp32 restatement of the reference network forward.

Follows the reference's CPU (libtorch) semantics layer by layer:
  conv stack        dorado/nn/ConvStack.cpp:103-163  (Conv1d pad=winlen//2, swish / swish_clamp 3.5 / tanh)
  LSTM stack        dorado/nn/LSTMStack.cpp:19-41    (torch LSTM equations, gates i,f,g,o; layers run
                                                       reverse,forward,reverse,... when reverse_first)
  linear CRF, clamp dorado/nn/CRFModules.cpp:15-34,125-134 ; model wiring dorado/basecall/model/CRFModel.cpp:29-62
  transformer       dorado/nn/TxModules.cpp:140-182 (GatedMLP), :184-250 (RoPE, half-split rotation),
                    :310-317 (window mask), :346-426 (MHA), :859-906 (encoder layer, deepnorm residual),
                    :1004-1016 (scaled CRF linear); RMSNorm dorado/nn/RMSNorm.cpp:14-18;
                    upsample dorado/nn/LinearUpsample.cpp:17-23; wiring dorado/basecall/model/TxModel.cpp:20-41
Checked against the compiled reference itself in tests/test_oracle_vs_reference.py.
"""
from __future__ import annotations

import numpy as np

from dorado_b200.config import ACT_SWISH, ACT_SWISH_CLAMP, ACT_TANH, BasecallModelConfig


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def conv1d(x, w, b, stride, act):
    """x [N,Cin,T] -> [N,Cout,T_out]."""
    N, Cin, T = x.shape
    Cout, _, W = w.shape
    pad = W // 2
    xp = np.pad(x, ((0, 0), (0, 0), (pad, pad)))
    T_out = (T + 2 * pad - W) // stride + 1
    s = xp.strides
    win = np.lib.stride_tricks.as_strided(xp, (N, T_out, Cin, W), (s[0], s[2] * stride, s[1], s[2]))
    y = win.reshape(N * T_out, Cin * W) @ w.reshape(Cout, Cin * W).T + b
    if act == ACT_SWISH:
        y = y * _sigmoid(y)
    elif act == ACT_SWISH_CLAMP:
        y = np.minimum(y * _sigmoid(y), 3.5)
    elif act == ACT_TANH:
        y = np.tanh(y)
    else:
        raise ValueError("Unrecognised activation function id.")
    return y.reshape(N, T_out, Cout).transpose(0, 2, 1).astype(np.float32)


def lstm_layer(x, w_ih, w_hh, b_ih, b_hh, reverse, quant=lambda a: a):
    """x [N,T,C] -> [N,T,C]; reverse runs the recurrence from the last timestep."""
    N, T, C = x.shape
    if reverse:
        x = x[:, ::-1]
    gx = quant(x @ w_ih.T + (b_ih + b_hh))   # the engine's x-projection GEMM stores gx as fp16
    h = np.zeros((N, C), np.float32)
    c = np.zeros((N, C), np.float32)
    out = np.empty((N, T, C), np.float32)
    whh_t = np.ascontiguousarray(w_hh.T)
    for t in range(T):
        g = gx[:, t] + h @ whh_t
        i, f, gg, o = g[:, :C], g[:, C:2 * C], g[:, 2 * C:3 * C], g[:, 3 * C:]
        c = _sigmoid(f) * c + _sigmoid(i) * np.tanh(gg)
        h = quant((_sigmoid(o) * np.tanh(c)).astype(np.float32))
        out[:, t] = h
    return out[:, ::-1] if reverse else out


def rmsnorm(x, w, eps=1e-5):
    return x * (1.0 / np.sqrt(np.mean(x * x, axis=-1, keepdims=True) + eps)) * w


def rope(qk, theta):
    """qk [N,T,H,D]: rotate (first half, second half) pairs by position (TxModules.cpp:220-250)."""
    N, T, H, D = qk.shape
    inv = (1.0 / np.power(np.float64(theta), np.arange(0, D, 2, dtype=np.float32) / np.float32(D))).astype(np.float32)
    ang = np.arange(T, dtype=np.float32)[:, None] * inv[None, :]
    cos, sin = np.cos(ang)[None, :, None, :], np.sin(ang)[None, :, None, :]
    a, b = qk[..., : D // 2], qk[..., D // 2:]
    return np.concatenate([cos * a - sin * b, sin * a + cos * b], axis=-1).astype(np.float32)


def windowed_attention(q, k, v, win, cpu_split_quirk=False, num_splits=12):
    """q,k,v [N,T,H,D]; query i attends keys j with -win[0] <= j-i <= win[1].

    cpu_split_quirk reproduces the reference's CPU fallback (TxModules.cpp:392-419), which slices
    keys to [qb-win_lower, qe+win_upper) per query split and so drops the key at +win_lower for the
    last query of every split."""
    N, T, H, D = q.shape
    up, lo = win
    i = np.arange(T)[:, None]
    j = np.arange(T)[None, :]
    mask = (j - i >= -up) & (j - i <= lo)
    if cpu_split_quirk:
        per = -(-T // num_splits)
        per = -(-per // 4) * 4
        for sp in range(num_splits):
            qb = sp * per
            if qb >= T:
                break
            qe = min(T, qb + per)
            kvb, kve = max(0, qb - lo), min(T, qe + up)
            mask[qb:qe, :kvb] = False
            mask[qb:qe, kve:] = False
    out = np.empty_like(q)
    scale = np.float32(1.0 / np.sqrt(D))
    for n in range(N):
        for h in range(H):
            s = (q[n, :, h] @ k[n, :, h].T) * scale
            s = np.where(mask, s, -np.inf)
            s = s - s.max(axis=-1, keepdims=True)
            p = np.exp(s)
            p /= p.sum(axis=-1, keepdims=True)
            out[n, :, h] = p @ v[n, :, h]
    return out


def _q16(a):
    return a.astype(np.float16).astype(np.float32)


def forward(cfg: BasecallModelConfig, w: dict, signal: np.ndarray, cpu_split_quirk: bool = False,
            return_intermediates: bool = False, emulate_fp16: bool = False):
    """signal [N,T] (or [N,1,T]) fp32 -> scores [N,T_out,C] fp32 (clamped when cfg.clamp).

    emulate_fp16=True models the storage precision of a CUDA half-precision path (the reference's own
    CUDA path, and this engine): matrix weights and every activation tensor that reaches HBM are rounded
    to fp16, arithmetic stays fp32."""
    x = np.ascontiguousarray(signal, np.float32).reshape(signal.shape[0], 1, -1)
    inter = {}
    q = _q16 if emulate_fp16 else (lambda a: a)
    w_in = w
    # LSTM models whose conv2 runs on the tensor cores (conv12_tc_kernel: conv1 -> 16 channels, conv2 with 5 taps): conv1's
    # output and conv2's weights are fp16 operands there; other shapes keep both in fp32 inside the fused FMA kernel
    conv2_tc = (not cfg.is_tx_model) and len(cfg.convs) == 3 and cfg.convs[0].size == 16 and cfg.convs[1].winlen == 5
    if emulate_fp16:
        keep32 = ("0.conv",) if conv2_tc else ("0.conv", "1.conv")
        w = {k: (_q16(v) if v.ndim >= 2 and not k.startswith(keep32) else v) for k, v in w.items()}
    if cfg.is_tx_model:
        tx = cfg.tx
        if emulate_fp16:
            w = dict(w)
            w["conv.0.conv.weight.tensor"] = w_in["conv.0.conv.weight.tensor"]  # conv1 runs in fp32
        for i, c in enumerate(cfg.convs):
            x = q(conv1d(x, w[f"conv.{i}.conv.weight.tensor"], w[f"conv.{i}.conv.bias.tensor"], c.stride, c.activation))
        x = x.transpose(0, 2, 1)
        inter["conv"] = x
        N, T, d = x.shape
        H, D = tx.nhead, tx.d_model // tx.nhead
        alpha = np.float32(tx.deepnorm_alpha)
        wc = q(w_in["crf.linear.weight.tensor"] * np.float32(tx.crf_scale))
        if emulate_fp16:
            # Rounding points of the engine (tx_model.cu): RMSNorm is folded into the GEMMs around it, so the normalised
            # x' = u * rsqrt(mean(u^2) + eps) * gain never reaches memory.  What is stored (fp16) is the un-normalised u;
            # its consumers multiply their fp32 accumulator rows by 1/rms and carry the gain in their (fp16) weight columns;
            # the residual term uses u, 1/rms and the gain in fp32.
            inv_rms = lambda u_: (1.0 / np.sqrt(np.mean(u_ * u_, axis=-1, keepdims=True) + 1e-5)).astype(np.float32)
            u_prev, r_prev, g_prev = x, None, None          # before layer 0 the conv output is used as is
            for l in range(tx.depth):
                p = f"transformer_encoder.{l}."
                n1, n2 = w_in[p + "norm1.weight.tensor"], w_in[p + "norm2.weight.tensor"]
                wq = w_in[p + "self_attn.Wqkv.weight.tensor"]
                wq = _q16(wq * g_prev[None, :]) if g_prev is not None else _q16(wq)
                acc = u_prev @ wq.T
                if r_prev is not None:
                    acc = acc * r_prev
                qkv = acc.reshape(N, T, 3, H, D)
                qq, k, v = q(rope(qkv[:, :, 0], tx.theta)), q(rope(qkv[:, :, 1], tx.theta)), q(qkv[:, :, 2])
                a = q(windowed_attention(qq, k, v, tx.attn_window, cpu_split_quirk).reshape(N, T, d))
                xn = u_prev * r_prev * g_prev if r_prev is not None else u_prev
                u_mid = q(a @ w[p + "self_attn.out_proj.weight.tensor"].T + w[p + "self_attn.out_proj.bias.tensor"] + xn * alpha)
                r_mid = inv_rms(u_mid)
                t = (u_mid @ _q16(w_in[p + "ff.fc1.weight.tensor"] * n1[None, :]).T) * r_mid
                y, gate = t[..., : tx.dim_feedforward], t[..., tx.dim_feedforward:]
                hid = q((gate * _sigmoid(gate)) * y)
                u_prev = q(hid @ w[p + "ff.fc2.weight.tensor"].T + (u_mid * r_mid * n1) * alpha)
                r_prev, g_prev = inv_rms(u_prev), n2
                if l == 0:
                    inter["layer0"] = u_prev * r_prev * g_prev
            inter["encoder"] = u_prev * r_prev * g_prev if r_prev is not None else u_prev
            wu = w_in["upsample.linear.weight.tensor"]
            wu = _q16(wu * g_prev[None, :]) if g_prev is not None else _q16(wu)
            acc = u_prev @ wu.T
            if r_prev is not None:
                acc = acc * r_prev
            u = q(acc + w["upsample.linear.bias.tensor"])
        else:
            for l in range(tx.depth):
                p = f"transformer_encoder.{l}."
                qkv = (x @ w[p + "self_attn.Wqkv.weight.tensor"].T).reshape(N, T, 3, H, D)
                qq, k, v = rope(qkv[:, :, 0], tx.theta), rope(qkv[:, :, 1], tx.theta), qkv[:, :, 2]
                a = windowed_attention(qq, k, v, tx.attn_window, cpu_split_quirk).reshape(N, T, d)
                a = a @ w[p + "self_attn.out_proj.weight.tensor"].T + w[p + "self_attn.out_proj.bias.tensor"] + x * alpha
                x = rmsnorm(a, w[p + "norm1.weight.tensor"]).astype(np.float32)
                t = x @ w[p + "ff.fc1.weight.tensor"].T
                y, gate = t[..., : tx.dim_feedforward], t[..., tx.dim_feedforward:]
                f = ((gate * _sigmoid(gate)) * y) @ w[p + "ff.fc2.weight.tensor"].T + x * alpha
                x = rmsnorm(f, w[p + "norm2.weight.tensor"]).astype(np.float32)
                if l == 0:
                    inter["layer0"] = x
            inter["encoder"] = x
            u = x @ w["upsample.linear.weight.tensor"].T + w["upsample.linear.bias.tensor"]
        u = u.reshape(N, tx.upsample_scale * T, d)
        scores = q(u @ wc.T)
        scores = scores.astype(np.float32)
        return (scores, inter) if return_intermediates else scores

    for i, c in enumerate(cfg.convs):
        x = conv1d(x, w[f"{i}.conv.weight.tensor"], w[f"{i}.conv.bias.tensor"], c.stride, c.activation)
        if i >= 1 or conv2_tc:
            x = q(x)  # conv1's output stays on chip (fused conv1+conv2 kernel); as the tensor-core operand it is fp16
        inter[f"conv{i}"] = x
    x = np.ascontiguousarray(x.transpose(0, 2, 1))
    nconv = len(cfg.convs)
    for l in range(cfg.lstm_layers):
        p = f"{nconv + l + 1}.rnn."
        if getattr(cfg, "lstm_inner_dim", None):
            # FLSTM (nn/FLSTMStack.cpp:108-124; the reference has no CPU forward for it): gates = up_ih (dn_ih x_t) +
            # up_hh (dn_hh h_{t-1}) + bias = an LSTM whose gate matrices are the products up @ dn
            f64 = lambda k: np.asarray(w_in[p + k + ".tensor"], np.float64)
            w_ih = (f64("up_weight_ih") @ f64("dn_weight_ih")).astype(np.float32)
            w_hh = (f64("up_weight_hh") @ f64("dn_weight_hh")).astype(np.float32)
            if emulate_fp16:
                w_ih, w_hh = _q16(w_ih), _q16(w_hh)
            x = lstm_layer(x, w_ih, w_hh, w[p + "up_bias_ih.tensor"], w[p + "up_bias_hh.tensor"], reverse=(l % 2 == 0), quant=q)
        else:
            x = lstm_layer(x, w[p + "weight_ih_l0.tensor"], w[p + "weight_hh_l0.tensor"], w[p + "bias_ih_l0.tensor"],
                           w[p + "bias_hh_l0.tensor"], reverse=(l % 2 == 0), quant=q)
        inter[f"lstm{l}"] = x
    layer = nconv + cfg.lstm_layers + 1
    scores = x @ w[f"{layer}.linear.weight.tensor"].T
    if f"{layer}.linear.bias.tensor" in w:
        scores = scores + w[f"{layer}.linear.bias.tensor"]
    if cfg.out_features is not None:
        scores = q(scores) @ w[f"{layer + 1}.linear.weight.tensor"].T
    if cfg.scale == 5.0:
        scores = np.tanh(scores) * np.float32(5.0)
    scores = q(scores)
    if cfg.clamp:
        scores = np.clip(scores, -5.0, 5.0)
    scores = scores.astype(np.float32)
    return (scores, inter) if return_intermediates else scores
