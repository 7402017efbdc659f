"""Float64 reference of every kernel launch of the transformer plan (TxModel::make_plan and TxPlan::run in
dorado_b200/csrc/tx_model.cu), each fed the engine's own input buffers, with a per-element error bound.

The semantics are the modules', not the engine's fold: TxEncoderImpl with an explicit RMSNorm(u) = u rsqrt(mean(u^2) +
1e-5) g, RoPE at the position t within the chunk (half-split rotation), the true window -win_upper <= j - i <= win_lower,
SwiGLU as silu(gate) y with y the first dim_feedforward rows of fc1, the deepnorm residual + alpha x', the upsample's
rows read as [N][T scale][d_model] by the CRF linear, whose weights are scaled by crf_scale.  The weights are the
model's float32 values; in the fp8_ffn precision those of tests/tx_fp8_ref.prepare_weights (remove_bits on the fp16
weights and gains, E4M3 fc1 / fc2).

Modes: "fold" (the default: RMSNorm folded into the GEMMs around it), "rmsnorm_pass" (B200_TX_RMSNORM_PASS=1: a
separate rmsnorm_kernel after every sub-layer) and "fp8_ffn" (an explicit norm1 pass writing fp16 and E4M3, E4M3 fc1 and
fc2).  The launches of each mode, their buffers and the workspace layout are restated in launches(), writes() and
workspace_layout().

The bound on |kernel - reference| is tests/gemm_ref.py's, per element:
  - the fp32 accumulation C_ACC K 2^-24 sum_k |a_k w_k| (a the normalised input where there is a norm);
  - one fp16 rounding per weight, 2^-11 sum_k |a_k w_k| (+ 2^-24 sum_k |a_k| for subnormal weights, gains above 1/2):
    the reference holds W, the engine fp16(W) or, where a gain g is folded into the columns, fp16(W g);
  - the fp32 epilogue (a few 2^-24 of each term), rsqrtf and the fp32 sums of squares behind 1/rms (gemm_ref._r_rel),
    the fp32 RoPE table, swish_fast (1e-5 relative) with the activation's largest slope;
  - 2^-11 |ref| + 2^-25 for the fp16 rounding of the output.
Attention: per element, 2^-11 sum_j p_j |v_j| for the fp16 weights P before P V, the relative error of the weights
(the fp32 sums of q . k, ex2.approx), the fp32 accumulation of P V and 2^-11 |out| for the output (attention()).  This
is the per-element form of test_attention_kernel's 1.5e-3 max|v|: on a model's near-uniform attention sum_j p_j |v_j| is
several times below max|v|, and the coarser budget would not see a window one key narrower.
fp8_ffn fc1 / fc2: the E4M3 wgmma accumulation (K / 32) 2^-14 sum |a b| (tests/test_tx_fp8_gpu.py); fc1's E4M3 output
must be the saturating cast of a value within the bound of the float64 one.
rmsnorm: the fp32 sum of d_model squares and rsqrtf (_r_rel), two fp32 products and the fp16 output; its E4M3 copy must be
the cvt.rn.satfinite cast of the fp16 output, bit for bit.
"""
from __future__ import annotations

import numpy as np

import gemm_ref as R
from tx_fp8_ref import decode_e4m3, e4m3_bytes, prepare_weights

MODES = ("fold", "rmsnorm_pass", "fp8_ffn")
U11 = 2.0 ** -11            # fp16 unit roundoff
U32 = R.U32
EPS = 1e-5
E4M3_MAX = 448.0

# the mistakes the sensitivity checks simulate, each on the reference of one launch kind
MUTATIONS = {
    "qkv_gain_of_layer_l": "qkv",         # the norm2 gain of layer l instead of layer l - 1 in qkv
    "rope_global_position": "qkv",        # RoPE at the row g instead of g % T
    "window_narrower": "attention",       # a window one key narrower (win_upper - 1)
    "out_proj_no_alpha": "out_proj",      # the residual without alpha
    "out_proj_raw_residual": "out_proj",  # the residual u in place of the normalised x'
    "fc1_swap": "fc1",                    # the y and gate halves of fc1 swapped
    "fc2_n2_gain": "fc2",                 # fc2's residual with the n2 gain in place of n1
    "upsample_step_major": "crf",         # the upsample's rows read step-major instead of row-major
}


# ---- the plan and its workspace ---------------------------------------------------------------------------------------
def conv_shapes(cfg, T_in):
    """TxModel::shapes: per conv (t, pad, t_pad): its output length, the front padding of its buffer (the next conv's
    winlen / 2, 0 for the last) and the buffer's rows t + 2 pad + 16."""
    out, t = [], T_in
    for i, c in enumerate(cfg.convs):
        t = (t + 2 * (c.winlen // 2) - c.winlen) // c.stride + 1
        pad = cfg.convs[i + 1].winlen // 2 if i + 1 < len(cfg.convs) else 0
        out.append((t, pad, t + 2 * pad + 16))
    return out


def launches(cfg, mode):
    """[(profile name, kind, layer or conv index)] in TxPlan::run's order."""
    assert mode in MODES
    out = [("tx_conv1", "conv1", 0)] + [("tx_conv_gemm", "conv", i) for i in range(1, len(cfg.convs))]
    for l in range(cfg.tx.depth):
        out += [("qkv_gemm", "qkv", l), ("tx_attention", "attention", l), ("out_proj_gemm", "out_proj", l)]
        if mode != "fold":
            out.append(("rmsnorm_e4m3" if mode == "fp8_ffn" else "rmsnorm", "norm1", l))
        out += [("fc1_swiglu_gemm", "fc1", l), ("fc2_gemm", "fc2", l)]
        if mode == "rmsnorm_pass":
            out.append(("rmsnorm", "norm2", l))
    return out + [("upsample_gemm", "upsample", 0), ("crf_gemm", "crf", 0)]


def launch_count(cfg, mode):
    """TxPlan::launches(): conv1, the conv GEMMs, 5 (fold), 7 (rmsnorm_pass) or 6 (fp8_ffn) per layer, upsample, CRF."""
    per = {"fold": 5, "rmsnorm_pass": 7, "fp8_ffn": 6}[mode]
    return 1 + (len(cfg.convs) - 1) + cfg.tx.depth * per + 2


def workspace_layout(cfg, N, T_in, mode):
    """TxModel::carve: {buffer: (byte offset, bytes)} in carve order, each block 256-byte aligned, and the shapes.
    The layout is the same in every mode; what each mode keeps where is writes()'s business."""
    assert mode in MODES
    tx = cfg.tx
    sh = conv_shapes(cfg, T_in)
    T = sh[-1][0]
    rows, dm = N * T, tx.d_model
    blocks = [(f"cbuf{i}", N * sh[i][2] * cfg.convs[i].size * 2) for i in range(len(cfg.convs) - 1)]
    blocks += [("x", rows * dm * 2), ("y", rows * dm * 2), ("att", rows * dm * 2), ("qkv", rows * 3 * dm * 2),
               ("hid", rows * tx.dim_feedforward * 2), ("ups", rows * tx.upsample_scale * dm * 2),
               ("ss_a", rows * (dm // 32) * 4), ("ss_b", rows * (dm // 32) * 4)]
    buffers, off = {}, 0
    for name, nbytes in blocks:
        buffers[name] = (off, nbytes)
        off += (nbytes + 255) // 256 * 256
    return {"buffers": buffers, "bytes": off, "T": T, "rows": rows, "convs": sh}


def writes(cfg, lay, kind, idx, mode):
    """{buffer: byte range written (None: all of it)} of one launch.  The CRF writes the scores, outside the workspace."""
    rows, dm, ff = lay["rows"], cfg.tx.d_model, cfg.tx.dim_feedforward
    nconv = len(cfg.convs)
    if kind == "conv1":
        return {"cbuf0": None}
    if kind == "conv":
        return {"x": None} if idx == nconv - 1 else {f"cbuf{idx}": None}
    if kind == "qkv":
        return {"qkv": None}
    if kind == "attention":
        return {"att": None}
    if kind == "out_proj":
        return {"y": None, "ss_b": None} if mode == "fold" else {"y": None}
    if kind == "norm1":
        return {"att": None, "qkv": (0, rows * dm)} if mode == "fp8_ffn" else {"x": None}
    if kind == "fc1":
        return {"hid": (0, rows * ff)} if mode == "fp8_ffn" else {"hid": None}
    if kind == "fc2":
        return {"y": None} if mode == "rmsnorm_pass" else {"x": None, "ss_a": None}
    if kind == "norm2":
        return {"x": None}
    if kind == "upsample":
        return {"ups": None}
    if kind == "crf":
        return {}
    raise ValueError(kind)


class _Lazy(dict):
    """A dict whose values are computed on first use."""

    def __init__(self, loaders):
        super().__init__()
        self._loaders = loaders

    def __missing__(self, key):
        self[key] = self._loaders[key]()
        return self[key]


def logical_inputs(cfg, lay, raw, mode):
    """The buffers of a workspace snapshot (raw: {buffer: uint8 bytes}) as float64 arrays, converted when first read:
    conv{i} the valid rows [N][t][C] of cbuf i (conv{n-1} is x as [N][T][d_model]), x, y, att [rows][d_model], qkv
    [rows][3 d_model], hid [rows][ff], ups [rows][scale d_model]; in fp8_ffn also a8 (the E4M3 rows at the start of
    qkv's buffer) and hid8 (the E4M3 rows at the start of hid's)."""
    rows, T, dm, ff = lay["rows"], lay["T"], cfg.tx.d_model, cfg.tx.dim_feedforward
    N = rows // T
    f16 = lambda name, shape: raw[name].view(np.float16).reshape(shape).astype(np.float64)
    loaders = {"x": lambda: f16("x", (rows, dm)), "y": lambda: f16("y", (rows, dm)), "att": lambda: f16("att", (rows, dm)),
               "qkv": lambda: f16("qkv", (rows, 3 * dm)), "hid": lambda: f16("hid", (rows, ff)),
               "ups": lambda: f16("ups", (rows, cfg.tx.upsample_scale * dm)),
               f"conv{len(cfg.convs) - 1}": lambda: f16("x", (N, T, dm))}
    for i in range(len(cfg.convs) - 1):
        t, pad, tp = lay["convs"][i]
        loaders[f"conv{i}"] = lambda i=i, t=t, pad=pad, tp=tp: f16(f"cbuf{i}", (N, tp, cfg.convs[i].size))[:, pad:pad + t]
    if mode == "fp8_ffn":
        loaders["a8"] = lambda: decode_e4m3(raw["qkv"][:rows * dm]).astype(np.float64).reshape(rows, dm)
        loaders["hid8"] = lambda: decode_e4m3(raw["hid"][:rows * ff]).astype(np.float64).reshape(rows, ff)
    return _Lazy(loaders)


def cbuf_padding_nonzero(cfg, lay, raw, i):
    """Elements of cbuf i outside its valid rows that are not +0.0 (the next conv reads them as its zero padding)."""
    t, pad, tp = lay["convs"][i]
    N = lay["rows"] // lay["T"]
    bits = raw[f"cbuf{i}"].view(np.uint16).reshape(N, tp, cfg.convs[i].size)
    keep = np.ones(tp, bool)
    keep[pad:pad + t] = False
    return int((bits[:, keep] != 0).sum())


# ---- float64 pieces ---------------------------------------------------------------------------------------------------
def sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def rmsnorm(u, g):
    return u / np.sqrt(np.mean(u * u, axis=1, keepdims=True) + EPS) * g


def _linear(a, W, bias=None, r_rel=0.0, w_fp16=True):
    """(a W^T + bias, bound before the epilogue's activation and output rounding); a [R][K] the module's input (already
    normalised), W [N][K] the module's weights, r_rel the relative error of the engine's 1/rms where it computes one."""
    K = a.shape[1]
    acc = a @ W.T
    absacc = np.abs(a) @ np.abs(W).T
    e = R.C_ACC * K * U32 * absacc + (r_rel + 2 * U32) * np.abs(acc)
    if w_fp16:
        e += (U11 + U32) * absacc + 2.0 ** -24 * np.abs(a).sum(axis=1, keepdims=True)
    v = acc
    if bias is not None:
        v = acc + bias[None, :]
        e = e + 2 * U32 * (np.abs(v) + np.abs(bias)[None, :])
    return v, e


def _residual(v, e, res, alpha, r_rel):
    """+ alpha res (the deepnorm residual; r_rel where the engine normalises res itself)."""
    term = float(np.float32(alpha)) * res
    v = v + term
    return v, e + (r_rel + 4 * U32) * np.abs(term) + 2 * U32 * np.abs(v)


def _out16(v, e):
    return v, e + U11 * np.abs(v) + 2.0 ** -25


def _swish(v, e, act):
    out = v * sigmoid(v)
    eo = R.SWISH_SLOPE * e + R.EPS_SWISH_FAST * np.abs(out)
    if act == R.ACT_SWISH_CLAMP:
        out = np.minimum(out, 3.5)
    elif act != R.ACT_SWISH:
        raise ValueError(f"transformer convs use swish, got activation {act}")
    return out, eo


def _swiglu(v, e, ff, swap=False):
    y, gate, ey, eg = v[:, :ff], v[:, ff:], e[:, :ff], e[:, ff:]
    if swap:
        y, gate, ey, eg = gate, y, eg, ey
    sw = gate * sigmoid(gate)
    out = y * sw
    eo = np.abs(sw) * ey + np.abs(y) * R.SWISH_SLOPE * eg + ey * R.SWISH_SLOPE * eg + (R.EPS_SWISH_FAST + 2 * U32) * np.abs(out)
    return out, eo


def _rope(v, e, pos, theta, cols):
    """RotaryEmbedding on the first `cols` columns, 64-column heads split (x1, x2) = (0..31, 32..63), angle
    pos theta^(-2i/64); with the bound of the fp32 table (gemm_ref's ACT_ROPE)."""
    out, eo = v.copy(), e.copy()
    inv = float(theta) ** (-2.0 * np.arange(32) / 64.0)
    ang = pos.astype(np.float64)[:, None] * inv[None, :]
    cos, sin = np.cos(ang), np.sin(ang)
    e_tab = np.abs(ang) * 2 * U32 + 2 * U32
    for h0 in range(0, cols, 64):
        x1, x2 = v[:, h0:h0 + 32], v[:, h0 + 32:h0 + 64]
        e1, e2 = e[:, h0:h0 + 32], e[:, h0 + 32:h0 + 64]
        out[:, h0:h0 + 32] = cos * x1 - sin * x2
        out[:, h0 + 32:h0 + 64] = sin * x1 + cos * x2
        common = (e_tab + 2 * U32) * (np.abs(x1) + np.abs(x2))
        eo[:, h0:h0 + 32] = np.abs(cos) * e1 + np.abs(sin) * e2 + common
        eo[:, h0 + 32:h0 + 64] = np.abs(sin) * e1 + np.abs(cos) * e2 + common
    return out, eo


def attention(qkv, N, T, H, win):
    """softmax(q k^T / 8) v over -win[0] <= j - i <= win[1] from qkv [N T][3][H][64], and its bound per element.

    tx_attention_tc_kernel rounds each weight p_j = exp2(s_j - m) to fp16 before P V while its normaliser l sums the fp32
    weights: at most 2^-11 sum_j p_j |v_j| (relative 2^-11 per normal weight; n 2^-25 max|v| for subnormal ones, l >= 1).
    A relative error eps of every weight moves the output by at most 2 eps sum_j p_j |v_j|: eps holds the fp32 sums of
    s = q . k (64 2^-24 sum_d |q_d k_d| in log2 units), the fp32 scaling and running max (4 2^-24 |s|), ex2.approx
    (2^-22) and the running-max rescaling.  P V and l accumulate n fp32 terms (n 2^-24 each, C_ACC = 1 as the fp16 GEMM),
    1 / l and the product 2 2^-24, and the output is rounded to fp16: 2^-11 |out| + 2^-25."""
    up, lo = win
    x = qkv.reshape(N, T, 3, H, 64)
    i, j = np.arange(T)[:, None], np.arange(T)[None, :]
    mask = (j - i >= -up) & (j - i <= lo)
    nkeys = mask.sum(axis=1)[:, None].astype(np.float64)
    log2e = 1.0 / np.log(2.0)
    out = np.empty((N, T, H, 64))
    bound = np.empty((N, T, H, 64))
    for n in range(N):
        for h in range(H):
            q, k, v = x[n, :, 0, h], x[n, :, 1, h], x[n, :, 2, h]
            s = np.where(mask, q @ k.T / 8.0, -np.inf)
            p = np.exp(s - s.max(axis=1, keepdims=True))
            p /= p.sum(axis=1, keepdims=True)
            o = p @ v
            pv = p @ np.abs(v)
            qk = np.where(mask, np.abs(q) @ np.abs(k).T, 0.0).max(axis=1, keepdims=True)
            smax = np.where(mask, np.abs(s), 0.0).max(axis=1, keepdims=True)
            eps = np.log(2.0) * (64 * U32 * qk / 8.0 * log2e + 4 * U32 * smax * log2e) + 2.0 ** -22 + 6 * U32
            vmax = np.where(mask, np.abs(v).max(axis=1)[None, :], 0.0).max(axis=1)[:, None]
            out[n, :, h] = o
            bound[n, :, h] = ((U11 + 2 * eps + (2 * nkeys + 4) * U32) * pv + nkeys * 2.0 ** -25 * vmax
                              + U11 * np.abs(o) + 2.0 ** -25)
    return out.reshape(N * T, H * 64), bound.reshape(N * T, H * 64)


def e4m3_sat_bytes(v):
    """cvt.rn.satfinite.e4m3x2.f32: round to nearest even, +-448 beyond the range."""
    return e4m3_bytes(np.clip(np.asarray(v, np.float32), -E4M3_MAX, E4M3_MAX))


def e4m3_cast_check(got_bytes, v, tol):
    """(outside, ratio): an E4M3 output must be the saturating cast of a value within tol of the float64 v.  outside
    counts the elements that are not; ratio = |got - v| / the largest |cast - v| the criterion admits there (<= 1 inside
    the interval; printed, and the sensitivity mutations must reach 3)."""
    cast = lambda a: decode_e4m3(e4m3_sat_bytes(a)).astype(np.float64)
    g = decode_e4m3(got_bytes).astype(np.float64)
    lo, hi = cast(v - tol), cast(v + tol)
    outside = int(((g < lo) | (g > hi)).sum())
    admit = np.maximum(np.maximum(hi - v, v - lo), 2.0 ** -10)
    return outside, np.abs(g - v) / admit


# ---- one launch -------------------------------------------------------------------------------------------------------
class TxLayerRef:
    """The reference of each launch of one model in one mode.  reference(kind, idx, inp) takes the float64 input
    buffers (logical_inputs' names, plus "signal" [N][T_in]) and returns {output: (ref, bound)}; for fc1 in fp8_ffn the
    pair is (v, tol) of e4m3_cast_check."""

    def __init__(self, cfg, w, mode, N, T_in):
        assert mode in MODES
        self.cfg, self.mode, self.N, self.T_in = cfg, mode, N, T_in
        self.lay = workspace_layout(cfg, N, T_in, mode)
        self.T = self.lay["T"]
        w64 = {k: np.asarray(v, np.float64) for k, v in w.items()}
        if mode == "fp8_ffn":
            w64.update({k + ".tensor": np.asarray(v, np.float64) for k, v in prepare_weights(cfg, w).items()})
        self.w = w64
        tx = cfg.tx
        self.dm, self.ff, self.H = tx.d_model, tx.dim_feedforward, tx.nhead
        self.r_rel = R._r_rel(self.dm)

    def _lw(self, l, name):
        return self.w[f"transformer_encoder.{l}.{name}.tensor"]

    def _gain2(self, l):
        return self._lw(l, "norm2.weight")

    def _layer_input(self, l, x, raw=False, gain_layer=None):
        """(module input of layer l's qkv / out_proj residual from the x buffer, r_rel): x itself before layer 0 and in
        rmsnorm_pass (the buffer holds the normalised rows), else RMSNorm(x) with layer l - 1's norm2 gain."""
        if l == 0 or self.mode == "rmsnorm_pass" or raw:
            return x, 0.0
        g = self._gain2(l - 1 if gain_layer is None else gain_layer)
        return rmsnorm(x, g), self.r_rel

    def reference(self, kind, idx, inp, mutation=None):
        if mutation is not None:
            assert MUTATIONS[mutation] == kind, (mutation, kind)
        cfg, tx, N, T = self.cfg, self.cfg.tx, self.N, self.T
        if kind == "conv1":
            c = cfg.convs[0]
            W = self.w["conv.0.conv.weight.tensor"][:, 0, :]
            b = self.w["conv.0.conv.bias.tensor"]
            sig = inp["signal"]
            pad = c.winlen // 2
            xp = np.pad(sig, ((0, 0), (pad, pad)))
            win = np.lib.stride_tricks.sliding_window_view(xp, c.winlen, axis=1)[:, :sig.shape[1]].reshape(-1, c.winlen)
            v = win @ W.T + b[None, :]
            e = (c.winlen + 1) * U32 * (np.abs(win) @ np.abs(W).T + np.abs(b)[None, :])
            out, eo = _out16(*_swish(v, e, c.activation))
            return {"conv0": (out.reshape(N, -1, c.size), eo.reshape(N, -1, c.size))}
        if kind == "conv":
            c = cfg.convs[idx]
            Wt = self.w[f"conv.{idx}.conv.weight.tensor"]            # [Cout][Cin][winlen]
            Wm = Wt.transpose(0, 2, 1).reshape(c.size, c.winlen * c.insize)
            xin = inp[f"conv{idx - 1}"]                               # [N][t_in][Cin]
            pad = c.winlen // 2
            t_out = self.lay["convs"][idx][0]
            xp = np.pad(xin, ((0, 0), (pad, pad), (0, 0)))
            win = np.lib.stride_tricks.sliding_window_view(xp, c.winlen, axis=1)   # [N][t][Cin][winlen]
            win = win[:, ::c.stride][:, :t_out].transpose(0, 1, 3, 2).reshape(N * t_out, -1)
            v, e = _linear(win, Wm, bias=self.w[f"conv.{idx}.conv.bias.tensor"])
            out, eo = _out16(*_swish(v, e, c.activation))
            name = "x" if idx == len(cfg.convs) - 1 else f"conv{idx}"
            shape = (N * t_out, c.size) if name == "x" else (N, t_out, c.size)
            return {name: (out.reshape(shape), eo.reshape(shape))}
        l = idx
        if kind == "qkv":
            gl = l if mutation == "qkv_gain_of_layer_l" else None
            a, rr = self._layer_input(l, inp["x"], gain_layer=gl)
            v, e = _linear(a, self._lw(l, "self_attn.Wqkv.weight"), r_rel=rr)
            g = np.arange(N * T)
            pos = g if mutation == "rope_global_position" else g % T
            return {"qkv": _out16(*_rope(v, e, pos, tx.theta, 2 * self.dm))}
        if kind == "attention":
            win = tx.attn_window
            if mutation == "window_narrower":
                win = (win[0] - 1, win[1])
            return {"att": attention(inp["qkv"], N, T, self.H, win)}
        if kind == "out_proj":
            v, e = _linear(inp["att"], self._lw(l, "self_attn.out_proj.weight"), bias=self._lw(l, "self_attn.out_proj.bias"))
            res, rr = self._layer_input(l, inp["x"], raw=mutation == "out_proj_raw_residual")
            alpha = 1.0 if mutation == "out_proj_no_alpha" else tx.deepnorm_alpha
            return {"y": _out16(*_residual(v, e, res, alpha, rr))}
        if kind in ("norm1", "norm2"):
            u = inp["y"]
            g = self._lw(l, "norm1.weight" if kind == "norm1" else "norm2.weight")
            ref = rmsnorm(u, g)
            bound = (self.r_rel + 3 * U32 + U11) * np.abs(ref) + 2.0 ** -25
            return {"att" if self.mode == "fp8_ffn" else "x": (ref, bound)}
        if kind == "fc1":
            if self.mode == "fp8_ffn":
                a, W = inp["a8"], self._lw(l, "ff.fc1.weight")
                t = a @ W.T
                bt = a.shape[1] / 32 * 2.0 ** -14 * (np.abs(a) @ np.abs(W).T)
                return {"hid8": _swiglu(t, bt, self.ff, swap=mutation == "fc1_swap")}
            if self.mode == "fold":
                a, rr = rmsnorm(inp["y"], self._lw(l, "norm1.weight")), self.r_rel
            else:
                a, rr = inp["x"], 0.0
            v, e = _linear(a, self._lw(l, "ff.fc1.weight"), r_rel=rr)
            return {"hid": _out16(*_swiglu(v, e, self.ff, swap=mutation == "fc1_swap"))}
        if kind == "fc2":
            W = self._lw(l, "ff.fc2.weight")
            if self.mode == "fp8_ffn":
                a = inp["hid8"]
                acc = a @ W.T
                e = a.shape[1] / 32 * 2.0 ** -14 * (np.abs(a) @ np.abs(W).T) + 2 * U32 * np.abs(acc)
                return {"x": _out16(*_residual(acc, e, inp["att"], tx.deepnorm_alpha, 0.0))}
            v, e = _linear(inp["hid"], W)
            if self.mode == "fold":
                g = self._lw(l, "norm2.weight" if mutation == "fc2_n2_gain" else "norm1.weight")
                return {"x": _out16(*_residual(v, e, rmsnorm(inp["y"], g), tx.deepnorm_alpha, self.r_rel))}
            return {"y": _out16(*_residual(v, e, inp["x"], tx.deepnorm_alpha, 0.0))}
        if kind == "upsample":
            a, rr = self._layer_input(tx.depth, inp["x"]) if tx.depth > 0 else (inp["x"], 0.0)
            v, e = _linear(a, self.w["upsample.linear.weight.tensor"], bias=self.w["upsample.linear.bias.tensor"], r_rel=rr)
            return {"ups": _out16(v, e)}
        if kind == "crf":
            s = tx.upsample_scale
            ups = inp["ups"].reshape(N, T, s, self.dm)
            if mutation == "upsample_step_major":
                ups = ups.transpose(0, 2, 1, 3)
            v, e = _linear(ups.reshape(N * T * s, self.dm), self.w["crf.linear.weight.tensor"] * float(tx.crf_scale))
            out, eo = _out16(v, e)
            return {"scores": (out.reshape(N, T * s, -1), eo.reshape(N, T * s, -1))}
        raise ValueError(kind)


def worst_ratio(got, ref, bound):
    return float((np.abs(got - ref) / bound).max())


def ss_ratio(rows, ss):
    """A partial-sums-of-squares buffer against the float64 sums of squares of the engine's own stored rows."""
    return R.check_out_ss(rows, ss.reshape(rows.shape[0], -1))
