"""TEST INFRASTRUCTURE ONLY: numpy restatement of the transformer in the engine's int8_qkv_fp8_ffn precision
(include/b200call.h, b200_model_desc.tx_precision = 2), with the rounding points of dorado_b200/csrc/tx_model.cu and
gemm.cu (DESIGN.md section 2):

  weights     as tests/tx_fp8_ref.prepare_weights (fp16, remove_bits = 4 on out_proj and both gains, E4M3 fc1 / fc2), and
              Wqkv as int8 per output row from the fp16 weights BEFORE remove_bits: quantize_act's arithmetic, with the
              factor inv = 1 / float(scale16) (quantize_tensor(fp16(Wqkv), -1), scale.reciprocal_()).  No gain is folded
              into any weight; the upsample weight is fp16(w).
  quantise    per row of fp16 values: scale16 = fp16(128 / absmax), q = clip(rne(fp16(x scale16)), -127, 127),
              inv = 1 / float(scale16) in fp32.  An all-zero row gets q = 0; a row whose scale overflows to +inf gets
              inv = 0, and in it a zero element's product 0 * inf is NaN, which the clip takes to -127 (quantize_rows_f16).
              Applied to the last conv's fp16 output (the stack input) and to every norm2 output.
  qkv         s32 accumulation of the int8 operands, v = (float32(acc) * inv_row) * inv_col with every step rounded to
              fp32 (float32(acc) rounds beyond 2^24), RoPE in fp32, fp16 output
  out_proj    fp16(att Wo^T + bo + alpha x), x the layer's normalised fp16 input (the conv output before layer 0)
  norm1, fc1  as fp8_ffn: an explicit pass writing fp16 and its E4M3 copy; E4M3 fc1 + SwiGLU -> E4M3
  fc2         fp16(E4M3 product + alpha * norm1's fp16 output)
  norm2       an explicit pass: x = fp16(RMSNorm(u) g2), then quantised as above

The second half restates the plan's launches for tests/test_tx_i8_gpu.py's launch-by-launch check: the launch list, the
workspace layout (fp8_ffn's blocks, then the int8 copy of x and its factors), the buffers each launch writes and a
per-launch float64 reference (I8LayerRef) built on tests/tx_layer_ref.py's.
"""
from __future__ import annotations

import numpy as np

import tx_layer_ref as X
from oracle.nn_oracle import _q16, _sigmoid, conv1d, rope, windowed_attention
from tx_fp8_ref import e4m3, e4m3_sat, prepare_weights as prepare_fp8_weights

MODE = "int8_qkv_fp8_ffn"
U32 = 2.0 ** -24


# ---- the quantiser and the weights ------------------------------------------------------------------------------------
def quantize_act(x, levels=128):
    """fp16 values [rows, cols] -> (int8 q [rows, cols], fp16 scale16 [rows], fp32 inv [rows]).  levels: the numerator of
    the scale (128 in the reference; other values only for the sensitivity checks)."""
    h = np.asarray(x, np.float16)
    absmax = np.abs(h).max(axis=1).astype(np.float32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        scale16 = (np.float32(levels) / absmax).astype(np.float16)
        s = scale16.astype(np.float32)
        prod = (h.astype(np.float32) * s[:, None]).astype(np.float16).astype(np.float32)
        # np.fmax / np.fmin return the non-NaN operand: a NaN product clips to -127, as fmaxf and std::max do
        q = np.fmin(np.float32(127), np.fmax(np.float32(-127), np.rint(prod)))
        inv = (np.float32(1) / s).astype(np.float32)
    q[absmax == 0] = 0
    return q.astype(np.int8), scale16, inv


def prepare_weights(cfg, w):
    """fp8_ffn's weights (tests/tx_fp8_ref.prepare_weights) with each layer's Wqkv replaced by its int8 rows
    ("self_attn.Wqkv.q") and their factors ("self_attn.Wqkv.inv")."""
    out = prepare_fp8_weights(cfg, w)
    for l in range(cfg.tx.depth):
        p = f"transformer_encoder.{l}.self_attn.Wqkv"
        del out[p + ".weight"]
        q, _, inv = quantize_act(np.asarray(w[p + ".weight.tensor"], np.float16))
        out[p + ".q"], out[p + ".inv"] = q, inv
    return out


def s8_product(qa, inv_a, qw, inv_w):
    """(float32(acc) * inv_a[row]) * inv_w[col] with fp32 rounding after each step; acc the exact integer product."""
    acc = qa.astype(np.int64) @ qw.astype(np.int64).T
    return (acc.astype(np.float32) * inv_a.astype(np.float32)[:, None]) * inv_w.astype(np.float32)[None, :]


# ---- the whole forward ------------------------------------------------------------------------------------------------
def forward(cfg, w, signal):
    """signal [N, T] -> scores [N, T_out, C] float32, emulating the int8_qkv_fp8_ffn engine's storage precision."""
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
    x = x.reshape(N * T, d)
    q, _, inv = quantize_act(x)
    for l in range(tx.depth):
        p = f"transformer_encoder.{l}."
        v = s8_product(q, inv, pw[p + "self_attn.Wqkv.q"], pw[p + "self_attn.Wqkv.inv"]).reshape(N, T, 3, H, D)
        qq, k, vv = _q16(rope(v[:, :, 0], tx.theta)), _q16(rope(v[:, :, 1], tx.theta)), _q16(v[:, :, 2])
        a = _q16(windowed_attention(qq, k, vv, tx.attn_window).reshape(N * T, d))
        u_mid = _q16(a @ pw[p + "self_attn.out_proj.weight"].T + pw[p + "self_attn.out_proj.bias"] + x * alpha)
        nrm = _q16(u_mid * inv_rms(u_mid) * pw[p + "norm1.weight"])
        t = e4m3(nrm) @ pw[p + "ff.fc1.weight"].T
        y, gate = t[..., :ff], t[..., ff:]
        hid = e4m3_sat((gate * _sigmoid(gate)) * y)
        u = _q16(hid @ pw[p + "ff.fc2.weight"].T + nrm * alpha)
        x = _q16(u * inv_rms(u) * pw[p + "norm2.weight"])
        q, _, inv = quantize_act(x)
    u = _q16(x @ _q16(w["upsample.linear.weight.tensor"]).T + w["upsample.linear.bias.tensor"])
    u = u.reshape(N, tx.upsample_scale * T, d)
    wc = _q16(w["crf.linear.weight.tensor"] * np.float32(tx.crf_scale))
    return _q16(u @ wc.T).astype(np.float32)


# ---- the plan, launch by launch ---------------------------------------------------------------------------------------
# the mistakes the sensitivity checks simulate, each on the reference of one launch kind
MUTATIONS = {
    "quantiser_127_levels": "qkv",   # the int8 copy of x quantised with 127 / absmax in place of 128 / absmax
    "w_factor_not_inverted": "qkv",  # Wqkv's column factor scale16 in place of 1 / scale16
    "norm2_gain_twice": "norm2",     # norm2 with its gain applied twice
}


def launches(cfg):
    """[(profile name, kind, layer or conv index)] in TxPlan::run's order."""
    out = [("tx_conv1", "conv1", 0)] + [("tx_conv_gemm", "conv", i) for i in range(1, len(cfg.convs))]
    out.append(("quantize_i8", "quantize", 0))
    for l in range(cfg.tx.depth):
        out += [("qkv_gemm", "qkv", l), ("tx_attention", "attention", l), ("out_proj_gemm", "out_proj", l),
                ("rmsnorm_e4m3", "norm1", l), ("fc1_swiglu_gemm", "fc1", l), ("fc2_gemm", "fc2", l),
                ("rmsnorm_i8", "norm2", l)]
    return out + [("upsample_gemm", "upsample", 0), ("crf_gemm", "crf", 0)]


def launch_count(cfg):
    """conv1, the conv GEMMs, the stack input's quantise pass, 7 per layer, upsample, CRF."""
    return 1 + (len(cfg.convs) - 1) + 1 + 7 * cfg.tx.depth + 2


def workspace_layout(cfg, N, T_in):
    """TxModel::carve in this precision: fp8_ffn's blocks, then x8 (rows x d_model bytes) and x_inv (rows x 4 bytes)."""
    lay = X.workspace_layout(cfg, N, T_in, "fp8_ffn")
    rows, off = lay["rows"], lay["bytes"]
    for name, nbytes in (("x8", rows * cfg.tx.d_model), ("x_inv", rows * 4)):
        lay["buffers"][name] = (off, nbytes)
        off += (nbytes + 255) // 256 * 256
    lay["bytes"] = off
    return lay


def writes(cfg, lay, kind, idx):
    """{buffer: byte range written (None: all of it)} of one launch."""
    rows, dm, ff = lay["rows"], cfg.tx.d_model, cfg.tx.dim_feedforward
    if kind == "quantize":
        return {"x8": None, "x_inv": None}
    if kind == "out_proj":
        return {"y": None}
    if kind == "norm1":
        return {"att": None, "qkv": (0, rows * dm)}
    if kind == "fc1":
        return {"hid": (0, rows * ff)}
    if kind == "fc2":
        return {"y": None}
    if kind == "norm2":
        return {"x": None, "x8": None, "x_inv": None}
    return X.writes(cfg, lay, kind, idx, "fp8_ffn")


def logical_inputs(cfg, lay, raw):
    """tx_layer_ref.logical_inputs of fp8_ffn, plus x8 (int8 [rows][d_model]) and x_inv (fp32 [rows])."""
    inp = X.logical_inputs(cfg, lay, raw, "fp8_ffn")
    rows, dm = lay["rows"], cfg.tx.d_model
    inp._loaders["x8"] = lambda: raw["x8"].view(np.int8).reshape(rows, dm)
    inp._loaders["x_inv"] = lambda: raw["x_inv"].view(np.float32)
    return inp


class I8LayerRef(X.TxLayerRef):
    """The float64 reference of each launch in this precision.  reference(kind, idx, inp) as tx_layer_ref's; "quantize"
    and the int8 copy norm2 writes are checked bit for bit against quantize_act of the engine's own fp16 rows instead
    (the returned x is norm2's fp16 output with its bound)."""

    def __init__(self, cfg, w, N, T_in):
        super().__init__(cfg, w, "fp8_ffn", N, T_in)   # fp8_ffn's weights and the launches it shares
        self.lay = workspace_layout(cfg, N, T_in)
        self.q = {l: (q, inv) for l in range(cfg.tx.depth)
                  for q, _, inv in [quantize_act(np.asarray(w[f"transformer_encoder.{l}.self_attn.Wqkv.weight.tensor"],
                                                            np.float16))]}

    def _layer_input(self, l, x, raw=False, gain_layer=None):
        # nothing is folded: x holds the normalised rows (the conv output before layer 0)
        return x, 0.0

    def reference(self, kind, idx, inp, mutation=None):
        if mutation is not None:
            assert MUTATIONS[mutation] == kind, (mutation, kind)
        if kind == "qkv":
            qw, invw = self.q[idx]
            if mutation == "w_factor_not_inverted":
                invw = (np.float32(1) / invw).astype(np.float32)
            if mutation == "quantiser_127_levels":
                qa, _, inva = quantize_act(inp["x"].astype(np.float16), levels=127)
            else:
                qa, inva = inp["x8"], inp["x_inv"]
            acc = qa.astype(np.int64) @ qw.astype(np.int64).T
            v = acc.astype(np.float64) * inva.astype(np.float64)[:, None] * invw.astype(np.float64)[None, :]
            # float32(acc) (exact below 2^24, else one rounding) and two fp32 products
            e = 3 * U32 * np.abs(v)
            g = np.arange(self.N * self.T)
            return {"qkv": X._out16(*X._rope(v, e, g % self.T, self.cfg.tx.theta, 2 * self.dm))}
        if kind == "fc2":
            (_, pair), = super().reference(kind, idx, inp).items()
            return {"y": pair}
        if kind == "norm2":
            g = self._lw(idx, "norm2.weight")
            ref = X.rmsnorm(inp["y"], g * g if mutation == "norm2_gain_twice" else g)
            return {"x": (ref, (self.r_rel + 3 * U32 + X.U11) * np.abs(ref) + 2.0 ** -25)}
        if kind == "quantize":
            raise ValueError("the quantise pass is checked bit for bit, not within a bound")
        return super().reference(kind, idx, inp, mutation)
