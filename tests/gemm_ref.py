"""Float64 reference of the fp16 wgmma GEMM (dorado_b200/csrc/gemm.cu), restated from GemmDesc's documented semantics
(gemm.h) rather than from the kernel, with a per-element error bound.  Used by tests/test_gemm_plans_gpu.py against the
kernel (through b200_test_gemm_desc) and by tests/test_gemm_plans_cpu.py, which checks the addressing against plain loops
and that every check the GPU tests make can fail.

A descriptor is the keyword dict dorado_b200.lib.test_gemm_desc takes.  Semantics:
  - row g = batch * rows_per_batch + r reads A at batch * a_batch_stride + r * a_row_stride + k; elements with
    k >= a_inner (when a_inner > 0) read as zero;
  - v[g][n] = r_a[g] * sum_k A[g][k] W[n][k] + bias[n] (+ alpha * r_res[g] * res_gain[n] * residual[g * N + n]);
    r_a = rsqrt(mean(u^2) + eps) of A's own fp16 row u when a_ss is given (the gain is in W's columns), r_res the same
    of the residual row when res_ss is given;
  - output row g starts at out_offset + (g / out_m1) * out_s0 + (g % out_m1) * out_s1;
  - RoPE: within each 64-column head among the first rope_cols columns, (x1, x2) = (cols 0..31, cols 32..63) ->
    (cos x1 - sin x2, sin x1 + cos x2) at angle t * theta^(-2i / 64), t = g % rope_T, i the column within x1;
  - SwiGLU: columns (2j, 2j + 1) = (y, gate) -> y * silu(gate) in output column j;
  - out_ss: per row, the sum of squares of the stored fp16 values of each 32-column chunk.

The bound on |kernel - reference| per element, before the fp16 rounding of the output, is built from:
  - the accumulation, C_ACC K 2^-24 sum_k |a_k w_k|, times r_a where there is one.  C_ACC is the constant measured for the
    fp16 wgmma (DESIGN.md section 2);
  - the fp32 epilogue arithmetic, a few 2^-24 of each term;
  - rsqrtf (2 ulp) and the fp32 sums of the partial sums of squares, relative to r;
  - the fp32 RoPE table: the angle t * inv_freq rounded twice, the cos and sin rounded once;
  - tanh_fast (5e-5 absolute, the budget tests/test_lstm_int8_gpu.py uses) and swish_fast (1e-5 relative,
    tests/test_tx_fp8_gpu.py), each with the activation's largest slope times the pre-activation's bound.
then 2^-11 |ref| + 2^-25 for the fp16 rounding of the output.
"""
from __future__ import annotations

import numpy as np

ACT_NONE, ACT_SWISH, ACT_SWISH_CLAMP, ACT_TANH, ACT_TANH_X5, ACT_SWIGLU, ACT_ROPE = -1, 0, 1, 2, 3, 4, 5
U32 = 2.0 ** -24
C_ACC = 1.0
EPS_RSQRT = 2.0 ** -22      # rsqrtf: 2 ulp
EPS_TANH_FAST = 5e-5        # absolute
EPS_SWISH_FAST = 1e-5       # relative
SWISH_SLOPE = 1.1           # max |d/dv v sigmoid(v)| = 1.0998
SENTINEL = np.uint16(0x7E5A)   # a NaN the kernel never writes (its NaNs are 0x7FFF) and the inputs never hold


def rows_of(d):
    return d.get("batches", 1) * d["rows_per_batch"]


def n_out(d):
    return d["N"] // 2 if d.get("act", ACT_NONE) == ACT_SWIGLU else d["N"]


def a_index(d, g, k):
    """Flat A index of element k of row g (int64 arrays broadcast)."""
    rpb = d["rows_per_batch"]
    return (g // rpb) * d.get("a_batch_stride", 0) + (g % rpb) * d["a_row_stride"] + k


def a_rows(a, d, g):
    """float64 [len(g), K]: the K elements each row reads, zeros at and beyond a_inner."""
    K = d["K"]
    inner = d.get("a_inner", 0) or K
    k = np.arange(K)
    idx = a_index(d, g[:, None], k[None, :])
    live = np.broadcast_to(k[None, :] < inner, idx.shape)
    out = np.zeros(idx.shape)
    out[live] = a.astype(np.float64)[idx[live]]
    return out


def out_offsets(d, g=None):
    g = np.arange(rows_of(d), dtype=np.int64) if g is None else g
    m1 = d.get("out_m1", 1)
    return d.get("out_offset", 0) + (g // m1) * d["out_s0"] + (g % m1) * d.get("out_s1", 0)


def covered_a(d, a_len):
    """Boolean [a_len]: the A elements some row's K window covers (the others may hold anything, NaN included)."""
    cov = np.zeros(a_len, bool)
    inner = d.get("a_inner", 0) or d["K"]
    starts = a_index(d, np.arange(rows_of(d), dtype=np.int64), 0)
    for s in np.unique(starts):
        cov[s:s + inner] = True
    return cov


def rope_positions(d, g):
    return g % d["rope_T"]


def rope_angles(d, g):
    """float64 [len(g), 32]: t * theta^(-2i/64), t = g % rope_T."""
    i = np.arange(32)
    inv = float(d["theta"]) ** (-2.0 * i / 64.0)
    return rope_positions(d, g).astype(np.float64)[:, None] * inv[None, :]


def rope_cos_sin(ang):
    return np.cos(ang), np.sin(ang)


def inv_rms(u, norm_dim, eps):
    u = u[:, :norm_dim].astype(np.float64)
    return 1.0 / np.sqrt(np.mean(u * u, axis=1) + eps)


def partial_ss(rows):
    """fp32 [R, N / 32]: sums of squares of 32-column chunks of the fp16 rows (as out_ss lays them out), in float64."""
    r = rows.astype(np.float64)
    return (r * r).reshape(r.shape[0], -1, 32).sum(axis=2).astype(np.float32)


def _r_rel(norm_dim):
    """Relative error of the kernel's 1/rms: the fp32 sums of norm_dim squares, rsqrtf."""
    return 0.5 * (norm_dim + 2) * U32 + EPS_RSQRT


def reference(d, a, w, g, *, bias=None, residual=None, res_gain=None, a_ss=None, res_ss=None, alpha=0.0,
              c_acc=None, **_):
    """(ref [len(g), n_out], bound [len(g), n_out]) at rows g, float64.  a_ss / res_ss only say that the folded RMSNorm is
    on: the reference takes the norm of A's and the residual's own fp16 rows."""
    c_acc = C_ACC if c_acc is None else c_acc
    K, N, act = d["K"], d["N"], d.get("act", ACT_NONE)
    ar = a_rows(a, d, g)
    wf = w.astype(np.float64)
    acc = ar @ wf.T
    abs_acc = np.abs(ar) @ np.abs(wf).T
    r_a = np.ones(len(g))
    r_rel = 0.0
    if a_ss is not None:
        r_a = inv_rms(ar, d["norm_dim"], d.get("norm_eps", 1e-5))
        r_rel = _r_rel(d["norm_dim"])
    v = acc * r_a[:, None]
    e = (c_acc * K * U32 * abs_acc + r_rel * np.abs(acc) + 2 * U32 * np.abs(acc)) * r_a[:, None]
    if bias is not None:
        b = bias.astype(np.float64)[None, :]
        v = v + b
        e = e + 2 * U32 * (np.abs(v) + np.abs(b))
    if residual is not None:
        res = residual.astype(np.float64).reshape(-1)[(g[:, None] * N + np.arange(N)[None, :])]
        scale = np.full((len(g), 1), float(np.float32(alpha)))
        rr = 0.0
        if res_ss is not None:
            scale = scale * inv_rms(res, d["norm_dim"], d.get("norm_eps", 1e-5))[:, None]
            rr = _r_rel(d["norm_dim"])
        gain = res_gain.astype(np.float64)[None, :] if res_gain is not None else 1.0
        term = scale * gain * res
        v = v + term
        e = e + (rr + 4 * U32) * np.abs(term) + 2 * U32 * np.abs(v)
    if act == ACT_NONE:
        out, eo = v, e
    elif act in (ACT_SWISH, ACT_SWISH_CLAMP):
        out = v / (1.0 + np.exp(-v))
        eo = SWISH_SLOPE * e + EPS_SWISH_FAST * np.abs(out)
        if act == ACT_SWISH_CLAMP:
            out = np.minimum(out, 3.5)
    elif act == ACT_TANH:
        out, eo = np.tanh(v), e + EPS_TANH_FAST
    elif act == ACT_TANH_X5:
        out, eo = 5.0 * np.tanh(v), 5.0 * (e + EPS_TANH_FAST)
    elif act == ACT_SWIGLU:
        y, gate, ey, eg = v[:, 0::2], v[:, 1::2], e[:, 0::2], e[:, 1::2]
        sw = gate / (1.0 + np.exp(-gate))
        out = y * sw
        eo = np.abs(sw) * ey + np.abs(y) * SWISH_SLOPE * eg + ey * SWISH_SLOPE * eg + (EPS_SWISH_FAST + 2 * U32) * np.abs(out)
    elif act == ACT_ROPE:
        out, eo = v.copy(), e.copy()
        ang = rope_angles(d, g)
        cos, sin = rope_cos_sin(ang)
        e_tab = np.abs(ang) * 2 * U32 + 2 * U32   # the fp32 angle (inv_freq and the product rounded), then cos / sin
        for h0 in range(0, min(d["rope_cols"], N), 64):
            x1, x2 = v[:, h0:h0 + 32], v[:, h0 + 32:h0 + 64]
            e1, e2 = e[:, h0:h0 + 32], e[:, h0 + 32:h0 + 64]
            out[:, h0:h0 + 32] = cos * x1 - sin * x2
            out[:, h0 + 32:h0 + 64] = sin * x1 + cos * x2
            common = e_tab * (np.abs(x1) + np.abs(x2)) + 2 * U32 * (np.abs(x1) + np.abs(x2))
            eo[:, h0:h0 + 32] = np.abs(cos) * e1 + np.abs(sin) * e2 + common
            eo[:, h0 + 32:h0 + 64] = np.abs(sin) * e1 + np.abs(cos) * e2 + common
    else:
        raise ValueError(f"unknown activation {act}")
    return out, eo + 2.0 ** -11 * np.abs(out) + 2.0 ** -25


def logical_mask(d, out_len):
    """Boolean [out_len]: the elements the GEMM must write."""
    m = np.zeros(out_len, bool)
    offs = out_offsets(d)
    idx = offs[:, None] + np.arange(n_out(d))[None, :]
    m[idx.reshape(-1)] = True
    return m


def sentinel_buffer(out_len):
    return np.full(out_len, SENTINEL, np.uint16).view(np.float16)


def check_sentinel(d, out):
    """Nothing written outside the logical output, every element inside it written (and finite)."""
    bits = out.view(np.uint16)
    m = logical_mask(d, out.size)
    outside = int((bits[~m] != SENTINEL).sum())
    unwritten = int((bits[m] == SENTINEL).sum())
    nonfinite = int((~np.isfinite(out[m].astype(np.float32))).sum())
    assert outside == 0, f"{outside} elements written outside the logical output"
    assert unwritten == 0, f"{unwritten} elements of the logical output left unwritten"
    assert nonfinite == 0, f"{nonfinite} non-finite outputs"


def gather_out(d, out, g):
    """float64 [len(g), n_out] of the output buffer at rows g."""
    idx = out_offsets(d, g)[:, None] + np.arange(n_out(d))[None, :]
    return out.astype(np.float64)[idx]


def worst_ratio(got, ref, bound):
    return float((np.abs(got - ref) / bound).max())


def check_out_ss(got_rows, ss):
    """out_ss against float64 sums of squares of the kernel's own stored fp16 rows: 32 fp32 additions per partial."""
    want = (got_rows * got_rows).reshape(got_rows.shape[0], -1, 32).sum(axis=2)
    assert ss.shape == want.shape and np.isfinite(ss).all()
    return worst_ratio(ss.astype(np.float64), want, 32 * U32 * want + 1e-30)
