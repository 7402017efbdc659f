"""Float64 reference of one LSTM layer of the engine, teacher-forced on the engine's own outputs, and its error budget.

For layer l the engine's sequence buffer holds X (the layer input, after l layers) and H (its output, after l + 1 layers),
both fp16 [T_out][N][C].  The reference follows the kernels' rounding points in float64:
  - W_ih and W_hh rounded to fp16; the bias b_ih + b_hh summed in fp32 (LstmModel's constructor);
  - gx = fp16(X W_ih^T + b), rounded once;
  - teacher forcing: the recurrent input of step s is the engine's own h of step s - 1 (0 at the first step), so
    pre = gx + W_hh H[t_prev] and errors do not compound through h; only the cell state c is carried along the
    reference's own chain, in float64;
  - h_ref = sigmoid(o) tanh(c) before rounding, compared with H[t].
Layers with even l run reversed (reverse_first).  With variable chunk sizes chunk n runs over its own steps_n = len_n /
stride steps, a reversed layer from t = steps_n - 1; rows t >= steps_n are unspecified and not compared.

The tolerance is a first-order error budget computed along the reference.  Each activated gate carries
  - the MUFU error of tanh.approx.f32, a relative error of at most 2^-10.987 (PTX ISA, tanh); the sigmoid is
    0.5 tanh(0.5 v) + 0.5 (gate_act in lstm_model.cu), so its absolute error is 0.5 eps |tanh(v / 2)|;
  - the error of its pre-activation times the activation's slope: one fp16 ulp of gx (the kernel may round a gx
    one ulp away from the float64 one) plus the fp32 accumulation terms gamma_C (sum |W_ih x| + sum |W_hh h|).
The cell error follows dc_t <= f dc_{t-1} + |c_{t-1}| d_f + |g| d_i + |i| d_g, the output error
dh_t <= |tanh c| d_o + o (eps |tanh c| + (1 - tanh^2 c) dc_t), and every element must satisfy
|H - h_ref| <= ulp16(h_ref) + KAPPA dh_t.  Two refinements keep the bound valid where the linearisation is not: each
product of two inexact factors also carries the product of their errors (it dominates where o and tanh c are both
near 0), and each slope is the largest within the argument's error, not the slope at the reference's point.
The budget grows like 1 / (1 - f) only where the reference's own f is near 1, so one rule covers short and long cell
memory.  A simulated kernel with the full MUFU error on every activation reaches 2/3 of it (1 / KAPPA: the rounding of
h to fp16 is the one term not scaled by KAPPA); the H100 kernels stay below 0.41 (tests/test_lstm_layers_gpu.py).
"""
from __future__ import annotations

import dataclasses

import numpy as np

EPS_TANH = 2.0 ** -10.987   # max relative error of tanh.approx.f32
KAPPA = 1.5
U32 = 2.0 ** -24            # fp32 unit roundoff


def q16(a):
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


def ulp16(a):
    """fp16 spacing at |a| (at a power of two, the spacing of the binade above)."""
    return np.spacing(np.abs(np.asarray(a, np.float64)).astype(np.float16)).astype(np.float64)


def _tanh_slope(slope, dv):
    """Largest slope of tanh within v +- dv, from its slope at v: |tanh''| <= 4 / (3 sqrt 3) < 0.77, tanh' <= 1."""
    return np.minimum(slope + 0.77 * dv, 1.0)


def _sig_slope(slope, dv):
    """Largest slope of the sigmoid within v +- dv: |sigmoid''| <= 1 / (6 sqrt 3) < 0.097, sigmoid' <= 1 / 4."""
    return np.minimum(slope + 0.097 * dv, 0.25)


# ---- the engine's workspace -------------------------------------------------------------------------------------------
def workspace_layout(cfg, N, T_in):
    """Byte offsets of LstmModel::make_plan's first two workspace blocks, which it carves with take() (256-byte aligned):
    x2, the conv2 output [N][Tp][16] fp16 with Tp = T_in + 2 (winlen3 // 2) + 8, then the sequence buffer
    [T_out + 1][N][C] fp16 that conv3 writes and every LSTM layer overwrites in place."""
    pad = cfg.convs[2].winlen // 2
    Tp = T_in + 2 * pad + 8
    x2_bytes = N * Tp * 16 * 2
    return {"pad": pad, "Tp": Tp, "x2": 0, "x2_bytes": x2_bytes, "seq": (x2_bytes + 255) & ~255,
            "T_out": T_in // cfg.stride}


def read_x2(runner, cfg, N, T_in):
    """conv2's output [N][Tp][16] (fp32 copy of the fp16 buffer)."""
    lay = workspace_layout(cfg, N, T_in)
    raw = runner.debug_read_workspace(lay["x2"], lay["x2_bytes"])
    return raw.view(np.float16).reshape(N, lay["Tp"], 16).astype(np.float32)


def read_seq(runner, cfg, N, T_in):
    """The sequence buffer's first T_out rows [T_out][N][C] as fp16."""
    lay = workspace_layout(cfg, N, T_in)
    C = cfg.lstm_size
    raw = runner.debug_read_workspace(lay["seq"], lay["T_out"] * N * C * 2)
    return raw.view(np.float16).reshape(lay["T_out"], N, C).copy()


# ---- weights -----------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class LayerWeights:
    w_ih: np.ndarray   # [4C][C] float64 holding fp16 values, gate order i | f | g | o
    w_hh: np.ndarray   # [4C][C]
    bias: np.ndarray   # [4C] float64 holding the fp32 sum b_ih + b_hh


def layer_weights(cfg, w, l):
    p = f"{len(cfg.convs) + l + 1}.rnn."
    return make_layer_weights(w[p + "weight_ih_l0.tensor"], w[p + "weight_hh_l0.tensor"], w[p + "bias_ih_l0.tensor"],
                              w[p + "bias_hh_l0.tensor"])


def make_layer_weights(w_ih, w_hh, b_ih, b_hh):
    b = (np.asarray(b_ih, np.float32) + np.asarray(b_hh, np.float32)).astype(np.float64)
    return LayerWeights(q16(w_ih), q16(w_hh), b)


# ---- the reference -----------------------------------------------------------------------------------------------------
def step_times(T, N, reverse, steps=None):
    """t of step s of every chunk, [T][N]; -1 where s >= steps_n (the chunk has ended)."""
    st = np.full(N, T) if steps is None else np.minimum(np.asarray(steps), T)
    s = np.arange(T)[:, None]
    t = st[None, :] - 1 - s if reverse else np.broadcast_to(s, (T, N))
    return np.where(s < st[None, :], t, -1)


def _gather(A, tidx):
    return np.asarray(A)[np.maximum(tidx, 0), np.arange(tidx.shape[1])[None, :]].astype(np.float64)


def reference_layer(X, lw, reverse, steps=None, H=None, eps=EPS_TANH, block=64):
    """One layer over X [T][N][C], in step order.  With H, teacher-forced on H; without, run free on its own fp16-rounded
    h.  Returns (h [T][N][C] before rounding, dh [T][N][C] its first-order error budget, tidx [T][N]), all in step order."""
    T, N, C = X.shape
    tidx = step_times(T, N, reverse, steps)
    Xs = _gather(X, tidx)
    if H is not None:
        Hs = _gather(H, tidx)
        Hprev = np.concatenate([np.zeros((1, N, C)), Hs[:-1]])
    gamma = (C + 2) * U32   # C products, the bias and the final add of W_hh h + gx in fp32
    w_ihT, w_hhT = lw.w_ih.T, lw.w_hh.T
    a_ihT, a_hhT = np.abs(w_ihT).astype(np.float32), np.abs(w_hhT).astype(np.float32)
    c = np.zeros((N, C))
    dc = np.zeros((N, C))
    hq = np.zeros((N, C))
    h_out = np.empty((T, N, C))
    dh_out = np.empty((T, N, C))
    for s0 in range(0, T, block):
        xs = Xs[s0:s0 + block]
        gx = q16(xs @ w_ihT + lw.bias)
        dgx = ulp16(gx) + gamma * (np.abs(xs).astype(np.float32) @ a_ihT + np.abs(lw.bias))
        if H is not None:
            hp = Hprev[s0:s0 + block]
            rec = hp @ w_hhT
            drec = gamma * (np.abs(hp).astype(np.float32) @ a_hhT)
        for j in range(xs.shape[0]):
            if H is not None:
                pre, dpre = gx[j] + rec[j], dgx[j] + drec[j]
            else:
                pre = gx[j] + hq @ w_hhT
                dpre = dgx[j] + gamma * (np.abs(hq) @ a_hhT)
            pi, pf, pg, po = (pre[:, k * C:(k + 1) * C] for k in range(4))
            di, df, dg, do = (dpre[:, k * C:(k + 1) * C] for k in range(4))
            ti, tf, to = np.tanh(0.5 * pi), np.tanh(0.5 * pf), np.tanh(0.5 * po)
            i, f, o = 0.5 * ti + 0.5, 0.5 * tf + 0.5, 0.5 * to + 0.5
            g = np.tanh(pg)
            # activated gates: MUFU error + the largest slope within the pre-activation's error x that error (+ the
            # final fma's rounding)
            e_i = 0.5 * eps * np.abs(ti) + _sig_slope(i * (1 - i), di) * di + U32
            e_f = 0.5 * eps * np.abs(tf) + _sig_slope(f * (1 - f), df) * df + U32
            e_o = 0.5 * eps * np.abs(to) + _sig_slope(o * (1 - o), do) * do + U32
            e_g = eps * np.abs(g) + _tanh_slope(1 - g * g, dg) * dg
            # products of two inexact factors: |a' b' - a b| <= e_a (|b| + e_b) + |a| e_b
            c_new = f * c + i * g
            dc = (e_f * (np.abs(c) + dc) + f * dc + e_i * (np.abs(g) + e_g) + np.abs(i) * e_g
                  + U32 * (np.abs(f * c) + np.abs(c_new)))
            c = c_new
            tc = np.tanh(c)
            e_tc = eps * np.abs(tc) + _tanh_slope(1 - tc * tc, dc) * dc
            h = o * tc
            h_out[s0 + j] = h
            dh_out[s0 + j] = e_o * (np.abs(tc) + e_tc) + o * e_tc + U32 * np.abs(h)
            hq = q16(h)
    return h_out, dh_out, tidx


def free_run(X, lw, reverse, steps=None):
    """The float64 reference fed back its own fp16 h: [T][N][C] fp16 values in time order (zero beyond a chunk's end)."""
    h, _, tidx = reference_layer(X, lw, reverse, steps)
    out = np.zeros(X.shape)
    s, n = np.nonzero(tidx >= 0)
    out[tidx[s, n], n] = q16(h[s, n])
    return out


@dataclasses.dataclass
class LayerCheck:
    """|H - h_ref| / (ulp16(h_ref) + kappa dh) of every compared element, in step order (0 where not compared)."""
    ratio: np.ndarray
    tidx: np.ndarray
    got: np.ndarray
    want: np.ndarray
    bound: np.ndarray
    label: str = ""

    @property
    def valid(self):
        return self.tidx >= 0

    @property
    def max_ratio(self):
        return float(self.ratio.max())

    @property
    def median_ratio(self):
        return float(np.median(self.ratio[self.valid]))

    @property
    def ok(self):
        return self.max_ratio <= 1.0

    def worst(self):
        s, n, u = np.unravel_index(int(np.argmax(self.ratio)), self.ratio.shape)
        return int(s), int(self.tidx[s, n]), int(n), int(u)

    def describe(self):
        s, t, n, u = self.worst()
        msg = (f"{self.label}: max ratio {self.max_ratio:.3g} at step {s} (t {t}, chunk {n}, unit {u}): got "
               f"{self.got[s, n, u]:.6g}, want {self.want[s, n, u]:.6g}, bound {self.bound[s, n, u]:.3g}; "
               f"median ratio {self.median_ratio:.3g}")
        bad = self.ratio > 1.0
        if bad.any():
            bs, bn, bu = np.nonzero(bad)
            msg += (f"; {int(bad.sum())} elements over the bound, in chunks {np.unique(bn)[:24].tolist()}, steps "
                    f"{np.unique(bs)[:24].tolist()}, units {np.unique(bu)[:24].tolist()}")
        return msg


def check_layer(X, H, lw, reverse, steps=None, kappa=KAPPA, eps=EPS_TANH, label=""):
    """Hold the engine's output H of one layer to the teacher-forced reference on its input X."""
    h, dh, tidx = reference_layer(X, lw, reverse, steps, H=H, eps=eps)
    got = _gather(H, tidx)
    bound = ulp16(h) + kappa * dh
    ratio = np.where((tidx >= 0)[..., None], np.abs(got - h) / bound, 0.0)
    return LayerCheck(ratio, tidx, got, h, bound, label)
