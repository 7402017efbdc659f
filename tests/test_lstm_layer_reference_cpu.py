"""The float64 LSTM layer reference of tests/lstm_layer_ref.py and its error budget, without a GPU.

- Run free (on its own fp16 h), the reference is nn_oracle's lstm_layer with fp16 storage, to fp32 noise.
- The budget covers a simulated kernel: fp32 arithmetic, every activation off by up to the MUFU error (a fixed-sign
  bias and at random), gx and h rounded to fp16, its recurrent input its own fp16 h -- in every weight regime the GPU
  tests use.
- The same check rejects, by a wide margin, the kernel bugs the GPU tests are meant to catch: two chunks swapped, one
  step left stale, the direction flipped, one gate bias dropped, the cell state reset once, the last row left holding the
  layer input.
- The bound has teeth: in the nominal regime it is a few fp16 ulps of h, and the controls exceed it many times over.
"""
import numpy as np
import pytest

from lstm_layer_ref import EPS_TANH, check_layer, free_run, make_layer_weights, reference_layer, step_times, ulp16

REGIMES = ["nominal", "long_memory", "saturating"]


def _weights(C, regime, seed=7):
    """The fan-in uniform LSTM weights of dorado_b200.weights.synthetic_weights (W_ih gain 6, W_hh gain 1.5, b_ih in
    +-0.1, b_hh 0), edited like the GPU tests' weight regimes."""
    rng = np.random.default_rng(seed)
    bound = 1.0 / np.sqrt(C)
    w_ih = (6.0 * bound * rng.uniform(-1, 1, (4 * C, C))).astype(np.float32)
    w_hh = (1.5 * bound * rng.uniform(-1, 1, (4 * C, C))).astype(np.float32)
    b_ih = (0.1 * rng.uniform(-1, 1, 4 * C)).astype(np.float32)
    b_hh = np.zeros(4 * C, np.float32)
    if regime == "long_memory":
        b_ih[C:2 * C] += 3.0
    elif regime == "saturating":
        w_ih *= 3.0
    return w_ih, w_hh, b_ih, b_hh


def _inputs(T, N, C, seed=3):
    """A conv3-like layer input: tanh of a smooth random signal, different in every chunk, fp16."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((T, N, C)) + 0.5 * np.roll(rng.standard_normal((T, N, C)), 1, axis=0)
    return np.tanh(z).astype(np.float16)


def simulated_kernel(X, w_ih, w_hh, b_ih, b_hh, reverse, steps=None, act_err="random", seed=0, reset_at=None):
    """What the kernels compute, in fp32: gx = fp16(W_ih x + b), pre = W_hh h + gx, gates on a tanh with a relative error
    of EPS_TANH (act_err: "high" / "low" = fixed sign, "random" = uniform in +-EPS_TANH), fp32 cell state, h stored as fp16
    and fed back.  reset_at: the step at which the cell state is (wrongly) zeroed.  [T][N][C] fp16 in time order."""
    T, N, C = X.shape
    rng = np.random.default_rng(seed)
    w_ih16, w_hh16 = w_ih.astype(np.float16).astype(np.float32), w_hh.astype(np.float16).astype(np.float32)
    b = (b_ih.astype(np.float32) + b_hh.astype(np.float32)).astype(np.float32)
    eps = np.float32(EPS_TANH)

    def tanh_k(v):
        if act_err == "high":
            r = np.float32(1) + eps
        elif act_err == "low":
            r = np.float32(1) - eps
        else:
            r = np.float32(1) + eps * rng.uniform(-1, 1, v.shape).astype(np.float32)
        return (np.tanh(v) * r).astype(np.float32)

    sig = lambda v: np.float32(0.5) * tanh_k(np.float32(0.5) * v) + np.float32(0.5)
    tidx = step_times(T, N, reverse, steps)
    out = np.zeros((T, N, C), np.float16)
    h = np.zeros((N, C), np.float32)
    c = np.zeros((N, C), np.float32)
    nn = np.arange(N)
    for s in range(T):
        alive = tidx[s] >= 0
        x = X[np.maximum(tidx[s], 0), nn].astype(np.float32)
        gx = (x @ w_ih16.T + b).astype(np.float16).astype(np.float32)
        pre = h @ w_hh16.T + gx
        i, f, g, o = sig(pre[:, :C]), sig(pre[:, C:2 * C]), tanh_k(pre[:, 2 * C:3 * C]), sig(pre[:, 3 * C:])
        if reset_at == s:
            c[:] = 0
        c = np.where(alive[:, None], f * c + i * g, 0).astype(np.float32)
        h = np.where(alive[:, None], o * tanh_k(c), 0).astype(np.float16).astype(np.float32)
        out[tidx[s, alive], nn[alive]] = h[alive]
    return out


@pytest.mark.parametrize("C", [96, 192])
@pytest.mark.parametrize("reverse", [True, False])
def test_reference_matches_nn_oracle(C, reverse):
    """Free-running, the reference and nn_oracle's fp32 lstm_layer (fp16 storage) differ only where fp32 and float64 round
    a gx or an h to different fp16 values (measured: 97-99 % of the outputs identical, the rest one fp16 ulp of h apart).
    Teacher-forced on the oracle's own output, the reference's h rounds to the oracle's h (within half an ulp plus fp32
    noise) almost everywhere."""
    from oracle import nn_oracle
    T, N = 60, 8
    X = _inputs(T, N, C)
    w_ih, w_hh, b_ih, b_hh = _weights(C, "nominal")
    lw = make_layer_weights(w_ih, w_hh, b_ih, b_hh)
    q = lambda a: a.astype(np.float16).astype(np.float32)
    orc = nn_oracle.lstm_layer(X.astype(np.float32).transpose(1, 0, 2), q(w_ih), q(w_hh), b_ih, b_hh, reverse, quant=q)
    orc = orc.transpose(1, 0, 2).astype(np.float64)
    diff = np.abs(free_run(X, lw, reverse) - orc)
    assert (diff == 0).mean() >= 0.96, (diff == 0).mean()
    assert (diff <= ulp16(np.maximum(np.abs(orc), 0.25))).mean() >= 0.999 and diff.max() <= 1e-3, float(diff.max())
    h, _, tidx = reference_layer(X, lw, reverse, H=orc.astype(np.float16))
    got = orc[np.maximum(tidx, 0), np.arange(N)[None, :]]
    err = np.abs(got - h)
    assert (err <= 0.5 * ulp16(h) * (1 + 1e-3) + 1e-7).mean() >= 0.995
    assert err.max() <= 1e-3, float(err.max())


def _sim_and_check(C, regime, reverse, act_err, steps=None, T=200, N=16, **kw):
    X = _inputs(T, N, C, seed=C)
    w = _weights(C, regime)
    H = simulated_kernel(X, *w, reverse=reverse, steps=steps, act_err=act_err, **kw)
    return X, w, H, check_layer(X, H, make_layer_weights(*w), reverse, steps)


@pytest.mark.parametrize("C", [96, 192])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("act_err", ["random", "high", "low"])
def test_budget_covers_a_simulated_kernel(C, regime, act_err):
    for reverse in (True, False):
        *_, res = _sim_and_check(C, regime, reverse, act_err)
        print(f"\n[C {C} {regime} {act_err} reverse {reverse}] max ratio {res.max_ratio:.3f} median {res.median_ratio:.3f}")
        assert res.ok, res.describe()


def test_budget_covers_variable_chunk_lengths():
    """Chunks of 1, 2, 9 and T steps, and a whole half of the batch short: a reversed layer starts each chunk at its own
    last step."""
    T, N = 60, 16
    steps = np.full(N, T)
    steps[:4] = [1, 2, 9, T - 1]
    steps[8:] = np.arange(8) + 20
    for reverse in (True, False):
        X, w, H, res = _sim_and_check(96, "nominal", reverse, "random", steps=steps, T=T, N=N)
        assert res.ok, res.describe()
        # the same output held to fixed-length steps is wrong for a reversed layer (it starts at t = T - 1)
        if reverse:
            assert not check_layer(X, H, make_layer_weights(*w), reverse).ok


def test_bound_has_teeth():
    """In the nominal regime the bound stays within a few fp16 ulps of the values that carry the signal (ulps of
    max(|h|, 1/4)): median 3.6, 99th percentile 13.4 on this data.  Most of it is one fp16 ulp of gx through the gate
    slopes and the MUFU error of four activations."""
    X, w, H, res = _sim_and_check(96, "nominal", True, "random")
    h = res.want[res.valid]
    ulps = res.bound[res.valid] / ulp16(np.maximum(np.abs(h), 0.25))
    p50, p99 = float(np.median(ulps)), float(np.percentile(ulps, 99))
    print(f"\n[bound in fp16 ulps of max(|h|, 1/4)] median {p50:.2f}, p99 {p99:.2f}, max {ulps.max():.2f}")
    assert p50 <= 5.0 and p99 <= 16.0


MARGIN = 5.0   # a negative control must exceed the bound at least this many times


def _mutations(X, w, H, reverse, T):
    steps_t = step_times(T, X.shape[1], reverse)[:, 0]     # t of step s
    out = {}
    m = H.copy()
    m[:, [7, 8]] = m[:, [8, 7]]
    out["chunks 7 and 8 swapped"] = m
    for s in (0, 8, T - 1):
        m = H.copy()
        m[steps_t[s]] = H[steps_t[s - 1]] if s > 0 else 0
        out[f"step {s} stale"] = m
    out["direction flipped"] = simulated_kernel(X, *w, reverse=not reverse)
    m = H.copy()
    m[steps_t[-1]] = X[steps_t[-1]]
    out["last row holds the layer input"] = m
    out["cell state reset at step 100"] = simulated_kernel(X, *w, reverse=reverse, reset_at=100)
    return out


@pytest.mark.parametrize("reverse", [True, False])
def test_negative_controls_are_rejected(reverse):
    T = 200
    X, w, H, res = _sim_and_check(96, "nominal", reverse, "random", T=T)
    assert res.ok
    lw = make_layer_weights(*w)
    for name, m in _mutations(X, w, H, reverse, T).items():
        bad = check_layer(X, m, lw, reverse, label=name)
        print(f"\n[{name}] max ratio {bad.max_ratio:.1f}")
        assert bad.max_ratio >= MARGIN, bad.describe()


@pytest.mark.parametrize("gate", range(4))
def test_dropped_gate_bias_is_rejected(gate):
    C, T = 96, 200
    X = _inputs(T, 16, C, seed=C)
    w_ih, w_hh, b_ih, b_hh = _weights(C, "nominal")
    u = int(np.argmax(np.abs(b_ih[gate * C:(gate + 1) * C])))
    dropped = b_ih.copy()
    dropped[gate * C + u] = 0
    H = simulated_kernel(X, w_ih, w_hh, dropped, b_hh, reverse=True)
    bad = check_layer(X, H, make_layer_weights(w_ih, w_hh, b_ih, b_hh), True, label=f"gate {gate} unit {u} bias dropped")
    print(f"\n[{bad.label}] max ratio {bad.max_ratio:.1f}")
    assert bad.max_ratio >= MARGIN, bad.describe()
    assert bad.worst()[3] == u
