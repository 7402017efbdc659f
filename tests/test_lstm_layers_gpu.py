"""Every LSTM layer kernel, layer by layer, against the teacher-forced float64 reference of tests/lstm_layer_ref.py.

B200_DEBUG_LSTM_LAYERS=k (read when a runner is built) stops the forward after k LSTM layers; the sequence buffer then
holds the output of layer k - 1, which is the input of layer k.  Each case builds one runner per k from one B200Caller
per weight set, so layer l is checked on its own: X = buffer after l layers, H = buffer after l + 1 layers, every
element within ulp16(h_ref) + KAPPA dh of the reference.  The buffer after 0 layers is conv3's output, held to
nn_oracle's conv stack, which pins the workspace layout the reads rely on.

Kernels and launch shapes:
  96          lstm_layer_kernel: T_out 1, 2, 6, 7, 8, 9, 17 (shorter than the cp.async ring, around its wrap); 500 steps in
              three weight regimes; 2128 chunks = 133 CTAs, more than the H100's 132 SMs
  192, 384    lstm_rec_kernel<C, 4 / 8, 16 / 32 / 64>: every chunks-per-cluster shape, fixed and variable chunk lengths
  768, 1024   lstm_grid_rec_kernel<C, 32 / 64>: one group per launch, so a batch of 64 chunks takes 2 or 1 launches
Weight regimes: nominal (synthetic_weights), long memory (forget-gate biases + 3: f ~ 0.95, the cell state carries
the signal for ~20 steps) and saturating (W_ih x 3).  W_hh keeps its gain, so the recurrence stays contractive.
In one case per kernel the same output must fail against the reference run in the wrong direction: the bound is tight
enough to see a real error.

Measured on one H100 80GB HBM3 at a 700 W power limit, the worst |error| / budget of any element and the median of the
per-layer median ratios were: 96 0.40 / 0.031 (55 layers), 192 0.37 / 0.027 (20), 384 0.31 / 0.023 (35), 768 0.24 / 0.014
(6 distinct), 1024 0.25 / 0.010 (6 distinct); the long-memory and saturating layers stayed at or below 0.39.  A simulated
kernel whose every activation is off by the full MUFU error reaches 0.67 (tests/test_lstm_layer_reference_cpu.py).  The
file runs in about 5 minutes, most of it the float64 reference on the host.
"""
import hashlib

import numpy as np
import pytest

from conftest import model_dir
from lstm_layer_ref import check_layer, layer_weights, read_seq, workspace_layout
from test_wide_lstm_cpu import model_dir as wide_model_dir

pytestmark = pytest.mark.gpu

_callers = {}
_memo = {}
_stats = {}   # kernel -> [(max ratio, median ratio)]


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    print("\n[LSTM layers vs float64 reference] error / budget per kernel:")
    for kernel, rows in _stats.items():
        mx = max(r[0] for r in rows)
        med = float(np.median([r[1] for r in rows]))
        print(f"  {kernel:28s} {len(rows):3d} layers checked, worst ratio {mx:.3f}, median of per-layer medians {med:.3f}")
    for c in _callers.values():
        c.close()
    _callers.clear()


def _cfg(kind, tmp_path_factory=None):
    from dorado_b200.config import load_model_config
    if kind in ("lstm768", "lstm1024"):
        return load_model_config(wide_model_dir(kind))
    if kind == "lstm192":
        # the hac topology at lstm_size 192 (conv3 16 -> 192, five LSTM layers of 192)
        d = tmp_path_factory.mktemp("lstm192")
        (d / "config.toml").write_text((model_dir("hac") / "config.toml").read_text().replace("384", "192"))
        cfg = load_model_config(d)
        assert cfg.lstm_size == 192 and cfg.convs[2].size == 192
        return cfg
    return load_model_config(model_dir(kind))


def _regime(cfg, w, regime):
    """A copy of the weights, edited: long memory = forget-gate rows of bias_ih + 3; saturating = W_ih x 3."""
    if regime == "nominal":
        return w
    w = dict(w)
    C = cfg.lstm_size
    for l in range(cfg.lstm_layers):
        p = f"{len(cfg.convs) + l + 1}.rnn."
        if regime == "long_memory":
            b = w[p + "bias_ih_l0.tensor"].copy()
            b[C:2 * C] += 3.0
            w[p + "bias_ih_l0.tensor"] = b
        elif regime == "saturating":
            w[p + "weight_ih_l0.tensor"] = w[p + "weight_ih_l0.tensor"] * np.float32(3.0)
        else:
            raise ValueError(regime)
    return w


def _caller(kind, cfg, regime="nominal"):
    from dorado_b200.runner import B200Caller
    from dorado_b200.weights import synthetic_weights
    key = (kind, regime)
    if key not in _callers:
        w = _regime(cfg, synthetic_weights(cfg, 42), regime)
        _callers[key] = B200Caller(cfg, w)
        _callers[key].weights = w
    return _callers[key]


def _signals(cfg, N, T_in, seed, lens=None):
    """A different random signal in every chunk (a chunk-mapping error cannot cancel out); with lens, chunk i has lens[i]
    samples."""
    rng = np.random.default_rng(seed)
    sig = rng.standard_normal((N, T_in)).astype(np.float16) * np.linspace(0.6, 1.4, N, dtype=np.float16)[:, None]
    if lens is None:
        return sig
    return [sig[i, :int(lens[i])].copy() for i in range(N)]


def _snapshots(monkeypatch, caller, cfg, N, T_in, sig, layers, info_key=None):
    """The sequence buffer after k = 0 .. layers LSTM layers ([T_out][N][C] fp16 each), one runner per k."""
    from dorado_b200.runner import B200ModelRunner
    out = []
    info = None
    for k in range(layers + 1):
        monkeypatch.setenv("B200_DEBUG_LSTM_LAYERS", str(k))
        runner = B200ModelRunner(caller, N, T_in)
        assert runner.chunk_size() == T_in
        for i in range(N):
            if isinstance(sig, list):
                runner.accept_chunk_var(i, sig[i])
            else:
                runner.accept_chunk(i, sig[i])
        runner.forward_scores(N)
        out.append(read_seq(runner, cfg, N, T_in))
        info = runner.plan_info()
        runner.close()
    monkeypatch.delenv("B200_DEBUG_LSTM_LAYERS")
    return out, info


def _check_conv_stack(cfg, w, sig, seq0):
    """The buffer after 0 layers is conv3's output: nn_oracle's conv stack with the engine's fp16 storage points."""
    from oracle import nn_oracle
    _, inter = nn_oracle.forward(cfg, w, sig.astype(np.float32), return_intermediates=True, emulate_fp16=True)
    ref = inter[f"conv{len(cfg.convs) - 1}"].transpose(2, 0, 1)   # [N][C][T] -> [T][N][C]
    err = np.abs(seq0.astype(np.float32) - ref)
    scale = max(1.0, float(np.abs(ref).max()))
    assert err.max() <= 2e-3 * scale, f"conv3 output vs oracle: max err {err.max():.2e} (scale {scale:.2f})"


def _digest(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def _check_layers(kernel, cfg, w, wkey, snaps, layers, steps=None, label="", sensitivity=False):
    """Layer l of `layers` against the reference; each result is kept once per distinct (weights, X, H, lengths)."""
    for l in layers:
        X, H = snaps[l], snaps[l + 1]
        reverse = l % 2 == 0   # reverse_first
        key = (wkey, l, _digest(X), _digest(H), None if steps is None else _digest(steps))
        lw = layer_weights(cfg, w, l)
        if key not in _memo:
            _memo[key] = check_layer(X, H, lw, reverse, steps, label=f"{kernel} {label} layer {l}")
            _stats.setdefault(kernel, []).append((_memo[key].max_ratio, _memo[key].median_ratio))
        res = _memo[key]
        print(f"\n  {res.label}: max ratio {res.max_ratio:.3f}, median {res.median_ratio:.3f}")
        assert res.ok, res.describe()
        if sensitivity and l == layers[0]:
            wrong = check_layer(X, H, lw, not reverse, steps)
            assert wrong.max_ratio >= 10.0, f"the reference run in the wrong direction passes: {wrong.describe()}"


# ---- lstm_size 96: lstm_layer_kernel ------------------------------------------------------------------------------------
@pytest.mark.parametrize("T_out", [1, 2, 6, 7, 8, 9, 17])
def test_fused_layer_short_chunks(monkeypatch, T_out):
    """Fewer steps than the 8-slot x ring (the prologue waits on steps 0 and 1, the loop has no tail), around its wrap."""
    cfg = _cfg("fast")
    caller = _caller("fast", cfg)
    N, T_in = 16, T_out * cfg.stride
    sig = _signals(cfg, N, T_in, seed=100 + T_out)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, cfg.lstm_layers)
    assert info["lstm_layer.ctas"] == 1
    _check_conv_stack(cfg, caller.weights, sig, snaps[0])
    _check_layers("96 lstm_layer_kernel", cfg, caller.weights, "fast", snaps, range(cfg.lstm_layers), label=f"T_out {T_out}",
                  sensitivity=T_out == 17)


@pytest.mark.parametrize("regime", ["nominal", "long_memory", "saturating"])
def test_fused_layer_weight_regimes(monkeypatch, regime):
    cfg = _cfg("fast")
    caller = _caller("fast", cfg, regime)
    N, T_in = 48, 500 * cfg.stride
    sig = _signals(cfg, N, T_in, seed=7)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, cfg.lstm_layers)
    assert info["lstm_layer.ctas"] == 3
    _check_layers("96 lstm_layer_kernel", cfg, caller.weights, ("fast", regime), snaps, range(cfg.lstm_layers),
                  label=regime, sensitivity=regime == "nominal")


def test_fused_layer_more_ctas_than_sms(monkeypatch):
    cfg = _cfg("fast")
    caller = _caller("fast", cfg)
    N, T_in = 2128, 20 * cfg.stride
    sig = _signals(cfg, N, T_in, seed=8)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, cfg.lstm_layers)
    assert info["lstm_layer.ctas"] == 133
    _check_conv_stack(cfg, caller.weights, sig, snaps[0])
    _check_layers("96 lstm_layer_kernel", cfg, caller.weights, "fast", snaps, range(cfg.lstm_layers), label="133 CTAs")


# ---- lstm_size 192 and 384: lstm_rec_kernel -----------------------------------------------------------------------------
def _variable_lengths(cfg, N, T_in, un, seed):
    """Chunk lengths in samples: one step, full length, random, and a whole cluster of short chunks (the last `un`
    chunks), so that a cluster runs fewer steps than T_out and its reversed layers start below T_out - 1."""
    rng = np.random.default_rng(seed)
    T_out = T_in // cfg.stride
    steps = rng.integers(1, T_out + 1, size=N)
    steps[0], steps[1], steps[2], steps[3] = 1, T_out, 2, T_out - 1
    steps[N - un:] = rng.integers(1, T_out // 2, size=un)
    return steps * cfg.stride, steps


@pytest.mark.parametrize("un", [16, 32, 64])
def test_rec_kernel_192(monkeypatch, tmp_path_factory, un):
    cfg = _cfg("lstm192", tmp_path_factory)
    caller = _caller("lstm192", cfg)
    monkeypatch.setenv("B200_CLUSTER_CHUNKS", str(un))
    N, T_in = 128, 1200
    sig = _signals(cfg, N, T_in, seed=11)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, cfg.lstm_layers)
    assert info["lstm_rec.chunks_per_cluster"] == un and info["lstm_rec.ctas"] == N // un * 4
    _check_conv_stack(cfg, caller.weights, sig, snaps[0])
    _check_layers("192 lstm_rec_kernel", cfg, caller.weights, "lstm192", snaps, range(cfg.lstm_layers),
                  label=f"{un} chunks", sensitivity=un == 16)
    lens, steps = _variable_lengths(cfg, N, T_in, un, seed=12)
    snaps, _ = _snapshots(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, 13, lens), cfg.lstm_layers)
    _check_layers("192 lstm_rec_kernel", cfg, caller.weights, "lstm192", snaps, range(cfg.lstm_layers), steps=steps,
                  label=f"{un} chunks, variable lengths")


@pytest.mark.parametrize("un", [16, 32, 64])
@pytest.mark.parametrize("T_out", [1, 9, 200])
def test_rec_kernel_384(monkeypatch, un, T_out):
    cfg = _cfg("hac")
    caller = _caller("hac", cfg)
    monkeypatch.setenv("B200_CLUSTER_CHUNKS", str(un))
    N, T_in = 128, T_out * cfg.stride
    sig = _signals(cfg, N, T_in, seed=21)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, cfg.lstm_layers)
    assert info["lstm_rec.chunks_per_cluster"] == un and info["lstm_rec.ctas"] == N // un * 8
    if T_out == 200:
        _check_conv_stack(cfg, caller.weights, sig, snaps[0])
    _check_layers("384 lstm_rec_kernel", cfg, caller.weights, "hac", snaps, range(cfg.lstm_layers),
                  label=f"{un} chunks, T_out {T_out}", sensitivity=un == 16 and T_out == 200)
    if T_out == 200:
        lens, steps = _variable_lengths(cfg, N, T_in, un, seed=22)
        snaps, _ = _snapshots(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, 23, lens), cfg.lstm_layers)
        _check_layers("384 lstm_rec_kernel", cfg, caller.weights, "hac", snaps, range(cfg.lstm_layers), steps=steps,
                      label=f"{un} chunks, variable lengths")


def test_rec_kernel_384_long_memory(monkeypatch):
    cfg = _cfg("hac")
    caller = _caller("hac", cfg, "long_memory")
    monkeypatch.setenv("B200_CLUSTER_CHUNKS", "32")
    N, T_in = 128, 1200
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, seed=31), cfg.lstm_layers)
    assert info["lstm_rec.chunks_per_cluster"] == 32
    _check_layers("384 lstm_rec_kernel", cfg, caller.weights, ("hac", "long_memory"), snaps, range(cfg.lstm_layers),
                  label="32 chunks, long memory")


# ---- lstm_size 768 and 1024: lstm_grid_rec_kernel -----------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lstm768", "lstm1024"])
@pytest.mark.parametrize("nb", [32, 64])
def test_grid_rec_kernel(monkeypatch, kind, nb):
    """Layers 0 (reversed) and 1 (forward); one group per launch, so 64 chunks take 64 / nb launches per layer."""
    cfg = _cfg(kind)
    caller = _caller(kind, cfg)
    monkeypatch.setenv("B200_GRID_CHUNKS", str(nb))
    monkeypatch.setenv("B200_GRID_GROUPS", "1")
    N, T_in = 64, 600
    sig = _signals(cfg, N, T_in, seed=41)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, 2)
    assert (info["lstm_grid.chunks_per_group"], info["lstm_grid.groups"], info["lstm_grid.launches_per_layer"]) == (nb, 1, N // nb)
    _check_conv_stack(cfg, caller.weights, sig, snaps[0])
    _check_layers(f"{cfg.lstm_size} lstm_grid_rec_kernel", cfg, caller.weights, kind, snaps, range(2),
                  label=f"{nb} chunks per group", sensitivity=nb == 32)
    lens, steps = _variable_lengths(cfg, N, T_in, nb, seed=42)
    snaps, _ = _snapshots(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, 43, lens), 2)
    _check_layers(f"{cfg.lstm_size} lstm_grid_rec_kernel", cfg, caller.weights, kind, snaps, range(2), steps=steps,
                  label=f"{nb} chunks per group, variable lengths")


def test_workspace_layout_matches_the_plan():
    """The offsets the reads above use: x2 at 0, the sequence buffer after it, 256-byte aligned."""
    cfg = _cfg("fast")
    lay = workspace_layout(cfg, 16, 1200)
    assert lay["Tp"] == 1200 + 2 * 9 + 8 and lay["seq"] == (16 * lay["Tp"] * 16 * 2 + 255) // 256 * 256
