"""lstm_size 128 and 256 on the GPU: x-projection GEMM + lstm_rec_kernel<C, 4 | 8, NB>.  Scores are held to the numpy
oracle with the bounds of tests/test_forward_gpu.py, calls to the C oracle decoding the engine's own scores, every LSTM
layer to the teacher-forced float64 reference of tests/lstm_layer_ref.py; the result must not depend on the launch shape.

The 128 fixture has state_len 3, so its calls go through crf_decode_warp_kernel; its variable-chunk-size test runs that
kernel with per-chunk lengths, which the fast model (lstm_size 96, fixed-size chunks only) never does."""
import os

import numpy as np
import pytest

from lstm_layer_ref import check_layer, layer_weights, make_layer_weights
from test_forward_gpu import _check_scores
from test_lstm128_256_cpu import WIDTHS, lstm_rec_chunks, model_dir, rec_cluster
from test_lstm_layers_gpu import _regime, _signals, _snapshots, _variable_lengths, _check_conv_stack
from test_modbase_cpu import modbase_dir, modbase_inputs
from test_modbase_gpu import PROB_MAX, PROB_MEAN, PROB_P999, _resize

pytestmark = pytest.mark.gpu

KINDS = ["lstm128", "lstm256"]
_weights = {}
_callers = {}
_stats = {}   # kernel -> [(max ratio, median ratio)]


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    print("\n[lstm_size 128 / 256 LSTM layers vs float64 reference] error / budget:")
    for kernel, rows in _stats.items():
        print(f"  {kernel:28s} {len(rows):3d} layers checked, worst ratio {max(r[0] for r in rows):.3f}, "
              f"median of per-layer medians {float(np.median([r[1] for r in rows])):.3f}")
    for c in _callers.values():
        c.close()
    _callers.clear()


def _cfg_w(kind):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    if kind not in _weights:
        cfg = load_model_config(model_dir(kind))
        _weights[kind] = (cfg, synthetic_weights(cfg, 42))
    return _weights[kind]


def _runner(kind, N, T, seed=1234, num_runners=2):
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _cfg_w(kind)
    caller = B200Caller(cfg, w, num_runners=num_runners)
    runner = B200ModelRunner(caller, N, T)
    sig = np.random.default_rng(seed).standard_normal((N, runner.chunk_size())).astype(np.float16)
    for i in range(N):
        runner.accept_chunk(i, sig[i])
    return cfg, w, caller, runner, sig


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N,T", [(32, 1200), (64, 1998), (512, 300)])
def test_scores(kind, N, T):
    from oracle import nn_oracle
    cfg, w, caller, runner, sig = _runner(kind, N, T)
    C = WIDTHS[kind]
    info = runner.plan_info()
    nb = lstm_rec_chunks(N)
    assert (info["lstm_rec.chunks_per_cluster"], info["lstm_rec.ctas"]) == (nb, N // nb * rec_cluster(C))
    got = runner.forward_scores(N)
    ref32 = nn_oracle.forward(cfg, w, sig.astype(np.float32))
    ref16 = nn_oracle.forward(cfg, w, sig.astype(np.float32), emulate_fp16=True)
    assert got.shape == ref32.shape == (N, runner.chunk_size() // cfg.stride, cfg.outsize)
    _check_scores(got, ref16, ref32, cfg.clamp)


@pytest.mark.parametrize("kind", KINDS)
def test_calls_match_the_decoder_oracle(crf_oracle, kind):
    cfg, w, caller, runner, sig = _runner(kind, 32, 1200)
    scores = runner.forward_scores(32)
    chunks = runner.call_chunks(32)
    ref = crf_oracle.decode(scores, clamp_val=5.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(chunks):
        assert c.sequence == ref.sequences[i] and c.qstring == ref.qstrings[i]
        np.testing.assert_array_equal(c.moves, ref.moves[i])
    assert sum(len(c.sequence) for c in chunks) > 32 * 10      # real calls, not empty strings


@pytest.mark.parametrize("kind", KINDS)
def test_variable_chunk_sizes(crf_oracle, kind):
    from oracle import nn_oracle
    from dorado_b200.runner import B200ModelRunner
    cfg, w, caller, runner, _ = _runner(kind, 64, 1200)
    assert runner.variable_chunk_sizes()
    T = runner.chunk_size()
    rng = np.random.default_rng(77)
    lens = rng.integers(20, T // cfg.stride + 1, size=64) * cfg.stride
    lens[0], lens[1], lens[2], lens[33] = T, cfg.stride * 20, cfg.stride, T
    sig = [rng.standard_normal(int(l)).astype(np.float16) for l in lens]
    for i in range(64):
        runner.accept_chunk_var(i, sig[i])
    scores = runner.forward_scores(64)
    called = runner.call_chunks(64)
    for i in range(64):
        tn = int(lens[i]) // cfg.stride
        assert len(called[i].moves) == tn
        ref = crf_oracle.decode(scores[i:i + 1, :tn], clamp_val=5.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
        assert called[i].sequence == ref.sequences[0] and called[i].qstring == ref.qstrings[0]
        assert (called[i].moves == ref.moves[0]).all()
        if i in (0, 1, 2, 5, 33, 63):   # numpy forward of the chunk alone, at its own length
            want = nn_oracle.forward(cfg, w, sig[i][None].astype(np.float32), emulate_fp16=True)[0]
            got = np.clip(scores[i, :tn].astype(np.float32), -5, 5)
            err = np.abs(got - want)
            scale = max(1.0, float(np.abs(want).max()))
            # one chunk's scores alone, so a looser fraction than _check_scores' 1e-3 over a batch: 1e-3 * scale (5e-3)
            # is under 1.3 fp16 ulps for scores in [4, 5]; measured on an H100, chunk 33 of the 128 model had 2.5e-3 of
            # its scores beyond it, max error 1.8e-3 * scale
            assert (err > 1e-3 * scale).mean() <= 5e-3 and err.max() <= 6e-3 * scale, (i, tn, float(err.max()))
    for i in (1, 2, 5):   # a fixed-shape runner of exactly that chunk size gives the same call
        alone = B200ModelRunner(caller, 32, int(lens[i]))
        alone.accept_chunk(0, sig[i])
        a = alone.call_chunks(1)[0]
        assert a.sequence == called[i].sequence and a.qstring == called[i].qstring and (a.moves == called[i].moves).all()
        alone.close()


@pytest.mark.parametrize("kind", KINDS)
def test_launch_shapes_agree(kind):
    """Chunks per cluster (16, 32, 64) and num_runners (1, 4) change only how the batch is cut into clusters and how
    many SMs the x-projection GEMM takes: scores and calls are bit-identical, for fixed and variable chunk sizes."""
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _cfg_w(kind)
    CL = rec_cluster(cfg.lstm_size)
    N, T = 128, 600
    rng = np.random.default_rng(3)
    sig = rng.standard_normal((N, cfg.normalise_chunk_size(T))).astype(np.float16)
    lens = rng.integers(1, sig.shape[1] // cfg.stride + 1, size=N) * cfg.stride
    lens[0] = cfg.stride
    shapes = [(None, 1), (None, 4), ("16", 1), ("32", 4), ("64", 1), ("64", 4)]
    got = {}
    try:
        for nb, R in shapes:
            if nb is None:
                os.environ.pop("B200_CLUSTER_CHUNKS", None)
            else:
                os.environ["B200_CLUSTER_CHUNKS"] = nb
            caller = B200Caller(cfg, w, num_runners=R)
            runner = B200ModelRunner(caller, N, T)
            info = runner.plan_info()
            want_nb = lstm_rec_chunks(N, None if nb is None else int(nb))
            assert (info["lstm_rec.chunks_per_cluster"], info["lstm_rec.ctas"]) == (want_nb, N // want_nb * CL)
            for i in range(N):
                runner.accept_chunk(i, sig[i])
            fixed = runner.forward_scores(N).copy()
            for i in range(N):
                runner.accept_chunk_var(i, sig[i, :lens[i]])
            got[(nb, R)] = (fixed, runner.forward_scores(N).copy(), [np.array(a) for a in runner.call_chunks_raw(N)])
            runner.close()
            caller.close()
    finally:
        os.environ.pop("B200_CLUSTER_CHUNKS", None)
    base = got[shapes[0]]
    for key in shapes[1:]:
        np.testing.assert_array_equal(got[key][0], base[0])
        for i in range(N):
            tn = int(lens[i]) // cfg.stride
            np.testing.assert_array_equal(got[key][1][i, :tn], base[1][i, :tn])
        (mv, sq, qs, nb_), (mv0, sq0, qs0, nb0) = got[key][2], base[2]
        np.testing.assert_array_equal(nb_, nb0)
        for i in range(N):
            tn = int(lens[i]) // cfg.stride
            assert (mv[i, :tn] == mv0[i, :tn]).all() and (sq[i, :nb_[i]] == sq0[i, :nb_[i]]).all()
            assert (qs[i, :nb_[i]] == qs0[i, :nb_[i]]).all()


def test_flstm_256_folds_like_the_plain_lstm(tmp_path):
    """A 256-wide FLSTM model and the plain LSTM model with the folded products up @ dn as weights give identical scores."""
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import fold_flstm_weights, synthetic_weights
    src = (model_dir("lstm256") / "config.toml").read_text()
    flstm = src.replace('type = "lstm"\n', 'type = "flstm"\ninner_dim = 64\n')
    assert flstm.count("inner_dim = 64") == 5
    (tmp_path / "flstm256").mkdir()
    (tmp_path / "flstm256" / "config.toml").write_text(flstm)
    cfg_f = load_model_config(tmp_path / "flstm256")
    cfg_l = load_model_config(model_dir("lstm256"))
    assert cfg_f.is_flstm_model and cfg_f.lstm_size == 256 and cfg_f.lstm_layers == 5
    w_f = synthetic_weights(cfg_f, 11)
    w_l = fold_flstm_weights(cfg_f, w_f)
    N, T = 32, 1200
    sig = np.random.default_rng(5).standard_normal((N, cfg_f.normalise_chunk_size(T))).astype(np.float16)
    out = []
    for cfg, w in ((cfg_f, w_f), (cfg_l, w_l)):
        runner = B200ModelRunner(B200Caller(cfg, w), N, T)
        assert runner.variable_chunk_sizes() == (cfg is cfg_l)     # FLSTM models never run variable chunk sizes
        for i in range(N):
            runner.accept_chunk(i, sig[i])
        out.append(runner.forward_scores(N).copy())
    np.testing.assert_array_equal(out[0], out[1])
    assert np.abs(out[0].astype(np.float32)).max() > 1.0


# ---- every layer against the float64 reference -----------------------------------------------------------------------
def _caller(kind, regime="nominal"):
    from dorado_b200.runner import B200Caller
    from dorado_b200.weights import synthetic_weights
    key = (kind, regime)
    if key not in _callers:
        cfg = _cfg_w(kind)[0]
        w = _regime(cfg, synthetic_weights(cfg, 42), regime)
        _callers[key] = B200Caller(cfg, w)
        _callers[key].weights = w
    return _callers[key]


def _check_layers(kernel, cfg, w, snaps, steps=None, label="", sensitivity=False):
    for l in range(cfg.lstm_layers):
        X, H = snaps[l], snaps[l + 1]
        reverse = l % 2 == 0   # reverse_first
        lw = layer_weights(cfg, w, l)
        res = check_layer(X, H, lw, reverse, steps, label=f"{kernel} {label} layer {l}")
        _stats.setdefault(kernel, []).append((res.max_ratio, res.median_ratio))
        print(f"\n  {res.label}: max ratio {res.max_ratio:.3f}, median {res.median_ratio:.3f}")
        assert res.ok, res.describe()
        if sensitivity and l == 0:
            wrong = check_layer(X, H, lw, not reverse, steps)
            assert wrong.max_ratio >= 10.0, f"the reference run in the wrong direction passes: {wrong.describe()}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("un", [16, 32, 64])
def test_rec_kernel_layers(monkeypatch, kind, un):
    cfg = _cfg_w(kind)[0]
    caller = _caller(kind)
    C = cfg.lstm_size
    kernel = f"{C} lstm_rec_kernel"
    monkeypatch.setenv("B200_CLUSTER_CHUNKS", str(un))
    N, T_in = 128, 1200
    sig = _signals(cfg, N, T_in, seed=51)
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, sig, cfg.lstm_layers)
    assert info["lstm_rec.chunks_per_cluster"] == un and info["lstm_rec.ctas"] == N // un * rec_cluster(C)
    _check_conv_stack(cfg, caller.weights, sig, snaps[0])
    _check_layers(kernel, cfg, caller.weights, snaps, label=f"{un} chunks", sensitivity=un == 16)
    lens, steps = _variable_lengths(cfg, N, T_in, un, seed=52)
    snaps, _ = _snapshots(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, 53, lens), cfg.lstm_layers)
    _check_layers(kernel, cfg, caller.weights, snaps, steps=steps, label=f"{un} chunks, variable lengths")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("regime", ["long_memory", "saturating"])
def test_rec_kernel_weight_regimes(monkeypatch, kind, regime):
    cfg = _cfg_w(kind)[0]
    caller = _caller(kind, regime)
    monkeypatch.setenv("B200_CLUSTER_CHUNKS", "32")
    N, T_in = 128, 1200
    snaps, info = _snapshots(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, seed=61), cfg.lstm_layers)
    assert info["lstm_rec.chunks_per_cluster"] == 32
    _check_layers(f"{cfg.lstm_size} lstm_rec_kernel", cfg, caller.weights, snaps, label=f"32 chunks, {regime}")


# ---- modified-base models at 128 and 256 -------------------------------------------------------------------------------
_mb = {}


def _mb_cfg_w(width, tmp_factory):
    from dorado_b200.config import load_modbase_config
    from dorado_b200.weights import synthetic_modbase_weights
    if width not in _mb:
        cfg = load_modbase_config(_resize(modbase_dir("mb384"), tmp_factory.mktemp(f"mb{width}"), 384, width))
        assert cfg.lstm_size == width
        _mb[width] = (cfg, synthetic_modbase_weights(cfg, 5))
    return _mb[width]


def _mb_runner(caller, N, sig, seq):
    from dorado_b200.modbase import B200ModBaseRunner
    r = B200ModBaseRunner(caller, N)
    for i in range(N):
        r.accept_chunk(i, sig[i], seq[i])
    return r


@pytest.mark.parametrize("width,N", [(128, 64), (128, 1024), (256, 64), (256, 1024)])
def test_modbase_probabilities(tmp_path_factory, width, N):
    from dorado_b200.modbase import B200ModBaseCaller
    from oracle.modbase_oracle import modbase_forward
    cfg, w = _mb_cfg_w(width, tmp_path_factory)
    sig, seq = modbase_inputs(cfg, N, 21)
    r = _mb_runner(B200ModBaseCaller(cfg, w), N, sig, seq)
    got = r.call_chunks(N).astype(np.float32)
    ref = modbase_forward(cfg, w, sig, seq, emulate_fp16=True)
    assert got.shape == ref.shape == (N, cfg.out_steps() * cfg.num_out)
    assert np.isfinite(got).all()
    assert np.allclose(got.reshape(N, -1, cfg.num_out).sum(-1), 1.0, atol=1e-2)
    err = np.abs(got - ref)
    p50, p99, p999 = np.percentile(err, [50, 99, 99.9])
    print(f"mb{width} N={N}: |p - oracle| p50 {p50:.2e} p99 {p99:.2e} p99.9 {p999:.2e} max {err.max():.2e} "
          f"mean {err.mean():.2e}")
    assert err.max() <= PROB_MAX and p999 <= PROB_P999 and err.mean() <= PROB_MEAN


@pytest.mark.parametrize("width", [128, 256])
def test_modbase_lstm_layers_teacher_forced(tmp_path_factory, monkeypatch, width):
    from dorado_b200.modbase import B200ModBaseCaller
    cfg, w = _mb_cfg_w(width, tmp_path_factory)
    N = 64
    sig, seq = modbase_inputs(cfg, N, 33)
    caller = B200ModBaseCaller(cfg, w)
    bufs = []
    for layers in range(3):   # the sequence buffer after 0, 1 and 2 LSTM layers
        monkeypatch.setenv("B200_DEBUG_LSTM_LAYERS", str(layers))
        r = _mb_runner(caller, N, sig, seq)
        monkeypatch.delenv("B200_DEBUG_LSTM_LAYERS")
        r.call_chunks(N)
        bufs.append(r.read_sequence_buffer().astype(np.float64))
    ratios = []
    for l in range(2):
        p = f"lstm{l + 1}."
        lw = make_layer_weights(w[p + "weight_ih_l0.tensor"], w[p + "weight_hh_l0.tensor"], w[p + "bias_ih_l0.tensor"],
                                w[p + "bias_hh_l0.tensor"])
        reverse = l == 1   # lstm1 forward in time, lstm2 reversed
        chk = check_layer(bufs[l], bufs[l + 1], lw, reverse, label=f"mb{width} {p[:-1]}")
        print(chk.describe())
        assert chk.ok, chk.describe()
        wrong = check_layer(bufs[l], bufs[l + 1], lw, not reverse)
        assert wrong.max_ratio >= 10.0, f"{p[:-1]} in the wrong direction only reaches {wrong.max_ratio:.3g} x the budget"
        ratios.append(chk.max_ratio)
        _stats.setdefault(f"{width} lstm_rec_kernel (modbase)", []).append((chk.max_ratio, chk.median_ratio))
    print(f"mb{width}: worst error / budget per layer {ratios}")


# ---- error codes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_batch_not_a_multiple_of_32(kind):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _cfg_w(kind)
    caller = B200Caller(cfg, w)
    with pytest.raises(L.B200Error) as e:
        B200ModelRunner(caller, 48, 1200)
    assert e.value.status == L.B200_ERR_INVALID
    caller.close()
