"""lstm_size 768 and 1024 on the GPU: x-projection GEMM + lstm_grid_rec_kernel (groups of C / 16 CTAs exchanging h
through L2).  Scores are held to the numpy oracle with the bounds of tests/test_forward_gpu.py, calls to the C oracle
decoding the engine's own scores; the result must not depend on the launch shape the plan picks.

The pre-v4 768 model ends in 5 tanh(z) (no clamp).  Its slope, up to 5 at z = 0, multiplies the fp16 rounding noise of the
768 LSTM outputs that z sums: with the LSTM output itself as close to the oracle as hac's (max 3.9e-3 against 3.5e-3, 32
chunks of 1200 samples, measured on an H100), ~11 % of its scores differ by more than 1e-3 of max|ref|.  Its score bounds are
therefore those of _check_scores in the domain of z, i.e. every error bound multiplied by that slope."""
import os

import numpy as np
import pytest

from test_forward_gpu import _check_scores
from test_wide_lstm_cpu import UNITS, grid_shape, model_dir

pytestmark = pytest.mark.gpu

WIDE = ["lstm768", "lstm1024"]
_weights = {}


def _cfg_w(kind):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    if kind not in _weights:
        cfg = load_model_config(model_dir(kind))
        _weights[kind] = (cfg, synthetic_weights(cfg, 42))
    return _weights[kind]


def _slope(cfg):
    """Largest gain of the CRF output nonlinearity: 5 for tanh x 5, else 1."""
    return 5.0 if cfg.scale == 5.0 else 1.0


def _check_wide_scores(got, ref16, ref32, cfg):
    got = got.astype(np.float32)
    if cfg.clamp:
        got = np.clip(got, -5.0, 5.0)
    k = _slope(cfg)
    scale = max(1.0, float(np.abs(ref16).max()))
    err = np.abs(got - ref16)
    frac_bad = float((err > k * 1e-3 * scale).mean())
    assert frac_bad <= 1e-3, f"{frac_bad:.2e} of scores off by more than {k:g}e-3 relative (max err {err.max():.4f})"
    assert err.max() <= k * 4e-3 * scale, f"max score error vs fp16-storage oracle {err.max():.4f}"
    rel_l2 = float(np.linalg.norm(got - ref32) / np.linalg.norm(ref32))
    assert rel_l2 <= k * 5e-3, f"relative L2 error vs fp32 oracle {rel_l2:.2e}"
    assert np.abs(got - ref32).max() <= k * 2e-2 * scale


def _runner(kind, N, T, seed=1234, num_runners=2):
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _cfg_w(kind)
    caller = B200Caller(cfg, w, num_runners=num_runners)
    runner = B200ModelRunner(caller, N, T)
    sig = np.random.default_rng(seed).standard_normal((N, runner.chunk_size())).astype(np.float16)
    for i in range(N):
        runner.accept_chunk(i, sig[i])
    return cfg, w, caller, runner, sig


@pytest.mark.parametrize("kind", WIDE)
@pytest.mark.parametrize("N,T", [(32, 1200), (64, 1998), (128, 600)])
def test_wide_lstm_scores(kind, N, T):
    from oracle import nn_oracle
    cfg, w, caller, runner, sig = _runner(kind, N, T)
    info = runner.plan_info()
    assert info["lstm_grid.ctas"] == info["lstm_grid.groups"] * cfg.lstm_size // UNITS <= 132
    if N == 128:
        assert info["lstm_grid.launches_per_layer"] > 1     # the layer's chunks are split over several launches
    got = runner.forward_scores(N)
    ref32 = nn_oracle.forward(cfg, w, sig.astype(np.float32))
    ref16 = nn_oracle.forward(cfg, w, sig.astype(np.float32), emulate_fp16=True)
    assert got.shape == ref32.shape == (N, runner.chunk_size() // cfg.stride, 4096)
    if _slope(cfg) == 1.0:
        _check_scores(got, ref16, ref32, cfg.clamp)
    _check_wide_scores(got, ref16, ref32, cfg)


@pytest.mark.parametrize("kind", WIDE)
def test_wide_lstm_calls_match_the_decoder_oracle(crf_oracle, kind):
    cfg, w, caller, runner, sig = _runner(kind, 32, 1200)
    scores = runner.forward_scores(32)
    chunks = runner.call_chunks(32)
    ref = crf_oracle.decode(scores, clamp_val=5.0 if cfg.clamp else 0.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(chunks):
        assert c.sequence == ref.sequences[i] and c.qstring == ref.qstrings[i]
        np.testing.assert_array_equal(c.moves, ref.moves[i])
    assert sum(len(c.sequence) for c in chunks) > 32 * 10      # real calls, not empty strings


@pytest.mark.parametrize("kind", WIDE)
def test_wide_lstm_variable_chunk_sizes(crf_oracle, kind):
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
    clamp = 5.0 if cfg.clamp else 0.0
    for i in range(64):
        tn = int(lens[i]) // cfg.stride
        assert len(called[i].moves) == tn
        ref = crf_oracle.decode(scores[i:i + 1, :tn], clamp_val=clamp, q_shift=cfg.qbias, q_scale=cfg.qscale)
        assert called[i].sequence == ref.sequences[0] and called[i].qstring == ref.qstrings[0]
        assert (called[i].moves == ref.moves[0]).all()
        if i in (0, 1, 2, 5, 33, 63):   # numpy forward of the chunk alone, at its own length
            want = nn_oracle.forward(cfg, w, sig[i][None].astype(np.float32), emulate_fp16=True)[0]
            got = scores[i, :tn].astype(np.float32)
            got = np.clip(got, -5, 5) if cfg.clamp else got
            err = np.abs(got - want)
            scale = max(1.0, float(np.abs(want).max()))
            k = _slope(cfg)
            assert (err > k * 1e-3 * scale).mean() <= 2e-3 and err.max() <= k * 6e-3 * scale, (i, tn, float(err.max()))
    for i in (1, 5):   # a fixed-shape runner of exactly that chunk size gives the same call
        alone = B200ModelRunner(caller, 32, int(lens[i]))
        alone.accept_chunk(0, sig[i])
        a = alone.call_chunks(1)[0]
        assert a.sequence == called[i].sequence and a.qstring == called[i].qstring and (a.moves == called[i].moves).all()
        alone.close()


@pytest.mark.parametrize("kind", WIDE)
def test_wide_lstm_launch_shapes_agree(kind):
    """Chunks per group (32, 64), groups per launch and num_runners change only how the batch is cut into launches:
    scores and calls are bit-identical, for fixed and for variable chunk sizes; the plan follows the sizing rule that
    tests/test_wide_lstm_cpu.py checks."""
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _cfg_w(kind)
    G = cfg.lstm_size // UNITS
    N, T = 128, 600
    rng = np.random.default_rng(3)
    sig = rng.standard_normal((N, cfg.normalise_chunk_size(T))).astype(np.float16)
    lens = rng.integers(10, sig.shape[1] // cfg.stride + 1, size=N) * cfg.stride
    shapes = [(None, None, 1), (None, None, 4), ("32", "1", 2), ("32", "2", 2), ("64", "1", 2), ("64", "2", 2)]
    got = {}
    try:
        for nb, groups, R in shapes:
            for k, v in (("B200_GRID_CHUNKS", nb), ("B200_GRID_GROUPS", groups)):
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
            caller = B200Caller(cfg, w, num_runners=R)
            runner = B200ModelRunner(caller, N, T)
            info = runner.plan_info()
            assert info["lstm_grid.ctas"] <= 132
            if nb is None:
                mg = 132 // G
                assert (info["lstm_grid.chunks_per_group"], info["lstm_grid.groups"],
                        info["lstm_grid.launches_per_layer"]) == grid_shape(N, mg, mg, R)
            else:
                assert (info["lstm_grid.chunks_per_group"], info["lstm_grid.groups"]) == (int(nb), int(groups))
            for i in range(N):
                runner.accept_chunk(i, sig[i])
            fixed = runner.forward_scores(N).copy()
            for i in range(N):
                runner.accept_chunk_var(i, sig[i, :lens[i]])
            got[(nb, groups, R)] = (fixed, runner.forward_scores(N).copy(), [np.array(a) for a in runner.call_chunks_raw(N)])
            runner.close()
            caller.close()
    finally:
        os.environ.pop("B200_GRID_CHUNKS", None)
        os.environ.pop("B200_GRID_GROUPS", None)
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


def test_wide_flstm_folds_like_the_plain_lstm(tmp_path):
    """A 1024-wide FLSTM model and the plain LSTM model with the folded products up @ dn as weights give identical scores."""
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import fold_flstm_weights, synthetic_weights
    src = (model_dir("lstm1024") / "config.toml").read_text()
    flstm = src.replace('type = "lstm"\n', 'type = "flstm"\ninner_dim = 128\n')
    assert flstm.count("inner_dim = 128") == 5
    (tmp_path / "flstm1024").mkdir()
    (tmp_path / "flstm1024" / "config.toml").write_text(flstm)
    cfg_f = load_model_config(tmp_path / "flstm1024")
    cfg_l = load_model_config(model_dir("lstm1024"))
    assert cfg_f.is_flstm_model and cfg_f.lstm_size == 1024 and cfg_f.lstm_layers == 5
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


def test_wide_lstm_errors(tmp_path):
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    (tmp_path / "lstm512").mkdir()
    src = (model_dir("lstm1024") / "config.toml").read_text().replace("1024", "512")
    (tmp_path / "lstm512" / "config.toml").write_text(src)
    cfg = load_model_config(tmp_path / "lstm512")
    assert cfg.lstm_size == 512
    with pytest.raises(L.B200Error) as e:
        B200Caller(cfg, synthetic_weights(cfg, 1))
    assert e.value.status == L.B200_ERR_UNSUPPORTED
    cfg, w = _cfg_w("lstm768")
    caller = B200Caller(cfg, w)
    with pytest.raises(L.B200Error) as e:
        B200ModelRunner(caller, 48, 1200)
    assert e.value.status == L.B200_ERR_INVALID
