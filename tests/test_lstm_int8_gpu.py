"""The int8_lstm precision on the GPU (hac and the 256-wide fixture): the int8 GEMM and conv3's int8 store against float64,
every LSTM layer against the teacher-forced float64 reference, whole-model scores against tests/lstm_int8_ref.py, calls
against the C decoder oracle, int8 against fp16, launch-shape independence, memory and the error paths.

Every "measured" below is from one NVIDIA H100 80GB HBM3 at a 700 W power limit.
"""
import ctypes as C
import os

import numpy as np
import pytest

import lstm_int8_ref as I8
from conftest import model_dir
from lstm_layer_ref import read_x2, ulp16, workspace_layout
from test_lstm128_256_cpu import model_dir as synthetic_model_dir
from test_lstm_layers_gpu import _signals, _variable_lengths

pytestmark = pytest.mark.gpu

KINDS = ["hac", "lstm256"]
_models = {}
_callers = {}


@pytest.fixture(scope="module", autouse=True)
def _close():
    yield
    for c in _callers.values():
        c.close()
    _callers.clear()


def _cfg_w(kind):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    if kind not in _models:
        cfg = load_model_config(model_dir("hac") if kind == "hac" else synthetic_model_dir(kind))
        _models[kind] = (cfg, synthetic_weights(cfg, 42))
    return _models[kind]


def _caller(kind, precision="int8_lstm", num_runners=2):
    from dorado_b200.runner import B200Caller
    key = (kind, precision, num_runners)
    if key not in _callers:
        cfg, w = _cfg_w(kind)
        _callers[key] = B200Caller(cfg, w, num_runners=num_runners, precision=precision)
    return _callers[key]


def _runner(caller, N, T, sig):
    from dorado_b200.runner import B200ModelRunner
    runner = B200ModelRunner(caller, N, T)
    for i in range(N):
        if isinstance(sig, list):
            runner.accept_chunk_var(i, sig[i])
        else:
            runner.accept_chunk(i, sig[i])
    return runner


def _read_seq8(runner, cfg, N, T_in):
    """The int8 sequence buffer's first T_out rows [T_out][N][C]."""
    lay = workspace_layout(cfg, N, T_in)
    raw = runner.debug_read_workspace(lay["seq"], lay["T_out"] * N * cfg.lstm_size)
    return raw.view(np.int8).reshape(lay["T_out"], N, cfg.lstm_size).copy()


def _snapshots8(monkeypatch, caller, cfg, N, T_in, sig, layers):
    out = []
    for k in layers:
        monkeypatch.setenv("B200_DEBUG_LSTM_LAYERS", str(k))
        runner = _runner(caller, N, T_in, sig)
        monkeypatch.delenv("B200_DEBUG_LSTM_LAYERS")
        runner.forward_scores(N)
        out.append(_read_seq8(runner, cfg, N, T_in))
        info = runner.plan_info()
        runner.close()
    return out, info


# ---- the int8 GEMM ------------------------------------------------------------------------------------------------------
# gx shapes (N = 4C, K = C) and the CRF linear's (hac: 1024 x 384; the 256 fixture: 1024 x 256); M = 8192 stands for a full
# batch (64 row tiles: every CTA of the persistent grid takes tiles, some take two)
@pytest.mark.parametrize("N,K", [(1024, 256), (1536, 384), (1024, 384)])
@pytest.mark.parametrize("M", [1, 200, 333, 8192])
def test_gemm_s8(M, N, K):
    from dorado_b200 import lib as L
    rng = np.random.default_rng(M * 7 + N + K)
    a = rng.integers(-127, 128, size=(M, K)).astype(np.int8)
    w = rng.integers(-127, 128, size=(N, K)).astype(np.int8)
    a[0, :], w[0, :] = 127, -127                                  # the largest |acc| = 127^2 K
    scale = (rng.uniform(0.5, 2.0, N) / (127.0 * 128.0)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    acc = a.astype(np.float64) @ w.astype(np.float64).T          # exact
    for b in (None, bias):
        got = L.test_gemm_s8(a, w, scale, b).astype(np.float64)
        want = acc * scale.astype(np.float64) + (0 if b is None else b.astype(np.float64))
        want16 = want.astype(np.float16).astype(np.float64)
        err = np.abs(got - want16)
        assert (err <= ulp16(want16)).all(), f"max error {err.max():.3e}"
        # one rounding of a value computed in fp32: all but a few ties agree exactly
        assert (got != want16).mean() <= 1e-3
    if M == 200:   # tanh x 5 (the CRF linear of models with scale = 5)
        got = L.test_gemm_s8(a, w, scale, bias, activation=3).astype(np.float64)
        want = 5.0 * np.tanh(acc * scale.astype(np.float64) + bias.astype(np.float64))
        assert np.abs(got - want).max() <= 4e-3     # fp16 spacing at 5 is 3.9e-3


# ---- conv3's int8 store ---------------------------------------------------------------------------------------------------
# Budget of 127 * (tanh_fast's error + the fp32 accumulation of K = 16 winlen products): 127 * 5e-5 levels.
# Measured: 9.8e-6 (hac) and 1.7e-5 (lstm256) of the levels differ from round(127 tanh) of the float64 pre-activation.
@pytest.mark.parametrize("kind", KINDS)
def test_conv3_int8_store(monkeypatch, kind):
    cfg, w = _cfg_w(kind)
    N, T_in = 32, 600
    sig = _signals(cfg, N, T_in, seed=11)
    monkeypatch.setenv("B200_DEBUG_LSTM_LAYERS", "0")
    runner = _runner(_caller(kind), N, T_in, sig)
    monkeypatch.delenv("B200_DEBUG_LSTM_LAYERS")
    runner.forward_scores(N)
    got = _read_seq8(runner, cfg, N, T_in).astype(np.float64)       # [T_out][N][C]
    x2 = read_x2(runner, cfg, N, T_in).astype(np.float64)           # the engine's own conv2 output [N][Tp][16]
    runner.close()
    c3 = cfg.convs[2]
    w3 = np.asarray(w["2.conv.weight.tensor"], np.float16).astype(np.float64)      # [C][16][winlen]
    wk = w3.transpose(0, 2, 1).reshape(cfg.lstm_size, -1)                           # K index = tap * 16 + channel
    T_out = T_in // cfg.stride
    rows = np.stack([x2[:, t * c3.stride:t * c3.stride + c3.winlen].reshape(N, -1) for t in range(T_out)])   # [T_out][N][K]
    pre = rows @ wk.T + np.asarray(w["2.conv.bias.tensor"], np.float64)
    t127 = 127.0 * np.tanh(pre)
    differs = float((np.rint(t127) != got).mean())
    print(f"\n[{kind}] conv3 int8 store: {differs:.2e} of {got.size} levels differ from round(127 tanh(pre))")
    assert (np.abs(t127 - got) <= 0.5 + 127 * 5e-5).all()
    assert differs <= 1e-3 and np.abs(got).max() <= 127


# ---- every layer, teacher-forced ----------------------------------------------------------------------------------------
# Measured over the 60 layer checks: worst excess / budget 0.003 - 0.10; 0.8e-4 - 1.7e-4 of the levels differ from
# round(127 h_ref) (the tanh.approx error next to a rounding tie).  In the sensitivity test the wrong direction is 7578 x
# the budget or more with 0.92 of the levels different, the shifted scale rows 243 x with 0.77.
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("un", [16, 32, 64])
def test_rec_i8_kernel_layers(monkeypatch, kind, un):
    cfg, w = _cfg_w(kind)
    caller = _caller(kind)
    monkeypatch.setenv("B200_CLUSTER_CHUNKS", str(un))
    N, T_in = 64, 900
    lens, steps = _variable_lengths(cfg, N, T_in, un, seed=52)
    for label, sig, st in (("fixed", _signals(cfg, N, T_in, seed=51), None),
                           ("variable", _signals(cfg, N, T_in, 53, lens), steps)):
        snaps, info = _snapshots8(monkeypatch, caller, cfg, N, T_in, sig, range(cfg.lstm_layers + 1))
        assert info["lstm_rec.chunks_per_cluster"] == un and info["lstm_rec.ctas"] == N // un * 8 and info["lstm.int8"] == 1
        for l in range(cfg.lstm_layers):
            reverse = l % 2 == 0
            lw = I8.dequantised_layer_weights(cfg, w, l)
            ratio, differs, _ = I8.check_layer(snaps[l], snaps[l + 1], lw, reverse, st)
            print(f"\n  [{kind} {un} chunks, {label}] layer {l}: worst excess / budget {ratio.max():.3f}, "
                  f"{differs:.2e} of the levels differ from round(127 h_ref)")
            assert ratio.max() <= 1.0 and differs <= 5e-3
            assert np.abs(snaps[l + 1]).max() > 32     # the layer has real outputs


def test_rec_i8_kernel_check_is_sensitive(monkeypatch):
    """The same check must fail by a wide margin against the reference run in the wrong direction, and against one that
    takes every gate row's scale from the row above.  Every second gate row of W_ih and W_hh is halved here, so that
    neighbouring rows have scales a factor of two apart (the synthetic rows' scales are all alike otherwise)."""
    from dorado_b200.runner import B200Caller
    cfg, w = _cfg_w("hac")
    w = dict(w)
    halve = np.where(np.arange(4 * cfg.lstm_size) % 2 == 0, 1.0, 0.5).astype(np.float32)[:, None]
    for l in range(cfg.lstm_layers):
        for name in ("weight_ih_l0.tensor", "weight_hh_l0.tensor"):
            key = f"{len(cfg.convs) + l + 1}.rnn.{name}"
            w[key] = w[key] * halve
    caller = B200Caller(cfg, w, precision="int8_lstm")
    N, T_in = 32, 600
    snaps, _ = _snapshots8(monkeypatch, caller, cfg, N, T_in, _signals(cfg, N, T_in, seed=61), range(3))
    caller.close()
    for l in range(2):
        reverse = l % 2 == 0
        lw = I8.dequantised_layer_weights(cfg, w, l)
        ratio, differs, _ = I8.check_layer(snaps[l], snaps[l + 1], lw, reverse)
        assert ratio.max() <= 1.0 and differs <= 5e-3
        wrong_dir = I8.check_layer(snaps[l], snaps[l + 1], lw, not reverse)
        q_hh, inv = I8.layer_params(cfg, w, l)[1:3]
        lw.w_hh = q_hh.astype(np.float64) * (np.roll(inv, 1).astype(np.float64) * 127.0)[:, None]
        wrong_scale = I8.check_layer(snaps[l], snaps[l + 1], lw, reverse)
        print(f"\n  layer {l}: wrong direction {wrong_dir[0].max():.0f} x the budget, {wrong_dir[1]:.2f} of the levels differ; "
              f"scale rows shifted {wrong_scale[0].max():.0f} x, {wrong_scale[1]:.2f}")
        assert wrong_dir[0].max() >= 10 and wrong_dir[1] >= 0.2
        assert wrong_scale[0].max() >= 10 and wrong_scale[1] >= 0.2


# ---- whole model ----------------------------------------------------------------------------------------------------------
# |score - lstm_int8_ref| as a fraction of the score range (10, clamped to +-5).  The reference uses exact tanh and sigmoid,
# the engine tanh.approx: about 1e-4 of the levels of h flip next to a tie in every layer (above), each flip moves the
# pre-activations of the next step by a level's worth, and five quantised recurrences amplify that until the two runs
# differ like two independent roundings.  So this bound is loose by nature (about a third of the int8-against-fp16
# difference); the layer checks above carry the exactness claim.  Measured over the five cases: p50 2.4e-3 - 2.7e-3,
# p99 1.0e-2, p99.9 1.2e-2 - 1.4e-2, max 2.4e-2, mean 2.9e-3 - 3.2e-3.
SCORE_P50, SCORE_P999, SCORE_MEAN = 5e-3, 3e-2, 6e-3


def _check_model(crf_oracle, kind, N, T, ref_chunks):
    cfg, w = _cfg_w(kind)
    sig = _signals(cfg, N, cfg.normalise_chunk_size(T), seed=21)
    runner = _runner(_caller(kind), N, T, sig)
    scores = runner.forward_scores(N)
    chunks = runner.call_chunks(N)
    runner.close()
    want = I8.forward(cfg, w, sig[:ref_chunks].astype(np.float32))
    got = np.clip(scores[:ref_chunks].astype(np.float32), -5, 5)
    err = np.abs(got - want) / 10.0
    p50, p99, p999 = np.percentile(err, [50, 99, 99.9])
    print(f"\n[{kind} int8 {N} x {T}] |score - ref| / range over {ref_chunks} chunks: p50 {p50:.2e} p99 {p99:.2e} p99.9 {p999:.2e} "
          f"max {err.max():.2e} mean {err.mean():.2e}")
    assert p50 <= SCORE_P50 and p999 <= SCORE_P999 and err.mean() <= SCORE_MEAN
    ref = crf_oracle.decode(scores, clamp_val=5.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(chunks):
        assert c.sequence == ref.sequences[i] and c.qstring == ref.qstrings[i]
        np.testing.assert_array_equal(c.moves, ref.moves[i])
    assert sum(len(c.sequence) for c in chunks) > N * 10
    return scores, chunks


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N,T", [(32, 3000), (64, 1998)])
def test_model_scores_and_calls(crf_oracle, kind, N, T):
    _check_model(crf_oracle, kind, N, T, ref_chunks=N)


def test_model_full_size(crf_oracle):
    """hac at batch 512 x 9996 samples; the numpy reference runs the first 4 chunks (chunks are independent)."""
    _check_model(crf_oracle, "hac", 512, 9996, ref_chunks=4)


@pytest.mark.parametrize("kind", KINDS)
def test_int8_against_fp16(kind):
    """Synthetic weights: how far the precision moves scores and calls here, not a statement about accuracy on real reads."""
    cfg, w = _cfg_w(kind)
    N, T = 64, 3000
    sig = _signals(cfg, N, cfg.normalise_chunk_size(T), seed=31)
    out = {}
    for precision in ("int8_lstm", "fp16"):
        runner = _runner(_caller(kind, precision), N, T, sig)
        out[precision] = (np.clip(runner.forward_scores(N).astype(np.float32), -5, 5), runner.call_chunks(N))
        runner.close()
    a, b = out["int8_lstm"][0], out["fp16"][0]
    rel = float(np.linalg.norm(a - b) / np.linalg.norm(b))
    same = np.mean([x.sequence == y.sequence for x, y in zip(out["int8_lstm"][1], out["fp16"][1])])
    print(f"\n[{kind}] int8_lstm vs fp16, {N} x {T}: score relative L2 {rel:.3f}, {same:.2f} of the sequences identical")
    assert 0 < rel <= 0.1     # measured 0.035 for both models (0 and 0.03 of the 64 sequences identical); the CPU restatements: 0.034


def test_default_precision_is_fp16():
    cfg, w = _cfg_w("hac")
    from dorado_b200.runner import B200Caller
    N, T = 32, 1200
    sig = _signals(cfg, N, T, seed=41)
    explicit = _runner(_caller("hac", "fp16"), N, T, sig)
    default_caller = B200Caller(cfg, w)
    default = _runner(default_caller, N, T, sig)
    assert "lstm.int8" not in default.plan_info()
    np.testing.assert_array_equal(default.forward_scores(N), explicit.forward_scores(N))
    default.close()
    explicit.close()
    default_caller.close()


@pytest.mark.parametrize("kind", KINDS)
def test_launch_shapes_agree(kind):
    """num_runners and chunks per cluster change the launch shape only: int8 scores and calls are bit-identical, for fixed
    and variable chunk sizes."""
    from dorado_b200.runner import B200Caller
    cfg, w = _cfg_w(kind)
    N, T = 128, 600
    rng = np.random.default_rng(3)
    sig = rng.standard_normal((N, T)).astype(np.float16)
    lens = rng.integers(1, T // cfg.stride + 1, size=N) * cfg.stride
    shapes = [(None, 2), (None, 1), (None, 4), ("16", 1), ("32", 4), ("64", 2)]
    got = {}
    try:
        for nb, R in shapes:
            if nb is None:
                os.environ.pop("B200_CLUSTER_CHUNKS", None)
            else:
                os.environ["B200_CLUSTER_CHUNKS"] = nb
            caller = B200Caller(cfg, w, num_runners=R, precision="int8_lstm")
            runner = _runner(caller, N, T, sig)
            assert runner.plan_info()["lstm.int8"] == 1
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
        (mv, sq, qs, nb_), (mv0, sq0, qs0, nb0) = got[key][2], base[2]
        np.testing.assert_array_equal(nb_, nb0)
        for i in range(N):
            tn = int(lens[i]) // cfg.stride
            np.testing.assert_array_equal(got[key][1][i, :tn], base[1][i, :tn])
            assert (mv[i, :tn] == mv0[i, :tn]).all() and (sq[i, :nb_[i]] == sq0[i, :nb_[i]]).all()
            assert (qs[i, :nb_[i]] == qs0[i, :nb_[i]]).all()


@pytest.mark.parametrize("kind", KINDS)
def test_runner_bytes(kind):
    from dorado_b200.runner import B200ModelRunner
    cfg, _ = _cfg_w(kind)
    i8, f16 = _caller(kind), _caller(kind, "fp16")
    for N, T in ((64, 1998), (512, 9996)):
        want = i8.runner_bytes(N, T)
        before = i8.stats()["arena_bytes"]
        runner = B200ModelRunner(i8, N, T)
        assert i8.stats()["arena_bytes"] - before == want
        runner.close()
        # the sequence buffer [T_out + 1][N][C] is one byte per element instead of two
        saved = f16.runner_bytes(N, T) - want
        print(f"\n[{kind}] runner_bytes({N}, {T}): int8_lstm {want}, fp16 {want + saved}")
        seq = (T // cfg.stride + 1) * N * cfg.lstm_size
        assert 0 < saved and abs(saved - seq) < 256


# ---- error paths: every unsupported shape fails at engine creation ------------------------------------------------------
def _create(cfg, w, precision=None, **fields):
    from dorado_b200 import lib as L
    from dorado_b200.runner import _weight_array
    lib = L.load_library()
    desc = L.model_desc_from_config(cfg, precision or "fp16")
    for k, v in fields.items():
        setattr(desc, k, v)
    arr, keep = _weight_array(w)
    handle = C.c_void_p()
    status = lib.b200_engine_create_sized(C.byref(desc), C.sizeof(desc), arr, len(w), 0, C.byref(handle))
    msg = lib.b200_last_error().decode() if status != 0 else ""
    if status == 0:
        lib.b200_engine_destroy(handle)
    return status, msg


def _variant(tmp_path, kind, name, edit):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    src = ((model_dir("hac") if kind == "hac" else synthetic_model_dir(kind)) / "config.toml").read_text()
    d = tmp_path / name
    d.mkdir()
    (d / "config.toml").write_text(edit(src))
    cfg = load_model_config(d)
    return cfg, synthetic_weights(cfg, 1)


def test_error_paths(tmp_path):
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    from test_wide_lstm_cpu import model_dir as wide_model_dir
    hac, w_hac = _cfg_w("hac")
    status, msg = _create(hac, w_hac, lstm_precision=2)
    assert status == L.B200_ERR_INVALID and "lstm_precision" in msg
    sup = load_model_config(model_dir("sup"))
    status, msg = _create(sup, synthetic_weights(sup, 1), lstm_precision=1)
    assert status == L.B200_ERR_INVALID and "LSTM models only" in msg
    status, msg = _create(hac, w_hac, precision="fp8_ffn")
    assert status == L.B200_ERR_INVALID and "transformer models only" in msg
    unsupported = {
        "96": (load_model_config(model_dir("fast")), "lstm_size 96"),
        "128": (load_model_config(synthetic_model_dir("lstm128")), "lstm_size 128"),
        "768": (load_model_config(wide_model_dir("lstm768")), "lstm_size 768"),
        "1024": (load_model_config(wide_model_dir("lstm1024")), "lstm_size 1024"),
    }
    for name, (cfg, text) in unsupported.items():
        status, msg = _create(cfg, synthetic_weights(cfg, 1), precision="int8_lstm")
        assert status == L.B200_ERR_UNSUPPORTED and text in msg and "256 and 384" in msg, (name, status, msg)
    cfg, w = _variant(tmp_path, "hac", "hac192", lambda s: s.replace("384", "192"))
    status, msg = _create(cfg, w, precision="int8_lstm")
    assert status == L.B200_ERR_UNSUPPORTED and "lstm_size 192" in msg
    cfg, w = _variant(tmp_path, "hac", "hac_swish", lambda s: s.replace('activation = "tanh"', 'activation = "swish"'))
    assert cfg.lstm_size == 384 and cfg.convs[2].activation != hac.convs[2].activation
    status, msg = _create(cfg, w, precision="int8_lstm")
    assert status == L.B200_ERR_UNSUPPORTED and "tanh last convolution" in msg
    cfg, w = _variant(tmp_path, "lstm256", "flstm256", lambda s: s.replace('type = "lstm"\n', 'type = "flstm"\ninner_dim = 64\n'))
    assert cfg.is_flstm_model
    status, msg = _create(cfg, w, precision="int8_lstm")
    assert status == L.B200_ERR_UNSUPPORTED and "FLSTM" in msg
    assert _create(cfg, w)[0] == 0    # the same model runs in fp16


def test_binary_built_against_the_earlier_header_still_runs():
    """A caller compiled before lstm_precision existed passes a descriptor that ends at tx_precision, with whatever its
    stack holds behind it.  The exported b200_engine_create reads that far only, so the engine comes up in fp16."""
    from dorado_b200 import lib as L
    from dorado_b200.runner import _weight_array
    lib = L.load_library()
    cfg, w = _cfg_w("hac")
    desc = L.model_desc_from_config(cfg)
    old_size = L.ModelDesc.lstm_precision.offset
    buf = (C.c_ubyte * (old_size + 64))(*([0xA5] * (old_size + 64)))
    C.memmove(buf, C.byref(desc), old_size)
    arr, keep = _weight_array(w)
    handle = C.c_void_p()
    status = lib.b200_engine_create(C.cast(buf, C.POINTER(L.ModelDesc)), arr, len(w), 0, C.byref(handle))
    assert status == 0, lib.b200_last_error().decode()
    lib.b200_engine_destroy(handle)
    # the same bytes declared at the full size are a bad lstm_precision
    status = lib.b200_engine_create_sized(C.cast(buf, C.POINTER(L.ModelDesc)), C.sizeof(L.ModelDesc), arr, len(w), 0, C.byref(handle))
    assert status == L.B200_ERR_INVALID and "lstm_precision" in lib.b200_last_error().decode()

