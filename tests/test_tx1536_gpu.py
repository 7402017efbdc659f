"""The 1536-wide transformer on the GPU: the attention kernel against float64 numpy through b200_test_attention, the model's
scores against the numpy oracle with the bounds of tests/test_forward_gpu.py (reduced depths, cross shapes that change
one thing at a time, the full 18 layers), calls against the C oracle decoding the engine's own scores, concurrent
runners, the separate RMSNorm pass, the shapes the engine refuses and the runner's memory.  The fixture is described in
tests/test_tx1536_cpu.py."""
import threading

import numpy as np
import pytest

from test_forward_gpu import _check_scores
from test_tx1536_cpu import config_variant, model_dir

pytestmark = pytest.mark.gpu

_cache = {}


def _model(path, seed=42):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    key = (str(path), seed)
    if key not in _cache:
        cfg = load_model_config(path)
        _cache[key] = (cfg, synthetic_weights(cfg, seed))
    return _cache[key]


def _signal(cfg, N, T, seed):
    return np.random.default_rng(seed).standard_normal((N, cfg.normalise_chunk_size(T))).astype(np.float16)


def _scores(cfg, w, sig, num_runners=2):
    from dorado_b200.runner import B200Caller, B200ModelRunner
    caller = B200Caller(cfg, w, num_runners=num_runners)
    N, T = sig.shape
    runner = B200ModelRunner(caller, N, T)
    for i in range(N):
        runner.accept_chunk(i, sig[i])
    got = runner.forward_scores(N).copy()
    runner.close()
    caller.close()
    return got


def _against_oracle(cfg, w, sig, got, max_frac_bad=1e-3, label=""):
    from oracle import nn_oracle
    x = sig.astype(np.float32)
    ref32 = nn_oracle.forward(cfg, w, x)
    ref16 = nn_oracle.forward(cfg, w, x, emulate_fp16=True)
    assert got.shape == ref32.shape == (sig.shape[0], sig.shape[1] // cfg.stride, cfg.outsize)
    scale = max(1.0, float(np.abs(ref16).max()))
    err = np.abs(got.astype(np.float32) - ref16)
    rel_l2 = float(np.linalg.norm(got.astype(np.float32) - ref32) / np.linalg.norm(ref32))
    print(f"\n[{label}] vs fp16 oracle: {(err > 1e-3 * scale).mean():.2e} beyond 1e-3 x max|ref|, max {err.max() / scale:.2e} "
          f"x max|ref|; vs fp32 oracle: relative L2 {rel_l2:.2e}")
    _check_scores(got, ref16, ref32, cfg.clamp, max_frac_bad=max_frac_bad)


# ---- attention kernel ---------------------------------------------------------------------------------------------------
def _attention_ref(qkv, win_upper, win_lower):
    """float64 softmax(q k^T / 8) v over the window -win_upper <= j - i <= win_lower, from the fp16 inputs."""
    N, T, _, H, D = qkv.shape
    x = qkv.astype(np.float64)
    i = np.arange(T)[:, None]
    j = np.arange(T)[None, :]
    mask = (j - i >= -win_upper) & (j - i <= win_lower)
    out = np.empty((N, T, H, D))
    for n in range(N):
        for h in range(H):
            s = x[n, :, 0, h] @ x[n, :, 1, h].T / 8.0
            s = np.where(mask, s, -np.inf)
            p = np.exp(s - s.max(axis=1, keepdims=True))
            out[n, :, h] = (p / p.sum(axis=1, keepdims=True)) @ x[n, :, 2, h]
    return out.reshape(N, T, H * D)


ATT_WINDOWS = [(127, 128), (255, 256), (256, 256), (0, 256), (256, 0), (0, 0)]
ATT_TS = [1, 100, 127, 128, 129, 640, 1000, 1024, 2048]


@pytest.mark.parametrize("H", [8, 24])
@pytest.mark.parametrize("win", ATT_WINDOWS)
def test_attention_kernel(win, H):
    """tx_attention_tc_kernel as the model launches it, against float64.  The kernel rounds P = exp(s - m) to fp16 before
    P V (relative 2^-11 per weight, while the normaliser l sums the unrounded fp32 P) and rounds the output to fp16
    (2^-11 relative): together at most 2^-10 x max|v| per output, plus the fp32 accumulation of S and P V.  Bound:
    1.5e-3 x max|v|.  Ragged final tiles (T not a multiple of 128), T < 128, and two chunks back to back for some T."""
    from dorado_b200 import lib as L
    worst = 0.0
    for T in ATT_TS:
        N = 2 if T in (100, 129, 1000) else 1
        rng = np.random.default_rng(T * 31 + H)
        qkv = rng.standard_normal((N, T, 3, H, 64)).astype(np.float16)
        qkv[:, :, :2] *= np.float16(2.0)   # scores q.k / 8 of standard deviation 4: peaked, not one-hot
        got = L.test_attention(qkv, *win).astype(np.float64)
        ref = _attention_ref(qkv, *win)
        vmax = float(np.abs(qkv[:, :, 2].astype(np.float64)).max())
        err = float(np.abs(got - ref).max())
        worst = max(worst, err / vmax)
        assert err <= 1.5e-3 * vmax, (win, H, T, err, vmax)
        if T >= 640 and win != (0, 0):
            # the band matters: the one-key-narrower window is far outside the bound
            narrower = _attention_ref(qkv[:1, :640], max(win[0] - 1, 0), win[1] if win[0] > 0 else win[1] - 1)
            assert np.abs(got[:1, :640] - narrower).max() > 1e-2 * vmax
    print(f"\n[attention {win} H={H}] worst error {worst:.2e} x max|v|")


def test_attention_hook_rejects_wide_windows():
    from dorado_b200 import lib as L
    qkv = np.zeros((1, 256, 3, 8, 64), np.float16)
    for win in ((257, 0), (0, 257), (-1, 0)):
        with pytest.raises(L.B200Error) as e:
            L.test_attention(qkv, *win)
        assert e.value.status == L.B200_ERR_UNSUPPORTED


# ---- model scores -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth", [1, 2])
def test_reduced_depth_scores(tmp_path, depth):
    cfg, w = _model(config_variant(tmp_path, depth=depth, name=f"d{depth}"))
    sig = _signal(cfg, 2, 7680, seed=depth)
    _against_oracle(cfg, w, sig, _scores(cfg, w, sig), label=f"tx1536 depth {depth}")


@pytest.mark.parametrize("shape", ["512_wide_window", "1536_sup_window"])
def test_cross_shapes(tmp_path, shape):
    """Each change on its own at depth 2: sup's width with the +-256 window, and the 1536 width with sup's window."""
    if shape == "512_wide_window":
        d = config_variant(tmp_path, depth=2, d_model=512, nhead=8, ff=2048, name=shape)
    else:
        d = config_variant(tmp_path, depth=2, window=(127, 128), name=shape)
    cfg, w = _model(d)
    assert cfg.tx.attn_window == ((255, 256) if shape == "512_wide_window" else (127, 128))
    sig = _signal(cfg, 2, 7680, seed=3)
    _against_oracle(cfg, w, sig, _scores(cfg, w, sig), label=shape)


@pytest.mark.parametrize("T", [1920, 7680])
def test_full_depth_scores(T):
    """All 18 layers at N = 1: 1920 samples are 160 tokens (less than one window), 7680 are 640.  The bound is sup's
    (tests/test_forward_gpu.py): 18 layers re-round the fp16 residual stream 36 times."""
    cfg, w = _model(model_dir())
    sig = _signal(cfg, 1, T, seed=T)
    _against_oracle(cfg, w, sig, _scores(cfg, w, sig), max_frac_bad=3e-2, label=f"tx1536 18 layers, {T} samples")


def test_rmsnorm_pass(tmp_path, monkeypatch):
    """B200_TX_RMSNORM_PASS=1 (a separate rmsnorm_kernel after every sub-layer) at width 1536, depth 2."""
    cfg, w = _model(config_variant(tmp_path, depth=2, name="d2_norm"))
    sig = _signal(cfg, 2, 7680, seed=11)
    monkeypatch.setenv("B200_TX_RMSNORM_PASS", "1")
    got = _scores(cfg, w, sig)
    monkeypatch.delenv("B200_TX_RMSNORM_PASS")
    _against_oracle(cfg, w, sig, got, label="tx1536 depth 2, separate RMSNorm pass")
    assert not np.array_equal(got, _scores(cfg, w, sig))   # the option did change the path


# ---- calls, concurrency ---------------------------------------------------------------------------------------------------
def test_call_chunks_end_to_end(crf_oracle):
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _model(model_dir())
    N = 4
    caller = B200Caller(cfg, w)
    runner = B200ModelRunner(caller, N, 7680)
    sig = _signal(cfg, N, 7680, seed=21)
    for i in range(N):
        runner.accept_chunk(i, sig[i])
    scores = runner.forward_scores(N)
    chunks = runner.call_chunks(N)
    ref = crf_oracle.decode(scores, clamp_val=0.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(chunks):
        assert c.sequence == ref.sequences[i] and c.qstring == ref.qstrings[i]
        np.testing.assert_array_equal(c.moves, ref.moves[i])
        assert len(c.moves) == 7680 // cfg.stride and len(c.sequence) == int(c.moves.sum())
    assert sum(len(c.sequence) for c in chunks) > N * 50          # real calls, not empty strings
    part = runner.call_chunks(2)
    assert [(p.sequence, p.qstring, bytes(p.moves)) for p in part] == [(c.sequence, c.qstring, bytes(c.moves)) for c in chunks[:2]]
    runner.close()
    caller.close()


def test_concurrent_runners_match_serial():
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _model(model_dir())
    N, T = 4, 3840
    caller = B200Caller(cfg, w)
    runners = [B200ModelRunner(caller, N, T) for _ in range(2)]
    for k, r in enumerate(runners):
        sig = _signal(cfg, N, T, seed=40 + k)
        for i in range(N):
            r.accept_chunk(i, sig[i])
    serial = [[(c.sequence, c.qstring, bytes(c.moves)) for c in r.call_chunks(N)] for r in runners]
    assert serial[0] != serial[1]
    got = [[], []]

    def drive(i):
        for _ in range(3):
            got[i].append([(c.sequence, c.qstring, bytes(c.moves)) for c in runners[i].call_chunks(N)])

    ths = [threading.Thread(target=drive, args=(i,)) for i in range(2)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    for i in range(2):
        assert got[i] == [serial[i]] * 3
    assert B200ModelRunner.step_device_runners(runners, N, 4) > 0
    for i, r in enumerate(runners):
        assert [(c.sequence, c.qstring, bytes(c.moves)) for c in r.call_chunks(N)] == serial[i]
        r.close()
    caller.close()


# ---- shapes refused, memory -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("change", [dict(nhead=16), dict(d_model=1600, nhead=25), dict(d_model=2048, nhead=32),
                                    dict(window=(257, 256)), dict(window=(255, 257)), dict(ff=6100)])
def test_unsupported_shapes(tmp_path, change):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller
    cfg, w = _model(config_variant(tmp_path, depth=1, name="bad", **change))
    with pytest.raises(L.B200Error) as e:
        B200Caller(cfg, w)
    assert e.value.status == L.B200_ERR_UNSUPPORTED, str(e.value)


def test_chunk_beyond_max_seq_len(tmp_path):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _model(config_variant(tmp_path, depth=1, name="d1_len"))
    caller = B200Caller(cfg, w)
    B200ModelRunner(caller, 1, 24576).close()                      # 2048 tokens (12 samples each): the RoPE table's length
    with pytest.raises(L.B200Error) as e:
        B200ModelRunner(caller, 1, 24576 + 192)
    assert e.value.status == L.B200_ERR_INVALID
    caller.close()


def test_runner_bytes_is_the_arena():
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _model(model_dir())
    caller = B200Caller(cfg, w)
    want = caller.runner_bytes(128, 12288)
    before = caller.stats()["arena_bytes"]
    runner = B200ModelRunner(caller, 128, 12288)
    assert caller.stats()["arena_bytes"] - before == want
    print(f"\n[tx1536] runner of 128 x 12288 samples: {want / 2**30:.2f} GiB")
    runner.close()
    caller.close()
