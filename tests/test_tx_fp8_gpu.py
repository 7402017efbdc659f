"""The fp8_ffn transformer precision on the GPU: the E4M3 GEMM alone (lib.test_gemm_fp8) against float64 products of the
decoded operands, sup and tx1536 scores against the FP8-emulating oracle (tests/tx_fp8_ref.py), calls against the C decoder
oracle, FP8 against fp16 on the same batch, the default precision against an explicit fp16, independence of the runner
count and batch shape, and the error paths.  The CPU side is tests/test_tx_fp8_cpu.py."""
import numpy as np
import pytest

from conftest import CONFIG_DIR, edit_distance
from test_tx1536_cpu import config_variant, model_dir as tx1536_dir
import tx_fp8_ref

pytestmark = pytest.mark.gpu

SUP = CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0"
SWIGLU, NONE = 4, -1
_cache = {}


def _model(path, seed=42):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    key = (str(path), seed)
    if key not in _cache:
        cfg = load_model_config(path)
        _cache[key] = (cfg, synthetic_weights(cfg, seed))
    return _cache[key]


def _sup_variant(tmp_path, depth):
    text = (SUP / "config.toml").read_text()
    assert text.count("depth = 18\n") == 1
    d = tmp_path / f"sup_d{depth}"
    d.mkdir()
    (d / "config.toml").write_text(text.replace("depth = 18\n", f"depth = {depth}\n"))
    return d


def _signal(cfg, N, T, seed):
    return np.random.default_rng(seed).standard_normal((N, cfg.normalise_chunk_size(T))).astype(np.float16)


def _run(cfg, w, sig, precision="fp8_ffn", num_runners=2, calls=False):
    from dorado_b200.runner import B200Caller, B200ModelRunner
    caller = B200Caller(cfg, w, num_runners=num_runners, **({} if precision is None else {"precision": precision}))
    N, T = sig.shape
    runner = B200ModelRunner(caller, N, T)
    for i in range(N):
        runner.accept_chunk(i, sig[i])
    scores = runner.forward_scores(N).copy()
    info = runner.plan_info()
    chunks = runner.call_chunks(N) if calls else None
    runner.close()
    caller.close()
    return scores, chunks, info


# ---- the E4M3 GEMM alone -----------------------------------------------------------------------------------------------
def _e4m3_operand(rng, shape, scale):
    return tx_fp8_ref.e4m3_bytes(rng.standard_normal(shape).astype(np.float32) * scale)


# (N, K) of sup's and tx1536's fc1 (N = 2 ff, K = d_model) and fc2 (N = d_model, K = ff)
GEMM_SHAPES = {"sup_fc1": (4096, 512), "sup_fc2": (512, 2048), "tx1536_fc1": (12288, 1536), "tx1536_fc2": (1536, 6144)}


def _fp32_bound(a, b):
    """fp32 accumulation of K products: |error| <= K u sum_k |a_k b_k| (u = 2^-24), per output."""
    return a.shape[1] * 2.0 ** -24 * (np.abs(a) @ np.abs(b).T)


def _accum_bound(a, b):
    """The E4M3 wgmma accumulation as measured: an error of up to 2^-14 of sum |a b| per k32 step, so (K / 32) 2^-14
    sum_k |a_k b_k|.  The tensor cores do not accumulate E4M3 products in full fp32: on an H100 the plain GEMM's worst
    error was 7.7 x the fp32 bound above and 0.38 of this one (DESIGN.md section 2)."""
    return a.shape[1] / 32 * 2.0 ** -14 * (np.abs(a) @ np.abs(b).T)


@pytest.mark.parametrize("shape", list(GEMM_SHAPES))
@pytest.mark.parametrize("M", [1, 200, 333])
def test_gemm_fp8_plain(shape, M):
    """c = A W^T + alpha * residual in fp16 against float64, for M not a multiple of the 128-row tile: the E4M3 wgmma
    accumulation bound plus the fp16 rounding of the output (2^-11 relative).  Prints the error against the fp32 bound too."""
    from dorado_b200 import lib as L
    N, K = GEMM_SHAPES[shape]
    rng = np.random.default_rng(M * 7 + K)
    a8, b8 = _e4m3_operand(rng, (M, K), 1.0), _e4m3_operand(rng, (N, K), 0.05)
    a, b = tx_fp8_ref.decode_e4m3(a8).astype(np.float64), tx_fp8_ref.decode_e4m3(b8).astype(np.float64)
    res = rng.standard_normal((M, N)).astype(np.float16)
    alpha = 2.4494897
    for residual in (None, res):
        got = L.test_gemm_fp8(a8, b8, NONE, residual, alpha if residual is not None else 0.0).astype(np.float64)
        ref = a @ b.T + (alpha * res.astype(np.float64) if residual is not None else 0.0)
        bound = _accum_bound(a, b) + 2.0 ** -11 * np.abs(ref) + 1e-30
        ratio = np.abs(got - ref) / bound
        r32 = (np.abs(got - ref) / (_fp32_bound(a, b) + 2.0 ** -11 * np.abs(ref) + 1e-30)).max()
        print(f"\n[{shape} M={M} residual={residual is not None}] worst error {ratio.max():.3f} of the bound, "
              f"{r32:.3f} of the fp32 bound")
        assert ratio.max() <= 1.0


@pytest.mark.parametrize("shape", ["sup_fc1", "tx1536_fc1"])
@pytest.mark.parametrize("M", [1, 200, 333])
def test_gemm_fp8_swiglu(shape, M):
    """E4M3 y * silu(gate) against the float64 value v: the output must be the saturating E4M3 cast of some value within
    the accumulation bound (plus swish_fast's 1e-5 relative) of v, so it differs from the cast of v only where v lies
    that close to a rounding tie.  With the E4M3 accumulation's error that is 0.5-1.7 % of the outputs (printed)."""
    from dorado_b200 import lib as L
    N, K = GEMM_SHAPES[shape]
    rng = np.random.default_rng(M * 13 + K)
    a8, b8 = _e4m3_operand(rng, (M, K), 1.0), _e4m3_operand(rng, (N, K), 0.05)
    a, b = tx_fp8_ref.decode_e4m3(a8).astype(np.float64), tx_fp8_ref.decode_e4m3(b8).astype(np.float64)
    got = L.test_gemm_fp8(a8, b8, SWIGLU)
    t = a @ b.T
    bt = _accum_bound(a, b)
    y, gate = t[:, 0::2], t[:, 1::2]
    v = y * gate / (1.0 + np.exp(-gate))
    tol = np.abs(gate / (1.0 + np.exp(-gate))) * bt[:, 0::2] + np.abs(y) * 1.2 * bt[:, 1::2] + 1e-5 * np.abs(v)
    want = tx_fp8_ref.e4m3_bytes(np.clip(v, -448, 448).astype(np.float32))
    assert got.shape == want.shape == (M, N // 2)
    gv = tx_fp8_ref.decode_e4m3(got)
    cast = lambda x: tx_fp8_ref.decode_e4m3(tx_fp8_ref.e4m3_bytes(np.clip(x, -448, 448).astype(np.float32)))
    lo, hi = cast(v - tol), cast(v + tol)                  # rounding is monotone: the casts of [v - tol, v + tol]
    differ = int((gv != tx_fp8_ref.decode_e4m3(want)).sum())
    outside = (gv < lo) | (gv > hi)
    print(f"\n[{shape} SwiGLU M={M}] {differ} of {got.size} outputs differ from the cast of the float64 value, "
          f"{int(outside.sum())} outside the casts of its error interval")
    assert not outside.any()


def test_gemm_fp8_rejects_other_epilogues():
    from dorado_b200 import lib as L
    z = np.zeros((128, 128), np.uint8)
    with pytest.raises(L.B200Error) as e:
        L.test_gemm_fp8(z, z, 0)   # swish
    assert e.value.status == L.B200_ERR_INVALID


# ---- model scores ------------------------------------------------------------------------------------------------------
# Engine against the FP8-emulating oracle.  An E4M3 activation is 3 mantissa bits: where the engine's fp32 sums and the
# oracle's differ in the last bits and straddle a rounding tie, one activation moves by a whole E4M3 step (1/16 relative),
# so the agreement is looser than the fp16 path's.  Bounds: the first measured run's worst values with a margin (printed).
# Measured on an H100 (worst of the cases below): p99 4.3e-3, p99.9 5.5e-3, max 8.8e-3 x max|ref|, relative L2 6.4e-3.
SCORE_BOUNDS = {"p99": 1e-2, "max": 2e-2, "rel_l2": 1.5e-2}


def _against_fp8_oracle(cfg, w, sig, got, label):
    ref = tx_fp8_ref.forward(cfg, w, sig.astype(np.float32))
    assert got.shape == ref.shape
    scale = max(1.0, float(np.abs(ref).max()))
    err = np.abs(got.astype(np.float32) - ref) / scale
    p50, p99, p999 = np.percentile(err, [50, 99, 99.9])
    rel_l2 = float(np.linalg.norm(got.astype(np.float32) - ref) / np.linalg.norm(ref))
    print(f"\n[{label}] vs FP8 oracle (x max|ref|): p50 {p50:.2e}, p99 {p99:.2e}, p99.9 {p999:.2e}, max {err.max():.2e}; "
          f"relative L2 {rel_l2:.2e}")
    assert np.isfinite(got).all()
    assert p99 <= SCORE_BOUNDS["p99"] and err.max() <= SCORE_BOUNDS["max"] and rel_l2 <= SCORE_BOUNDS["rel_l2"]


@pytest.mark.parametrize("model,depth,N,T", [("sup", 1, 3, 3840), ("sup", 2, 2, 7680), ("tx1536", 1, 2, 3840),
                                             ("tx1536", 2, 1, 7680)])
def test_reduced_depth_scores(tmp_path, model, depth, N, T):
    d = _sup_variant(tmp_path, depth) if model == "sup" else config_variant(tmp_path, depth=depth, name=f"d{depth}")
    cfg, w = _model(d)
    sig = _signal(cfg, N, T, seed=depth + N)
    got, _, info = _run(cfg, w, sig)
    assert info == {"tx.fp8_ffn": 1}
    _against_fp8_oracle(cfg, w, sig, got, f"{model} depth {depth}, N {N}, {T} samples")


@pytest.mark.parametrize("model,N,T", [("sup", 2, 1920), ("sup", 1, 7680), ("tx1536", 1, 3840)])
def test_full_depth_scores(model, N, T):
    cfg, w = _model(SUP if model == "sup" else tx1536_dir())
    sig = _signal(cfg, N, T, seed=T)
    got, _, _ = _run(cfg, w, sig)
    _against_fp8_oracle(cfg, w, sig, got, f"{model} full depth, N {N}, {T} samples")


# ---- calls, FP8 against fp16 ------------------------------------------------------------------------------------------
# Same batch (8 chunks of 3840 samples), both precisions, full depth.  Measured on an H100: score relative L2 2.6e-2 (sup)
# and 2.9e-2 (tx1536); identical sequences 0 of 8 (sup, about 540 bases each) and 5 of 8 (tx1536).  Gated with a margin.
# Synthetic weights say little about basecall accuracy (DESIGN.md section 2).
FP8_VS_FP16_REL_L2 = 0.05
FP8_VS_FP16_MIN_IDENTICAL = {"sup": 0.0, "tx1536": 0.25}
FP8_VS_FP16_MAX_EDIT = 0.05   # mean edit distance per fp16 base


@pytest.mark.parametrize("model", ["sup", "tx1536"])
def test_calls_match_decoder_oracle_and_fp16(model, crf_oracle):
    cfg, w = _model(SUP if model == "sup" else tx1536_dir())
    sig = _signal(cfg, 8, 3840, seed=77)
    s8, c8, _ = _run(cfg, w, sig, calls=True)
    ref = crf_oracle.decode(s8, clamp_val=5.0 if cfg.clamp else 0.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(c8):
        assert c.sequence == ref.sequences[i] and c.qstring == ref.qstrings[i], f"chunk {i}"
        np.testing.assert_array_equal(c.moves, ref.moves[i])
    s16, c16, info16 = _run(cfg, w, sig, precision="fp16", calls=True)
    assert info16 == {}
    rel_l2 = float(np.linalg.norm(s8.astype(np.float32) - s16) / np.linalg.norm(s16.astype(np.float32)))
    same = float(np.mean([a.sequence == b.sequence for a, b in zip(c8, c16)]))
    edit = sum(edit_distance(a.sequence.encode(), b.sequence.encode()) for a, b in zip(c8, c16)) / sum(len(c.sequence) for c in c16)
    print(f"\n[{model}] FP8 vs fp16 engine: score relative L2 {rel_l2:.3e}, identical sequences {same:.2f}, edit distance "
          f"{edit:.4f} per base, bases {sum(len(c.sequence) for c in c8)} / {sum(len(c.sequence) for c in c16)}")
    assert 0 < rel_l2 <= FP8_VS_FP16_REL_L2 and same >= FP8_VS_FP16_MIN_IDENTICAL[model] and edit <= FP8_VS_FP16_MAX_EDIT
    assert sum(len(c.sequence) for c in c8) > 8 * 50


def test_default_precision_is_fp16():
    cfg, w = _model(SUP)
    sig = _signal(cfg, 4, 3840, seed=3)
    d, cd, _ = _run(cfg, w, sig, precision=None, calls=True)
    e, ce, _ = _run(cfg, w, sig, precision="fp16", calls=True)
    np.testing.assert_array_equal(d, e)
    assert [(c.sequence, c.qstring, bytes(c.moves)) for c in cd] == [(c.sequence, c.qstring, bytes(c.moves)) for c in ce]


def test_fp8_independent_of_runners_and_batch_shape():
    cfg, w = _model(tx1536_dir())
    sig = _signal(cfg, 5, 3840, seed=9)
    a, _, _ = _run(cfg, w, sig, num_runners=1)
    b, _, _ = _run(cfg, w, sig, num_runners=4)
    np.testing.assert_array_equal(a, b)
    c, _, _ = _run(cfg, w, sig[1:3])   # the same chunks in a batch of two: other row tiles, other grid
    np.testing.assert_array_equal(a[1:3], c)


# ---- errors ------------------------------------------------------------------------------------------------------------
def test_fp8_on_lstm_model_is_an_error():
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller
    cfg, w = _model(CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_fast@v5.0.0")
    with pytest.raises(L.B200Error) as e:
        B200Caller(cfg, w, precision="fp8_ffn")
    assert e.value.status == L.B200_ERR_INVALID and "transformer models only" in str(e.value)
    with pytest.raises(ValueError):
        B200Caller(cfg, w, precision="fp8")


def test_fp8_rejects_ff_not_multiple_of_128(tmp_path):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller
    cfg, w = _model(config_variant(tmp_path, depth=1, ff=6208, name="ff6208"))
    B200Caller(cfg, w).close()                                   # fp16 takes it (a multiple of 64)
    with pytest.raises(L.B200Error) as e:
        B200Caller(cfg, w, precision="fp8_ffn")
    assert e.value.status == L.B200_ERR_UNSUPPORTED and "multiple of 128" in str(e.value)
    cfg, w = _model(config_variant(tmp_path, depth=1, nhead=16, name="bad_heads"))
    with pytest.raises(L.B200Error) as e:                        # what fp16 refuses stays refused
        B200Caller(cfg, w, precision="fp8_ffn")
    assert e.value.status == L.B200_ERR_UNSUPPORTED
