"""The int8_qkv_fp8_ffn transformer precision on the GPU: the device quantiser (b200_test_quantize_act_rows) against the host
quantize_rows_f16 bit for bit, the s8 GEMM with row and column factors (lib.test_gemm_s8_scaled) against float64, every
launch of the plan against tests/tx_i8_ref.py's per-launch reference from the engine's own buffers, sup and tx1536 scores
against the int8 restatement, calls against the C decoder oracle, and the interface.  The CPU side is
tests/test_tx_i8_cpu.py.  Measured worst cases: DESIGN.md section 2."""
import time
import zlib

import numpy as np
import pytest

from conftest import CONFIG_DIR
from test_tx1536_cpu import config_variant, model_dir as tx1536_dir
from test_tx_i8_cpu import _edge_rows
import tx_i8_ref
import tx_layer_ref as X

pytestmark = pytest.mark.gpu

SUP = CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0"
PREC = "int8_qkv_fp8_ffn"
NONE, ROPE = -1, 5
U32, U11 = 2.0 ** -24, 2.0 ** -11
MARGIN = 3.0
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


def _run(cfg, w, sig, precision=PREC, num_runners=2, calls=False):
    from dorado_b200.runner import B200Caller, B200ModelRunner
    caller = B200Caller(cfg, w, num_runners=num_runners, precision=precision)
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


# ---- the device quantiser ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [128, 512, 1536])
def test_device_quantiser_matches_host(cols):
    """Every edge row of test_tx_i8_cpu._edge_rows plus random rows, 37 rows in all (a partial last block of 8 rows): q and
    inv = 1 / float(scale16) bit for bit those of the host quantize_rows_f16."""
    from dorado_b200 import lib as L
    rng = np.random.default_rng(cols)
    edge = _edge_rows(cols, rng)
    x = np.concatenate([edge, (rng.standard_normal((37 - len(edge), cols)) * 2).astype(np.float16)])
    q, inv = L.quantize_act_rows(x)
    hq, hscale = L.quantize_rows(x)
    np.testing.assert_array_equal(q, hq)
    with np.errstate(divide="ignore"):
        want = np.float32(1) / hscale.astype(np.float32)
    np.testing.assert_array_equal(inv.view(np.uint32), want.view(np.uint32))
    rq, _, rinv = tx_i8_ref.quantize_act(x)
    np.testing.assert_array_equal(q, rq)
    np.testing.assert_array_equal(inv.view(np.uint32), rinv.view(np.uint32))


def test_device_quantiser_rejects_bad_shapes():
    from dorado_b200 import lib as L
    with pytest.raises(L.B200Error) as e:
        L.quantize_act_rows(np.zeros((4, 96), np.float16))
    assert e.value.status == L.B200_ERR_INVALID


# ---- the s8 GEMM with row and column factors ---------------------------------------------------------------------------
# (N, K) of sup's and tx1536's QKV projection
GEMM_SHAPES = {"sup_qkv": (1536, 512), "tx1536_qkv": (4608, 1536)}


def _operands(M, N, K, seed):
    """int8 A and W with the factors the quantiser gives random fp16 rows; A's first row and W's first two rows at +-127
    so that |acc| passes 2^24 at K 1536 (float32(acc) rounds there)."""
    rng = np.random.default_rng(seed)
    qa, _, ia = tx_i8_ref.quantize_act((rng.standard_normal((M, K)) * 3).astype(np.float16))
    qw, _, iw = tx_i8_ref.quantize_act((rng.standard_normal((N, K)) * 0.04).astype(np.float16))
    qa[0] = 127
    qw[:2] = 127
    qw[1, 0] = 126
    return qa, ia, qw, iw


@pytest.mark.parametrize("shape", list(GEMM_SHAPES))
@pytest.mark.parametrize("M", [1, 200, 333])
def test_gemm_s8_scaled_plain(shape, M):
    """fp16(v) with v = (float32(acc) * row factor) * column factor: within one fp16 ulp of the fp32 chain restated in
    numpy, and within 3 2^-24 |v| + the fp16 rounding of the float64 value."""
    from dorado_b200 import lib as L
    N, K = GEMM_SHAPES[shape]
    qa, ia, qw, iw = _operands(M, N, K, M * 7 + K)
    got = L.test_gemm_s8_scaled(qa, qw, ia, iw, NONE)
    chain = tx_i8_ref.s8_product(qa, ia, qw, iw).astype(np.float16)
    ulps = np.abs(got.view(np.int16).astype(np.int32) - chain.view(np.int16).astype(np.int32))
    v = (qa.astype(np.int64) @ qw.astype(np.int64).T).astype(np.float64) * ia[:, None] * iw[None, :]
    ratio = np.abs(got.astype(np.float64) - v) / (3 * U32 * np.abs(v) + U11 * np.abs(v) + 2.0 ** -25)
    print(f"\n[{shape} M={M}] {int((ulps > 0).sum())} outputs differ from the fp32 chain (max {ulps.max()} ulp); worst "
          f"error {ratio.max():.3f} of the float64 bound; max |acc| {np.abs(v / ia[:, None] / iw[None, :]).max():.3g}")
    assert ulps.max() <= 1 and ratio.max() <= 1.0


@pytest.mark.parametrize("shape", list(GEMM_SHAPES))
@pytest.mark.parametrize("M", [1, 200, 333])
def test_gemm_s8_scaled_rope(shape, M):
    """The RoPE epilogue on v at position m % rope_T over the q and k columns, against float64 with tests/gemm_ref.py's
    RoPE bound (tx_layer_ref._rope) on top of the s8 conversion's 3 2^-24 |v| and the fp16 output."""
    from dorado_b200 import lib as L
    N, K = GEMM_SHAPES[shape]
    qa, ia, qw, iw = _operands(M, N, K, M * 11 + K)
    rope_T, theta = 96, 10000.0
    got = L.test_gemm_s8_scaled(qa, qw, ia, iw, ROPE, theta=theta, max_seq_len=2048, rope_T=rope_T, rope_cols=2 * N // 3)
    v = (qa.astype(np.int64) @ qw.astype(np.int64).T).astype(np.float64) * ia[:, None] * iw[None, :]
    ref, bound = X._out16(*X._rope(v, 3 * U32 * np.abs(v), np.arange(M) % rope_T, theta, 2 * N // 3))
    ratio = np.abs(got.astype(np.float64) - ref) / bound
    print(f"\n[{shape} RoPE M={M}] worst error {ratio.max():.3f} of the bound")
    assert ratio.max() <= 1.0


def test_gemm_s8_scaled_rejects_other_epilogues():
    from dorado_b200 import lib as L
    z = np.zeros((128, 128), np.int8)
    one = np.ones(128, np.float32)
    with pytest.raises(L.B200Error) as e:
        L.test_gemm_s8_scaled(z, z, one, one, 4)   # SwiGLU
    assert e.value.status == L.B200_ERR_INVALID


# ---- every launch of the plan ------------------------------------------------------------------------------------------
# name: (model, depth, N, samples per chunk)
CASES = {
    # 992 tokens: a ragged last query tile; chunk boundaries inside GEMM row tiles (RoPE at g % T)
    "sup": ("sup", 3, 3, 11904),
    # 640 tokens: five key blocks per query tile, K 1536 (|acc| beyond 2^24 possible), fc2's K 6144
    "tx1536": ("tx1536", 2, 1, 7680),
}
_stats = {}
_sensitivity = {}


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if _stats:
        print("\n[int8_qkv_fp8_ffn launches vs float64 reference] worst error / bound per launch kind:")
        for kind, r in sorted(_stats.items()):
            print(f"  {kind:18s} {r:.3f}")
    if _sensitivity:
        print("[int8_qkv_fp8_ffn launches] simulated mistakes, least worst ratio over the cases (must be >= 3):")
        for m, r in sorted(_sensitivity.items()):
            print(f"  {m:24s} {r:.1f}")


def _config(tmp_path, model, depth):
    from dorado_b200.config import load_model_config
    return load_model_config(_sup_variant(tmp_path, depth) if model == "sup" else
                             config_variant(tmp_path, depth=depth, name=f"tx1536_d{depth}"))


def _check_int8_copy(L, cur, rows, dm, what):
    x = cur["x"].view(np.float16).reshape(rows, dm)
    hq, hscale = L.quantize_rows(x)
    with np.errstate(divide="ignore"):
        want_inv = np.float32(1) / hscale.astype(np.float32)
    assert np.array_equal(cur["x8"].view(np.int8).reshape(rows, dm), hq), f"{what}: x8 is not quantize_rows_f16 of x"
    assert np.array_equal(cur["x_inv"].view(np.uint32), want_inv.view(np.uint32)), f"{what}: x_inv is not 1 / scale16"


@pytest.mark.parametrize("case", list(CASES))
def test_every_launch(tmp_path, monkeypatch, case):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    t0 = time.time()
    model, depth, N, T_in = CASES[case]
    cfg = _config(tmp_path, model, depth)
    assert cfg.normalise_chunk_size(T_in) == T_in
    w = synthetic_weights(cfg, 42)
    caller = B200Caller(cfg, w, precision=PREC)
    ref = tx_i8_ref.I8LayerRef(cfg, w, N, T_in)
    lay = ref.lay
    rows, dm = lay["rows"], cfg.tx.d_model
    plan = tx_i8_ref.launches(cfg)
    n = len(plan)
    assert n == tx_i8_ref.launch_count(cfg)
    sig = np.random.default_rng(zlib.crc32(case.encode())).standard_normal((N, T_in)).astype(np.float16)

    def snapshot(k):
        if k < n:
            monkeypatch.setenv("B200_DEBUG_TX_LAUNCHES", str(k))
        else:
            monkeypatch.delenv("B200_DEBUG_TX_LAUNCHES", raising=False)
        runner = B200ModelRunner(caller, N, T_in)
        try:
            for i in range(N):
                runner.accept_chunk(i, sig[i])
            scores = runner.forward_scores(N).astype(np.float64)
            ws = runner.debug_read_workspace(0, lay["bytes"])
            extra = {}
            if k == 0:
                with pytest.raises(L.B200Error):   # the layout's size is the workspace's
                    runner.debug_read_workspace(0, lay["bytes"] + 1)
                extra["info"] = runner.plan_info()
            if k in (3, n):
                extra["profile"] = [name for name, _ in runner.profile(N)]
        finally:
            runner.close()
            monkeypatch.delenv("B200_DEBUG_TX_LAUNCHES", raising=False)
        return {name: ws[off:off + nb] for name, (off, nb) in lay["buffers"].items()}, scores, extra

    prev, _, extra0 = snapshot(0)
    assert extra0["info"] == {"tx.fp8_ffn": 1, "tx.int8_qkv": 1}
    assert all((b == 0).all() for b in prev.values()), "the workspace is not all zero before the first launch"
    worst, short = {}, []
    for k in range(1, n + 1):
        name, kind, idx = plan[k - 1]
        cur, scores, extra = snapshot(k)
        if "profile" in extra:
            names = extra["profile"]
            assert names[:k] == [p[0] for p in plan[:k]], names[:k + 1]
            if k < n:
                assert len(names) == k or names[k] not in {p[0] for p in plan}, names[:k + 1]
        written = tx_i8_ref.writes(cfg, lay, kind, idx)
        for buf, b in cur.items():
            if buf in written:
                if written[buf] is not None:
                    lo, hi = written[buf]
                    assert np.array_equal(b[hi:], prev[buf][hi:]), f"launch {k} ({name}) wrote {buf} beyond its range"
                continue
            assert np.array_equal(b, prev[buf]), \
                f"launch {k} ({name}): {buf} changed, which it does not write (a stray write, or an earlier launch is not deterministic)"
        for i in range(len(cfg.convs) - 1):
            assert X.cbuf_padding_nonzero(cfg, lay, cur, i) == 0, f"launch {k} ({name}): padding rows of cbuf{i} not zero"
        if kind == "quantize":
            _check_int8_copy(L, cur, rows, dm, f"launch {k} ({name})")
            prev = cur
            continue
        inp = tx_i8_ref.logical_inputs(cfg, lay, prev)
        inp["signal"] = sig.astype(np.float64)
        got_all = tx_i8_ref.logical_inputs(cfg, lay, cur)
        got_all["scores"] = scores
        for out, (r, bnd) in ref.reference(kind, idx, inp).items():
            if out == "hid8":
                ff = cfg.tx.dim_feedforward
                outside, ratio = X.e4m3_cast_check(cur["hid"][:rows * ff].reshape(-1, ff), r, bnd)
                assert outside == 0, f"launch {k} ({name}): {outside} E4M3 outputs outside the casts of their interval"
                wr = float(ratio.max())
            else:
                got = got_all[out]
                assert np.isfinite(got).all(), f"launch {k} ({name}): non-finite {out}"
                wr = X.worst_ratio(got, r, bnd)
                assert wr <= 1.0, f"launch {k} ({name}) {out}: worst error {wr:.3f} of the bound"
            _stats[kind] = max(_stats.get(kind, 0.0), wr)
            worst[f"{k}:{name}"] = wr
        if kind == "norm1":
            want = X.e4m3_sat_bytes(cur["att"].view(np.float16).astype(np.float32))
            assert np.array_equal(cur["qkv"][:rows * dm], want), f"launch {k}: the E4M3 copy is not the cast of the fp16 output"
        if kind == "norm2":
            _check_int8_copy(L, cur, rows, dm, f"launch {k} ({name})")
        for m, mk in tx_i8_ref.MUTATIONS.items():
            if mk != kind or idx != 1:
                continue
            (out, (r, bnd)), = ref.reference(kind, idx, inp, mutation=m).items()
            mr = X.worst_ratio(got_all[out], r, np.abs(bnd))
            print(f"\n  [{case}] {m} at launch {k} ({name}): worst ratio {mr:.1f}")
            _sensitivity[m] = min(_sensitivity.get(m, np.inf), mr)
            if mr < MARGIN:
                short.append(f"{m}: the mistake reaches only {mr:.2f} bounds")
        prev = cur
    print(f"\n[{case}] {n} launches, worst ratio {max(worst.values()):.3f} ({max(worst, key=worst.get)}), "
          f"{time.time() - t0:.0f} s")
    caller.close()
    assert not short, short


# ---- model scores ------------------------------------------------------------------------------------------------------
# Engine against the int8 restatement.  Both quantise fp16 rows that can differ in their last bit (fp32 sums in another
# order), and where such a value straddles a rounding tie its int8 moves by one level: absmax / 128, at most 2^-7 of the
# row's largest value, against the 2^-4 relative step of an E4M3 activation flip that fp8_ffn already has.  So fp8_ffn's
# bounds against its own restatement (tests/test_tx_fp8_gpu.py) are kept.  Measured worst cases: DESIGN.md section 2.
SCORE_BOUNDS = {"p99": 1e-2, "max": 2e-2, "rel_l2": 1.5e-2}


def _against_i8_restatement(cfg, w, sig, got, label):
    ref = tx_i8_ref.forward(cfg, w, sig.astype(np.float32))
    assert got.shape == ref.shape
    scale = max(1.0, float(np.abs(ref).max()))
    err = np.abs(got.astype(np.float32) - ref) / scale
    p50, p99, p999 = np.percentile(err, [50, 99, 99.9])
    rel_l2 = float(np.linalg.norm(got.astype(np.float32) - ref) / np.linalg.norm(ref))
    print(f"\n[{label}] vs int8 restatement (x max|ref|): p50 {p50:.2e}, p99 {p99:.2e}, p99.9 {p999:.2e}, "
          f"max {err.max():.2e}; relative L2 {rel_l2:.2e}")
    assert np.isfinite(got).all()
    assert p99 <= SCORE_BOUNDS["p99"] and err.max() <= SCORE_BOUNDS["max"] and rel_l2 <= SCORE_BOUNDS["rel_l2"]


@pytest.mark.parametrize("model,depth,N,T", [("sup", 1, 3, 3840), ("sup", 2, 2, 7680), ("tx1536", 1, 2, 3840),
                                             ("tx1536", 2, 1, 7680)])
def test_reduced_depth_scores(tmp_path, model, depth, N, T):
    d = _sup_variant(tmp_path, depth) if model == "sup" else config_variant(tmp_path, depth=depth, name=f"d{depth}")
    cfg, w = _model(d)
    sig = _signal(cfg, N, T, seed=depth + N)
    got, _, info = _run(cfg, w, sig)
    assert info == {"tx.fp8_ffn": 1, "tx.int8_qkv": 1}
    _against_i8_restatement(cfg, w, sig, got, f"{model} depth {depth}, N {N}, {T} samples")


@pytest.mark.parametrize("model,N,T", [("sup", 2, 1920), ("sup", 1, 7680), ("tx1536", 1, 3840)])
def test_full_depth_scores(model, N, T):
    cfg, w = _model(SUP if model == "sup" else tx1536_dir())
    sig = _signal(cfg, N, T, seed=T)
    got, _, _ = _run(cfg, w, sig)
    _against_i8_restatement(cfg, w, sig, got, f"{model} full depth, N {N}, {T} samples")


@pytest.mark.parametrize("model", ["sup", "tx1536"])
def test_calls_match_decoder_oracle(model, crf_oracle):
    """Calls of the int8 scores through the C decoder oracle; and how far they move from fp8_ffn's (printed)."""
    from conftest import edit_distance
    cfg, w = _model(SUP if model == "sup" else tx1536_dir())
    sig = _signal(cfg, 8, 3840, seed=77)
    s8, c8, _ = _run(cfg, w, sig, calls=True)
    ref = crf_oracle.decode(s8, clamp_val=5.0 if cfg.clamp else 0.0, q_shift=cfg.qbias, q_scale=cfg.qscale)
    for i, c in enumerate(c8):
        assert c.sequence == ref.sequences[i] and c.qstring == ref.qstrings[i], f"chunk {i}"
        np.testing.assert_array_equal(c.moves, ref.moves[i])
    sf, cf, _ = _run(cfg, w, sig, precision="fp8_ffn", calls=True)
    rel_l2 = float(np.linalg.norm(s8.astype(np.float32) - sf) / np.linalg.norm(sf.astype(np.float32)))
    edit = sum(edit_distance(a.sequence.encode(), b.sequence.encode()) for a, b in zip(c8, cf)) / sum(len(c.sequence) for c in cf)
    print(f"\n[{model}] int8_qkv_fp8_ffn vs fp8_ffn engine: score relative L2 {rel_l2:.3e}, edit distance {edit:.4f} per base")
    assert 0 < rel_l2 <= 0.1 and sum(len(c.sequence) for c in c8) > 8 * 50


# ---- interface ---------------------------------------------------------------------------------------------------------
def test_independent_of_runners_and_batch_shape():
    cfg, w = _model(tx1536_dir())
    sig = _signal(cfg, 5, 3840, seed=9)
    a, _, _ = _run(cfg, w, sig, num_runners=1)
    b, _, _ = _run(cfg, w, sig, num_runners=4)
    np.testing.assert_array_equal(a, b)
    c, _, _ = _run(cfg, w, sig[1:3])   # the same chunks in a batch of two: other row tiles, other grid
    np.testing.assert_array_equal(a[1:3], c)


def test_fp16_and_fp8_unchanged_beside_int8(tmp_path):
    """fp16 and fp8_ffn give the same scores before and after an int8_qkv_fp8_ffn model has run in the same process, and
    fp16 still reports no plan keys."""
    cfg, w = _model(_sup_variant(tmp_path, 2))
    sig = _signal(cfg, 3, 3840, seed=21)
    before = {p: _run(cfg, w, sig, precision=p) for p in ("fp16", "fp8_ffn")}
    _run(cfg, w, sig)
    for p, (s, _, info) in before.items():
        again, _, info2 = _run(cfg, w, sig, precision=p)
        np.testing.assert_array_equal(s, again)
        assert info == info2 == ({} if p == "fp16" else {"tx.fp8_ffn": 1})


def test_int8_qkv_on_lstm_model_is_an_error():
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller
    cfg, w = _model(CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_fast@v5.0.0")
    with pytest.raises(L.B200Error) as e:
        B200Caller(cfg, w, precision=PREC)
    assert e.value.status == L.B200_ERR_INVALID and "transformer models only" in str(e.value)


def test_int8_qkv_rejects_ff_not_multiple_of_128(tmp_path):
    from dorado_b200 import lib as L
    from dorado_b200.runner import B200Caller
    cfg, w = _model(config_variant(tmp_path, depth=1, ff=64, name="ff64"))
    B200Caller(cfg, w).close()                                   # fp16 takes it (a multiple of 64)
    with pytest.raises(L.B200Error) as e:
        B200Caller(cfg, w, precision=PREC)
    assert e.value.status == L.B200_ERR_UNSUPPORTED and "multiple of 128" in str(e.value)
