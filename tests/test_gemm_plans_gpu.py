"""The fp16 wgmma GEMM (dorado_b200/csrc/gemm.cu) in every form the model plans launch it, through b200_test_gemm_desc,
against the float64 reference and per-element bound of tests/gemm_ref.py.  Every case starts from an output buffer filled
with a sentinel and checks the whole buffer: nothing written outside the logical output, nothing left unwritten inside it.
The conv cases fill the A elements no window covers with NaN, so a read of them shows in the output.  Each test prints its
worst error as a fraction of the bound.  The case builders are shared with tests/test_gemm_plans_cpu.py, which shows on
these same inputs that each check fails for a wrong kernel.  Last, a d_model 128 transformer end to end."""
from __future__ import annotations

import dataclasses
import zlib

import numpy as np
import pytest

import gemm_ref as R

pytestmark = pytest.mark.gpu

ALPHA = 2.4494897   # sup's deepnorm_alpha
THETA = 10000.0
MAX_SEQ = 2048


@dataclasses.dataclass
class Case:
    label: str
    d: dict                     # descriptor fields (gemm_ref's keys; K and N come from w when launched)
    a: np.ndarray               # flat fp16
    w: np.ndarray               # [N, K] fp16
    out_len: int
    inputs: dict = dataclasses.field(default_factory=dict)   # bias, residual, res_gain, a_ss, res_ss, alpha
    sample: np.ndarray | None = None                         # rows checked against the reference (None: every row)
    out_ss: bool = False


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def _f16(rng, shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float16)


def _sample(rows, n=512, seed=0):
    """At most n rows, always with the first and last rows of the buffer."""
    if rows <= n:
        return None
    pick = np.random.default_rng(seed).choice(rows, n - 2, replace=False)
    return np.unique(np.concatenate([pick, [0, rows - 1]])).astype(np.int64)


def _dense(label, rng, rows, K, N, act=R.ACT_NONE, *, bias=True, a_inner=0, a_scale=1.0, w_scale=None, **d):
    """A row-major [rows][a_inner or K] A, contiguous output of n_out columns."""
    inner = a_inner or K
    w_scale = w_scale or 1.0 / np.sqrt(inner)
    desc = dict(rows_per_batch=rows, a_row_stride=inner, a_batch_stride=rows * inner, a_inner=a_inner, K=K, N=N, act=act,
                out_s0=N // 2 if act == R.ACT_SWIGLU else N, **d)
    inputs = {"bias": (rng.standard_normal(N) * 0.1).astype(np.float32)} if bias else {}
    return Case(label, desc, _f16(rng, rows * inner, a_scale), _f16(rng, (N, K), w_scale), rows * R.n_out(desc), inputs,
                _sample(rows))


def _nan_uncovered(case):
    case.a = case.a.copy()
    case.a[~R.covered_a(case.d, case.a.size)] = np.float16(np.nan)
    return case


# ---- the LSTM models ---------------------------------------------------------------------------------------------------
def lstm_conv3(C, chunks, T_in, act, winlen=19, stride=6):
    """conv3 (lstm_model.cu make_plan): im2col rows of the NTC buffer x2 [N][Tp][16] with row stride stride * 16 < K,
    K = 19 * 16 = 304 padded to 320 with zero W columns, output TNC into seq [T_out + 1][Np][C]."""
    rng = _rng("conv3", C)
    Tp, T_out, Np = T_in + 2 * (winlen // 2) + 8, T_in // stride, (chunks + 31) // 32 * 32
    K3 = winlen * 16
    K = (K3 + 63) // 64 * 64
    w = np.zeros((C, K), np.float16)
    w[:, :K3] = _f16(rng, (C, K3), 1.0 / np.sqrt(K3))
    d = dict(batches=chunks, rows_per_batch=T_out, a_row_stride=stride * 16, a_batch_stride=Tp * 16, K=K, N=C, act=act,
             out_m1=T_out, out_s0=C, out_s1=Np * C)
    case = Case(f"conv3 C={C}", d, _f16(rng, chunks * Tp * 16), w, (T_out + 1) * Np * C,
                {"bias": (rng.standard_normal(C) * 0.1).astype(np.float32)}, _sample(chunks * T_out))
    return _nan_uncovered(case)


def lstm_xproj(C, T=100, Np=64, max_ctas=0):
    """The x-projection: rows (t, chunk) of the sequence buffer, A's extent C < K: W's K padding columns are NOT zero
    here, so a kernel that read the next row instead of the tensor map's zeros would be wrong."""
    return _dense(f"xproj C={C} max_ctas={max_ctas}", _rng("xproj", C), T * Np, (C + 63) // 64 * 64, 4 * C, a_inner=C,
                  max_ctas=max_ctas)


def lstm_crf(C, T_out, Np, outsize, act, a_inner=True, label="crf"):
    """The CRF linear (or the second of two): rows g = t * Np + n, written to scores[n][t][:]."""
    rng = _rng(label, C, act)
    K = (C + 63) // 64 * 64
    rows = T_out * Np
    w = np.zeros((outsize, K), np.float16)
    w[:, :C] = _f16(rng, (outsize, C), 1.0 / np.sqrt(C))
    d = dict(rows_per_batch=rows, a_row_stride=C, a_batch_stride=rows * C, a_inner=C if a_inner else 0, K=K, N=outsize,
             act=act, out_m1=Np, out_s0=outsize, out_s1=T_out * outsize)
    return Case(f"{label} C={C} act={act}", d, _f16(rng, rows * C), w, Np * T_out * outsize,
                {"bias": (rng.standard_normal(outsize) * 0.1).astype(np.float32)}, _sample(rows))


# ---- the transformer ----------------------------------------------------------------------------------------------------
SUP_CONVS = [(1, 64, 5, 1), (64, 64, 5, 1), (64, 128, 9, 3), (128, 128, 9, 2), (128, 512, 5, 2)]   # insize, size, winlen, stride


def tx_conv(i, chunks=2, T_in=1920, convs=SUP_CONVS):
    """Conv i >= 1 of the transformer's stack (tx_model.cu make_plan): reads the padded buffer of conv i - 1, writes at row
    pad into its own padded buffer (the last conv: x, unpadded)."""
    t, tl, pads, tpad = T_in, [], [], []
    for j, (_, _, wl, s) in enumerate(convs):
        t = (t + 2 * (wl // 2) - wl) // s + 1
        nxt = convs[j + 1][2] // 2 if j + 1 < len(convs) else 0
        tl.append(t)
        pads.append(nxt)
        tpad.append(t + 2 * nxt + 16)
    cin, cout, wl, s = convs[i]
    last = i + 1 == len(convs)
    rng = _rng("txconv", i)
    K = wl * cin
    d = dict(batches=chunks, rows_per_batch=tl[i], a_row_stride=s * cin, a_batch_stride=tpad[i - 1] * cin, K=K, N=cout,
             act=R.ACT_SWISH, out_offset=0 if last else pads[i] * cout, out_m1=tl[i],
             out_s0=(tl[i] if last else tpad[i]) * cout, out_s1=cout)
    out_len = chunks * (tl[i] if last else tpad[i]) * cout
    case = Case(f"tx conv {i + 1}", d, _f16(rng, chunks * tpad[i - 1] * cin), _f16(rng, (cout, K), 1.0 / np.sqrt(K)),
                out_len, {"bias": (rng.standard_normal(cout) * 0.1).astype(np.float32)}, _sample(chunks * tl[i]))
    return _nan_uncovered(case)


def _norm_inputs(case, dm):
    """The folded RMSNorm of A's rows: a_ss partials from A's own fp16 rows."""
    rows = R.rows_of(case.d)
    case.d.update(a_ss_parts=dm // 32, norm_dim=dm, norm_eps=1e-5)
    case.inputs["a_ss"] = R.partial_ss(case.a.reshape(rows, -1)[:, :dm])
    return case


def tx_qkv(dm, nhead, rope_T, rows, a_ss):
    """qkv + RoPE (q and k rotated, v not), with rows spanning several rope_T chunks."""
    case = _dense(f"qkv dm={dm} rope_T={rope_T} rows={rows} a_ss={a_ss}", _rng("qkv", dm, rope_T, a_ss), rows, dm, 3 * dm,
                  R.ACT_ROPE, bias=False, a_scale=4.0 if a_ss else 1.0, theta=THETA, max_seq_len=MAX_SEQ, rope_T=rope_T,
                  rope_cols=2 * nhead * 64)
    return _norm_inputs(case, dm) if a_ss else case


def _residual(case, rng, dm, gain=True):
    rows = R.rows_of(case.d)
    res = _f16(rng, rows * dm, 3.0)
    case.inputs.update(residual=res, res_ss=R.partial_ss(res.reshape(rows, dm)), alpha=ALPHA)
    if gain:
        case.inputs["res_gain"] = (1.0 + 0.2 * rng.standard_normal(dm)).astype(np.float32)
    case.d.update(res_ss_parts=dm // 32, norm_dim=dm, norm_eps=1e-5)
    case.out_ss = True
    return case


def tx_out_proj(dm, rows):
    rng = _rng("out_proj", dm)
    return _residual(_dense(f"out_proj dm={dm}", rng, rows, dm, dm), rng, dm)


def tx_fc1(dm, ff, rows):
    case = _dense(f"fc1 dm={dm}", _rng("fc1", dm), rows, dm, 2 * ff, R.ACT_SWIGLU, bias=False, a_scale=3.0)
    return _norm_inputs(case, dm)


def tx_fc2(ff, dm, rows):
    rng = _rng("fc2", ff)
    return _residual(_dense(f"fc2 K={ff}", rng, rows, ff, dm, bias=False), rng, dm)


def tx_upsample(dm, rows):
    return _norm_inputs(_dense(f"upsample dm={dm}", _rng("ups", dm), rows, dm, 2 * dm, a_scale=3.0), dm)


# ---- running and checking -----------------------------------------------------------------------------------------------
def launch(case, **over):
    from dorado_b200 import lib as L
    d = {k: v for k, v in case.d.items() if k not in ("K", "N")}
    d.update(over)
    assert case.w.shape == (case.d["N"], case.d["K"])
    return L.test_gemm_desc(case.a, case.w, R.sentinel_buffer(case.out_len), out_ss=case.out_ss, **d, **case.inputs)


def verify(case, out, ss=None, c_acc=None):
    """Every check of a launch; returns the worst error as a fraction of the bound (values, and out_ss's when there)."""
    R.check_sentinel(case.d, out)
    g = case.sample if case.sample is not None else np.arange(R.rows_of(case.d), dtype=np.int64)
    ref, bound = R.reference(case.d, case.a, case.w, g, c_acc=c_acc, **case.inputs)
    ratio = R.worst_ratio(R.gather_out(case.d, out, g), ref, bound)
    assert ratio <= 1.0, f"{case.label}: error {ratio:.3f} of the bound"
    if case.out_ss:
        r_ss = R.check_out_ss(R.gather_out(case.d, out, np.arange(R.rows_of(case.d))), ss)
        assert r_ss <= 1.0, f"{case.label}: out_ss error {r_ss:.3f} of its bound"
    return ratio


def run_and_verify(case, **over):
    out, ss = launch(case, **over)
    ratio = verify(case, out, ss)
    print(f"\n[{case.label}] worst error {ratio:.3f} of the bound")
    return out, ss, ratio


# ---- the plans ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,act", [(384, R.ACT_TANH), (128, R.ACT_SWISH)], ids=["hac", "lstm128"])
def test_lstm_conv3(C, act):
    run_and_verify(lstm_conv3(C, chunks=40, T_in=1200, act=act))


@pytest.mark.parametrize("C", [96, 192, 384])
def test_lstm_xprojection(C):
    run_and_verify(lstm_xproj(C))


def test_lstm_xprojection_max_ctas():
    """A persistent grid of 1, 7 and 100 CTAs over 96 tiles: the mbarrier ring changes phase across tiles.  The output
    is bit-identical to the uncapped grid's."""
    case = lstm_xproj(96, T=64, Np=64)
    base, _, _ = run_and_verify(case)
    for m in (1, 7, 100):
        out, _, _ = run_and_verify(dataclasses.replace(case, label=f"xproj C=96 max_ctas={m}"), max_ctas=m)
        assert np.array_equal(out.view(np.uint16), base.view(np.uint16)), m


@pytest.mark.parametrize("act", [R.ACT_TANH_X5, R.ACT_NONE])
def test_lstm_crf_linear(act):
    run_and_verify(lstm_crf(384, T_out=100, Np=32, outsize=1024, act=act))


def test_lstm_crf_two_stage():
    """The decomposed linear: C -> out_features (plain, contiguous), then out_features -> outsize transposed."""
    run_and_verify(_dense("crf linear1 C=768", _rng("lin1", 768), 100 * 32, 768, 128, a_inner=768))
    run_and_verify(lstm_crf(128, T_out=100, Np=32, outsize=1024, act=R.ACT_TANH_X5, a_inner=False, label="crf linear2"))


@pytest.mark.parametrize("i", [1, 2, 3, 4])
def test_tx_conv(i):
    run_and_verify(tx_conv(i))


@pytest.mark.parametrize("dm,nhead", [(512, 8), (1536, 24)], ids=["sup", "tx1536"])
@pytest.mark.parametrize("a_ss", [False, True])
def test_tx_qkv_rope(dm, nhead, a_ss):
    """Rows spanning two and three chunks of rope_T tokens, rope_T not a multiple of the 128-row tile."""
    for rope_T, rows in ((200, 400), (333, 900)):
        run_and_verify(tx_qkv(dm, nhead, rope_T, rows, a_ss))


def test_tx_out_proj():
    run_and_verify(tx_out_proj(512, 600))


def test_tx_fc1():
    run_and_verify(tx_fc1(512, 2048, 300))


@pytest.mark.parametrize("ff,dm", [(2048, 512), (6144, 1536)])
def test_tx_fc2(ff, dm):
    run_and_verify(tx_fc2(ff, dm, 300))


def test_tx_upsample():
    run_and_verify(tx_upsample(512, 600))


def test_out_ss_feeds_a_ss():
    """out_proj's partial sums feed fc1's row scales: fc1 must equal float64 RMSNorm of out_proj's stored fp16 rows."""
    first = tx_out_proj(512, 600)
    y, ss, _ = run_and_verify(first)
    second = tx_fc1(512, 2048, 600)
    second.a = y.copy()
    second.inputs["a_ss"] = ss
    second.label = "fc1 fed by out_proj's out_ss"
    run_and_verify(second)


def test_out_ss_is_deterministic():
    """out_ss and the output are bit-identical across grid caps and repeated calls."""
    case = tx_fc2(2048, 512, 1000)
    out0, ss0, _ = run_and_verify(case)
    for m in (0, 1, 7, 100):
        out, ss = launch(case, max_ctas=m)
        assert np.array_equal(out.view(np.uint16), out0.view(np.uint16)) and np.array_equal(ss.view(np.uint32), ss0.view(np.uint32)), m


# ---- edges --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 127, 128, 129])
@pytest.mark.parametrize("N", [32, 96, 128, 256, 4096])
def test_edges(M, N):
    """Row counts around the 128-row tile, column counts from one 32-column chunk to 32 tiles, K = 64 (one K block); M = 1
    with wide N runs the row tiles fastest (mfast), M = 129 with narrow N the column tiles.  With out_ss where N allows."""
    run_and_verify(_dense(f"edge M={M} N={N}", _rng("edge", M, N), M, 64, N))
    if N % 128 == 0:
        case = _residual(_dense(f"edge M={M} N={N} out_ss", _rng("edge_ss", M, N), M, 64, N), _rng("edge_res", M, N), N)
        run_and_verify(case)


@pytest.mark.parametrize("rows", [65 * 128, 66 * 128])
@pytest.mark.parametrize("out_ss", [False, True])
def test_split_threshold(rows, out_ss):
    """N = 128 on both sides of the 66-row-tile threshold below which the plan halves the tile width to fill the SMs; the
    plan keeps whole 128-column tiles when out_ss is written (d_model 128's out_proj and fc2)."""
    case = _dense(f"split rows={rows} out_ss={out_ss}", _rng("split", rows, out_ss), rows, 128, 128)
    if out_ss:
        case = _residual(case, _rng("split_res", rows), 128)
    run_and_verify(case)


# ---- a d_model 128 transformer --------------------------------------------------------------------------------------------
def test_d_model_128_model(tmp_path):
    """d_model 128 (nhead 2) at depth 2: runner_bytes equals what runner creation adds, and the scores match the oracle.
    2 x 7680 samples are 1280 token rows, fewer than 66 row tiles."""
    from test_tx1536_cpu import config_variant
    from test_tx1536_gpu import _against_oracle, _model, _scores, _signal
    from dorado_b200.runner import B200Caller, B200ModelRunner
    cfg, w = _model(config_variant(tmp_path, depth=2, d_model=128, nhead=2, ff=512, name="dm128"))
    sig = _signal(cfg, 2, 7680, seed=11)
    caller = B200Caller(cfg, w)
    want = caller.runner_bytes(2, 7680)
    before = caller.stats()["arena_bytes"]
    runner = B200ModelRunner(caller, 2, 7680)
    assert caller.stats()["arena_bytes"] - before == want
    runner.close()
    caller.close()
    _against_oracle(cfg, w, sig, _scores(cfg, w, sig), label="d_model 128 depth 2")
