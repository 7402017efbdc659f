"""The GEMM plan tests without a GPU: tests/gemm_ref.py's addressing against plain loops; that every check of
tests/test_gemm_plans_gpu.py fails for a kernel that made one of the mistakes those checks exist for (each simulated
on the GPU test's own inputs by writing a mis-computed reference, rounded to fp16, into the sentinel buffer), while
the correctly rounded reference passes; b200_test_gemm_desc's refusal of a descriptor that reaches beyond any buffer it
is given, or that has no kernel form or sets an input its form does not read, which happens before any device work; and
the d_model 128 configuration the GPU test runs."""
import dataclasses
import itertools

import numpy as np
import pytest

import gemm_ref as R
import test_gemm_plans_gpu as P


# ---- the reference's addressing ---------------------------------------------------------------------------------------
def test_reference_matches_plain_loops():
    """Overlapping rows in two batches, a_inner < K, a blocked output at an offset, bias and a residual; and RoPE."""
    rng = np.random.default_rng(1)
    d = dict(batches=2, rows_per_batch=3, a_row_stride=8, a_batch_stride=40, a_inner=24, K=64, N=64, act=R.ACT_NONE,
             out_offset=6, out_m1=2, out_s0=200, out_s1=70)
    a = rng.standard_normal(200).astype(np.float16)
    w = rng.standard_normal((64, 64)).astype(np.float16)
    bias = rng.standard_normal(64).astype(np.float32)
    res = rng.standard_normal(6 * 64).astype(np.float16)
    g = np.arange(6)
    ref, _ = R.reference(d, a, w, g, bias=bias, residual=res, alpha=0.5)
    offs = R.out_offsets(d)
    for gi in range(6):
        b, r = divmod(gi, 3)
        assert offs[gi] == 6 + (gi // 2) * 200 + (gi % 2) * 70
        for n in range(64):
            acc = sum(float(a[b * 40 + r * 8 + k]) * float(w[n, k]) for k in range(24))
            want = acc + float(bias[n]) + float(np.float32(0.5)) * float(res[gi * 64 + n])
            assert abs(ref[gi, n] - want) <= 1e-9 * (1 + abs(want))

    dr = dict(rows_per_batch=5, a_row_stride=64, K=64, N=128, act=R.ACT_ROPE, theta=10000.0, rope_T=3, rope_cols=64,
              out_s0=128)
    a = rng.standard_normal(5 * 64).astype(np.float16)
    w = rng.standard_normal((128, 64)).astype(np.float16)
    ref, _ = R.reference(dr, a, w, np.arange(5))
    v = a.astype(np.float64).reshape(5, 64) @ w.astype(np.float64).T
    for gi in range(5):
        t = gi % 3
        for i in range(32):
            ang = t * 10000.0 ** (-2 * i / 64)
            assert abs(ref[gi, i] - (np.cos(ang) * v[gi, i] - np.sin(ang) * v[gi, 32 + i])) < 1e-9
            assert abs(ref[gi, 32 + i] - (np.sin(ang) * v[gi, i] + np.cos(ang) * v[gi, 32 + i])) < 1e-9
        assert np.array_equal(ref[gi, 64:], v[gi, 64:])   # beyond rope_cols: not rotated


# ---- sensitivity ----------------------------------------------------------------------------------------------------------
def simulate(case, d=None, a=None, **inputs):
    """The output buffer (and out_ss) of a kernel that computed the reference with the given changes, rounded to fp16."""
    d = d or case.d
    a = case.a if a is None else a
    kw = dict(case.inputs, **inputs)
    g = np.arange(R.rows_of(d), dtype=np.int64)
    ref, _ = R.reference(d, a, case.w, g, **kw)
    out = R.sentinel_buffer(case.out_len).copy()
    idx = R.out_offsets(d, g)[:, None] + np.arange(R.n_out(d))[None, :]
    out[idx] = ref.astype(np.float16)
    ss = R.partial_ss(ref.astype(np.float16)) if case.out_ss else None
    return out, ss


def _fails(case, out, ss):
    with pytest.raises(AssertionError):
        P.verify(dataclasses.replace(case, sample=None), out, ss)


def _rope_case():
    return P.tx_qkv(512, 8, 200, 400, a_ss=True)


def test_correct_rounding_passes():
    """The control: the correctly rounded reference passes every check of every case used below."""
    for case in (_rope_case(), P.tx_out_proj(512, 600), P.tx_upsample(512, 600), P.lstm_crf(384, 100, 32, 1024, R.ACT_TANH_X5),
                 P.lstm_xproj(96)):
        assert P.verify(dataclasses.replace(case, sample=None), *simulate(case)) <= 1.0


@pytest.mark.parametrize("mutation", ["position_off_by_one", "position_not_modulo", "sin_sign"])
def test_rope_mistakes_fail(monkeypatch, mutation):
    case = _rope_case()
    T = case.d["rope_T"]
    if mutation == "position_off_by_one":
        monkeypatch.setattr(R, "rope_positions", lambda d, g: g % T + 1)
    elif mutation == "position_not_modulo":
        monkeypatch.setattr(R, "rope_positions", lambda d, g: g)
    else:
        cs = R.rope_cos_sin
        monkeypatch.setattr(R, "rope_cos_sin", lambda ang: (cs(ang)[0], -cs(ang)[1]))
    out, ss = simulate(case)
    monkeypatch.undo()
    _fails(case, out, ss)


@pytest.mark.parametrize("mutation", ["res_gain", "alpha"])
def test_residual_mistakes_fail(mutation):
    case = P.tx_out_proj(512, 600)
    _fails(case, *simulate(case, **({"res_gain": None} if mutation == "res_gain" else {"alpha": 1.0})))


def test_transposed_output_mistake_fails():
    case = P.lstm_crf(384, 100, 32, 1024, R.ACT_TANH_X5)
    swapped = dict(case.d, out_s0=case.d["out_s1"], out_s1=case.d["out_s0"])
    out = R.sentinel_buffer(case.out_len).copy()
    g = np.arange(R.rows_of(case.d), dtype=np.int64)
    ref, _ = R.reference(case.d, case.a, case.w, g, **case.inputs)
    idx = R.out_offsets(swapped, g)[:, None] + np.arange(R.n_out(case.d))[None, :]
    keep = idx[:, -1] < case.out_len   # what the swapped kernel would write inside the buffer
    out[idx[keep]] = ref[keep].astype(np.float16)
    _fails(case, out, None)


def test_dropped_a_ss_partial_fails(monkeypatch):
    case = P.tx_upsample(512, 600)
    full = R.inv_rms
    monkeypatch.setattr(R, "inv_rms", lambda u, dim, eps: 1.0 / np.sqrt((u[:, 32:dim].astype(np.float64) ** 2).sum(axis=1) / dim + eps))
    out, ss = simulate(case)
    monkeypatch.setattr(R, "inv_rms", full)
    _fails(case, out, ss)


def test_ignored_a_inner_fails():
    """W's K padding columns are not zero in the x-projection case: reading the next row's elements there shows."""
    case = P.lstm_xproj(96)
    padded = np.concatenate([case.a, np.zeros(case.d["K"], np.float16)])
    _fails(case, *simulate(case, d=dict(case.d, a_inner=0), a=padded))


def test_uncovered_conv_rows_are_nan():
    """The conv cases leave NaN where no window reads, so a kernel that read there would produce NaN."""
    for case in (P.lstm_conv3(384, 40, 1200, R.ACT_TANH), P.tx_conv(2)):
        nan = np.isnan(case.a.astype(np.float32))
        assert nan.any() and not nan[R.covered_a(case.d, case.a.size)].any()


# ---- the hook's refusals --------------------------------------------------------------------------------------------------
def _hook_case():
    """An out_proj-like descriptor using every buffer: transposed output at an offset, folded norms, RoPE off."""
    rows, K, N = 6, 64, 128
    d = dict(batches=2, rows_per_batch=3, a_row_stride=16, a_batch_stride=96, a_inner=48, out_offset=4, out_m1=3,
             out_s0=300, out_s1=128, a_ss_parts=2, res_ss_parts=4, norm_dim=128, alpha=1.5)
    a_len = 96 + 2 * 16 + 48
    out_len = 4 + 300 + 2 * 128 + N
    bufs = dict(a=np.ones(a_len, np.float16), w=np.ones((N, K), np.float16), bias=np.zeros(N, np.float32),
                residual=np.zeros(rows * N, np.float16), res_gain=np.ones(N, np.float32), a_ss=np.ones(rows * 2, np.float32),
                res_ss=np.ones(rows * 4, np.float32), out=np.zeros(out_len, np.float16), out_ss=np.zeros(rows * 4, np.float32))
    return d, bufs


def _hook_case_s8():
    """The int8 QKV-like descriptor without RoPE: int8 operands with row and column factors and a bias, over two batches."""
    rows, K, N = 6, 128, 128
    d = dict(batches=2, rows_per_batch=3, a_row_stride=128, a_batch_stride=400, K=K, in_type=2, act=R.ACT_NONE,
             out_m1=1, out_s0=N)
    bufs = dict(a=np.ones(400 + 2 * 128 + K, np.int8), w=np.ones((N, K), np.int8), bias=np.zeros(N, np.float32),
                col_scale=np.ones(N, np.float32), row_scale=np.ones(rows, np.float32), out=np.zeros(rows * N, np.float16))
    return d, bufs


def _call(d, bufs, short=None):
    """b200_test_gemm_desc on the buffers, N = 128 and K = 64 unless d sets it, each length as given except `short`'s,
    one less."""
    import ctypes as C
    from dorado_b200 import lib as L
    t = L.GemmTestDesc()
    for name, arr in bufs.items():
        setattr(t, name, arr.ctypes.data)
        setattr(t, name + "_len", arr.size - (name == short))
    t.K, t.N, t.norm_eps = 64, 128, 1e-5
    for k, v in d.items():
        setattr(t, k, v)
    L.check(L.load_library().b200_test_gemm_desc(0, C.byref(t)))


def _status(fn):
    from dorado_b200 import lib as L
    try:
        fn()
    except L.B200Error as e:
        return e.status, str(e)
    return L.B200_OK, ""


@pytest.mark.parametrize("buf", ["a", "w", "bias", "residual", "res_gain", "a_ss", "res_ss", "out", "out_ss", "col_scale",
                                 "row_scale"])
def test_hook_refuses_short_buffers(buf):
    """One element short of what the descriptor reaches: B200_ERR_INVALID, naming the buffer, before any device work.
    At the exact length the hook goes on (to the device check here, to the GEMM on a GPU)."""
    from dorado_b200 import lib as L
    d, bufs = _hook_case_s8() if buf in ("col_scale", "row_scale") else _hook_case()
    status, _ = _status(lambda: _call(d, bufs))
    assert status != L.B200_ERR_INVALID
    status, msg = _status(lambda: _call(d, bufs, short=buf))
    assert status == L.B200_ERR_INVALID and f"{buf} is too short" in msg.lower(), (buf, status, msg)


# gemm.cu's table of kernel forms: (A and W type, output type, activation, row factors) -> the optional inputs the form
# reads.  GemmType 0 fp16, 1 E4M3, 2 int8; col_scale is required where it is read.
F16, E4M3, S8 = 0, 1, 2
PLAIN = {"bias", "residual", "a_ss", "out_ss"}
FORMS = {
    **{(F16, F16, act, False): PLAIN for act in (R.ACT_NONE, R.ACT_SWISH, R.ACT_SWISH_CLAMP, R.ACT_TANH, R.ACT_TANH_X5)},
    (F16, F16, R.ACT_SWIGLU, False): {"bias", "a_ss"},
    (F16, F16, R.ACT_ROPE, False): {"a_ss"},
    (F16, S8, R.ACT_TANH, False): {"bias"},
    (E4M3, F16, R.ACT_NONE, False): PLAIN,
    (E4M3, E4M3, R.ACT_SWIGLU, False): {"bias", "a_ss"},
    (S8, F16, R.ACT_NONE, False): {"col_scale", "bias"},
    (S8, F16, R.ACT_TANH_X5, False): {"col_scale", "bias"},
    (S8, F16, R.ACT_NONE, True): {"col_scale", "bias"},
    (S8, F16, R.ACT_ROPE, True): {"col_scale"},
}
OPTIONAL = ("bias", "residual", "a_ss", "out_ss", "col_scale")


def _form_call(key, given):
    """b200_test_gemm_desc on 4 rows, K = N = 128, with the types, activation and row factors of `key` and the optional
    inputs named in `given`: buffers valid for every form, so that on a GPU an accepted form just runs."""
    from dorado_b200 import lib as L
    in_type, out_type, act, rows = key
    M, K, N = 4, 128, 128
    n_out = N // 2 if act == R.ACT_SWIGLU else N
    inputs = dict(bias=np.zeros(N, np.float32), residual=np.zeros(M * N, np.float16), a_ss=np.ones(M, np.float32),
                  col_scale=np.ones(N, np.float32))
    kw = {k: v for k, v in inputs.items() if k in given}
    if "residual" in given:
        kw.update(alpha=1.0)
    if "a_ss" in given:
        kw.update(a_ss_parts=1, norm_dim=K)
    if act == R.ACT_ROPE:
        kw.update(theta=1e4, max_seq_len=8, rope_T=4, rope_cols=N)
    dt = L.GEMM_DTYPES
    L.test_gemm_desc(np.zeros(M * K, dt[in_type]), np.zeros((N, K), dt[in_type]), np.zeros(M * n_out, dt[out_type]),
                     rows_per_batch=M, a_row_stride=K, out_s0=n_out, act=act, in_type=in_type, out_type=out_type,
                     row_scale=np.ones(M, np.float32) if rows else None, out_ss="out_ss" in given, **kw)


def test_hook_accepts_exactly_the_kernel_forms():
    """Every (A and W type, output type, activation, row factors): exactly the table's 14 get past the form check (to the
    device check here, to the GEMM on a GPU); every other one is refused before any device work."""
    from dorado_b200 import lib as L
    acts = (R.ACT_NONE, R.ACT_SWISH, R.ACT_SWISH_CLAMP, R.ACT_TANH, R.ACT_TANH_X5, R.ACT_SWIGLU, R.ACT_ROPE)
    accepted = set()
    for key in itertools.product((F16, E4M3, S8), (F16, E4M3, S8), acts, (False, True)):
        status, msg = _status(lambda: _form_call(key, {"col_scale"} if key[0] == S8 else set()))
        if status != L.B200_ERR_INVALID:
            accepted.add(key)
        else:
            assert "no kernel form" in msg, (key, msg)
    assert accepted == set(FORMS)


@pytest.mark.parametrize("key", list(FORMS), ids=str)
def test_hook_takes_the_inputs_each_form_reads(key):
    """Each optional input, added to (or, for the required col_scale, taken from) the form's required inputs: accepted
    exactly where the form reads it, and refused, naming it, before any device work where it does not."""
    from dorado_b200 import lib as L
    reads = FORMS[key]
    required = reads & {"col_scale"}
    for name in OPTIONAL:
        status, msg = _status(lambda: _form_call(key, required ^ {name}))
        if name in reads and name not in required:
            assert status != L.B200_ERR_INVALID, (key, name, msg)
        else:
            assert status == L.B200_ERR_INVALID and name in msg, (key, name, status, msg)


def test_hook_refuses_bad_addressing():
    """The residual is addressed g * N + n whatever the output strides; output offsets and strides must be even (the
    epilogue stores pairs); RoPE positions must lie in the table."""
    from dorado_b200 import lib as L
    d, bufs = _hook_case()
    for change, what in ((dict(out_offset=5), "even"), (dict(out_s1=127), "even"), (dict(a_inner=80), "a_inner"),
                         (dict(out_s0=301), "even"), (dict(act=R.ACT_ROPE, theta=1e4, max_seq_len=8, rope_T=9), "RoPE")):
        status, msg = _status(lambda: _call(dict(d, **change), bufs))
        assert status == L.B200_ERR_INVALID and what in msg, (change, msg)
    # the output shifted so that its last row ends one element past the buffer
    status, msg = _status(lambda: _call(dict(d, out_offset=6), bufs))
    assert status == L.B200_ERR_INVALID and "out" in msg


# ---- the d_model 128 configuration ----------------------------------------------------------------------------------------
def test_d_model_128_config(tmp_path):
    from test_tx1536_cpu import config_variant
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import tensor_specs
    cfg = load_model_config(config_variant(tmp_path, depth=2, d_model=128, nhead=2, ff=512, name="dm128"))
    assert (cfg.tx.d_model, cfg.tx.nhead, cfg.tx.depth, cfg.tx.dim_feedforward) == (128, 2, 2, 512)
    assert cfg.convs[-1].size == 128
    specs = tensor_specs(cfg)
    assert specs["transformer_encoder.1.self_attn.Wqkv.weight.tensor"] == (384, 128)
    assert specs["transformer_encoder.1.ff.fc1.weight.tensor"] == (1024, 128)
    assert specs["upsample.linear.weight.tensor"] == (256, 128)
    assert specs["crf.linear.weight.tensor"] == (4096, 128)
    d = L.model_desc_from_config(cfg)
    assert (d.d_model, d.nhead, d.dim_feedforward, d.depth) == (128, 2, 512, 2)
