"""The per-launch transformer reference of tests/tx_layer_ref.py without a GPU: chained launch by launch it reproduces the
numpy oracle's forward, each check of tests/test_tx_layers_gpu.py fails for a kernel that makes one of the mistakes it
is meant to catch and passes the correctly rounded result, and the workspace layout and launch lists match hand-computed
examples."""
import numpy as np
import pytest

import tx_layer_ref as X
from conftest import CONFIG_DIR

SUP = CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0"


def _sup(tmp_path, depth):
    from dorado_b200.config import load_model_config
    text = (SUP / "config.toml").read_text()
    d = tmp_path / f"sup_d{depth}"
    d.mkdir()
    (d / "config.toml").write_text(text.replace("depth = 18\n", f"depth = {depth}\n"))
    return load_model_config(d)


def _q16(a):
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


# ---- the chain against the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fold", "rmsnorm_pass"])
def test_chain_matches_oracle(tmp_path, mode):
    """Each launch's reference fed its own predecessors' float64 outputs, over sup at depth 2 with 2 chunks of 256 tokens
    (longer than the window), gives nn_oracle's float32 forward within float32 noise."""
    from dorado_b200.weights import synthetic_weights
    from oracle import nn_oracle
    cfg = _sup(tmp_path, 2)
    w = synthetic_weights(cfg, 42)
    N, T_in = 2, 3072
    sig = np.random.default_rng(5).standard_normal((N, T_in)).astype(np.float16)
    ref = X.TxLayerRef(cfg, w, mode, N, T_in)
    assert ref.T == 256
    inp = {"signal": sig.astype(np.float64)}
    for _, kind, idx in X.launches(cfg, mode):
        for out, (r, _) in ref.reference(kind, idx, inp).items():
            inp[out] = r
    want = nn_oracle.forward(cfg, w, sig.astype(np.float32)).astype(np.float64)
    got = inp["scores"]
    assert got.shape == want.shape
    err = np.abs(got - want).max() / np.abs(want).max()
    rel_l2 = np.linalg.norm(got - want) / np.linalg.norm(want)
    print(f"\n[{mode}] chain vs oracle: max {err:.2e} x max|ref|, relative L2 {rel_l2:.2e}")
    assert err < 1e-4 and rel_l2 < 1e-5


# ---- the checks can fail ----------------------------------------------------------------------------------------------
def _random_inputs(cfg, lay, rng):
    """fp16-valued buffers of a plausible scale: x, y un-normalised rows, att, hid, ups; qkv with q . k / 8 of standard
    deviation about 2."""
    rows, dm, ff = lay["rows"], cfg.tx.d_model, cfg.tx.dim_feedforward
    f = lambda shape, s=1.0: _q16(rng.standard_normal(shape) * s)
    qkv = f((rows, 3 * dm))
    qkv[:, :2 * dm] *= 1.4
    return {"x": f((rows, dm), 3.0), "y": f((rows, dm), 3.0), "att": f((rows, dm)), "qkv": _q16(qkv),
            "hid": f((rows, ff), 0.5), "ups": f((rows, cfg.tx.upsample_scale * dm))}


@pytest.mark.parametrize("mutation", list(X.MUTATIONS))
def test_checks_flag_each_mistake(tmp_path, mutation):
    """A kernel making the mistake (its result rounded to fp16) fails the check by the GPU test's margin; the correctly
    rounded result passes.  sup's shapes at depth 2, layer 1, 2 chunks of 256 tokens of random inputs."""
    from dorado_b200.weights import synthetic_weights
    cfg = _sup(tmp_path, 2)
    w = synthetic_weights(cfg, 42)
    ref = X.TxLayerRef(cfg, w, "fold", 2, 3072)
    inp = _random_inputs(cfg, ref.lay, np.random.default_rng(9))
    kind = X.MUTATIONS[mutation]
    idx = 0 if kind == "crf" else 1
    (out, (good, bound)), = ref.reference(kind, idx, inp).items()
    (_, (bad, _)), = ref.reference(kind, idx, inp, mutation=mutation).items()
    ok = X.worst_ratio(_q16(good), good, bound)
    wrong = X.worst_ratio(_q16(bad), good, bound)
    print(f"\n[{mutation}] correctly rounded {ok:.3f}, mistaken {wrong:.1f} x the bound")
    assert ok <= 1.0 and wrong >= 3.0


def test_e4m3_checks():
    """fc1's E4M3 criterion passes the saturating cast of v and fails a cast one E4M3 step away; norm1's copy is the
    satfinite cast, so 500 becomes 448 (0x7e) where torch's plain cast gives NaN."""
    rng = np.random.default_rng(3)
    v = rng.standard_normal((64, 128)) * 4
    tol = 1e-4 * np.abs(v)
    good = X.e4m3_sat_bytes(v)
    outside, ratio = X.e4m3_cast_check(good, v, tol)
    assert outside == 0 and ratio.max() <= 1.0
    off = good.copy()
    off[0, 0] = good[0, 0] + 1   # the next E4M3 value of the same sign
    outside, ratio = X.e4m3_cast_check(off, v, tol)
    assert outside == 1 and ratio.max() >= 3.0
    assert X.e4m3_sat_bytes(np.array([500.0, -500.0])).tolist() == [0x7E, 0xFE]


def test_fp8_swap_is_flagged(tmp_path):
    """The y and gate halves of fc1 swapped, on the fp8_ffn criterion."""
    from dorado_b200.weights import synthetic_weights
    cfg = _sup(tmp_path, 2)
    w = synthetic_weights(cfg, 42)
    ref = X.TxLayerRef(cfg, w, "fp8_ffn", 1, 1536)
    rng = np.random.default_rng(4)
    a8 = X.decode_e4m3(X.e4m3_sat_bytes(rng.standard_normal((ref.lay["rows"], cfg.tx.d_model)))).astype(np.float64)
    (_, (v, tol)), = ref.reference("fc1", 1, {"a8": a8}).items()
    (_, (vs, _)), = ref.reference("fc1", 1, {"a8": a8}, mutation="fc1_swap").items()
    outside, ratio = X.e4m3_cast_check(X.e4m3_sat_bytes(v), v, tol)
    assert outside == 0 and ratio.max() <= 1.0
    outside, ratio = X.e4m3_cast_check(X.e4m3_sat_bytes(vs), v, tol)
    assert outside > 0 and ratio.max() >= 3.0


def test_a_kernel_beyond_the_bound_fails(tmp_path):
    """Every check compares element by element: one output element moved by twice its bound fails it."""
    from dorado_b200.weights import synthetic_weights
    cfg = _sup(tmp_path, 2)
    ref = X.TxLayerRef(cfg, synthetic_weights(cfg, 42), "fold", 2, 3072)
    inp = _random_inputs(cfg, ref.lay, np.random.default_rng(2))
    for kind in ("qkv", "attention", "out_proj", "fc1", "fc2", "upsample", "crf"):
        (_, (r, b)), = ref.reference(kind, 0, inp).items()
        got = r.copy()
        got.reshape(-1)[7] += 2 * b.reshape(-1)[7]
        assert X.worst_ratio(got, r, b) == pytest.approx(2.0), kind


# ---- the layout ---------------------------------------------------------------------------------------------------------
# sup, one chunk of 3072 samples: convs (t, pad, t_pad) = (3072, 2, 3092), (3072, 4, 3096), (1024, 4, 1048), (512, 2, 532),
# (256, 0, 272); T = 256 tokens
SUP_3072 = {"cbuf0": (0, 3092 * 64 * 2), "cbuf1": (395776, 3096 * 64 * 2), "cbuf2": (792064, 1048 * 128 * 2),
            "cbuf3": (1060352, 532 * 128 * 2), "x": (1196544, 262144), "y": (1458688, 262144), "att": (1720832, 262144),
            "qkv": (1982976, 786432), "hid": (2769408, 1048576), "ups": (3817984, 524288), "ss_a": (4342272, 16384),
            "ss_b": (4358656, 16384)}
LAYER = {"fold": ["qkv_gemm", "tx_attention", "out_proj_gemm", "fc1_swiglu_gemm", "fc2_gemm"],
         "rmsnorm_pass": ["qkv_gemm", "tx_attention", "out_proj_gemm", "rmsnorm", "fc1_swiglu_gemm", "fc2_gemm", "rmsnorm"],
         "fp8_ffn": ["qkv_gemm", "tx_attention", "out_proj_gemm", "rmsnorm_e4m3", "fc1_swiglu_gemm", "fc2_gemm"]}


@pytest.mark.parametrize("mode", X.MODES)
def test_workspace_layout(tmp_path, mode):
    cfg = _sup(tmp_path, 2)
    lay = X.workspace_layout(cfg, 1, 3072, mode)
    assert lay["convs"] == [(3072, 2, 3092), (3072, 4, 3096), (1024, 4, 1048), (512, 2, 532), (256, 0, 272)]
    assert lay["T"] == 256 and lay["rows"] == 256
    assert lay["buffers"] == SUP_3072 and lay["bytes"] == 4375040
    names = [p[0] for p in X.launches(cfg, mode)]
    assert names == ["tx_conv1"] + ["tx_conv_gemm"] * 4 + LAYER[mode] * 2 + ["upsample_gemm", "crf_gemm"]
    assert len(names) == X.launch_count(cfg, mode) == {"fold": 17, "rmsnorm_pass": 21, "fp8_ffn": 19}[mode]
    # what the layer's launches write
    kinds = [p[1] for p in X.launches(cfg, mode) if p[2] == 1 and p[1] not in ("conv", "conv1", "upsample", "crf")]
    got = {k: X.writes(cfg, lay, k, 1, mode) for k in kinds}
    want = {"fold": {"out_proj": {"y": None, "ss_b": None}, "fc2": {"x": None, "ss_a": None}},
            "rmsnorm_pass": {"out_proj": {"y": None}, "norm1": {"x": None}, "fc2": {"y": None}, "norm2": {"x": None}},
            "fp8_ffn": {"out_proj": {"y": None}, "norm1": {"att": None, "qkv": (0, 256 * 512)},
                        "fc1": {"hid": (0, 256 * 2048)}, "fc2": {"x": None, "ss_a": None}}}[mode]
    for k, v in want.items():
        assert got[k] == v, k
    assert X.writes(cfg, lay, "conv", 4, mode) == {"x": None} and X.writes(cfg, lay, "conv", 2, mode) == {"cbuf2": None}


def test_logical_inputs_and_padding(tmp_path):
    """The snapshot views read the rows the layout says: cbuf i's valid rows start after its front padding."""
    cfg = _sup(tmp_path, 2)
    lay = X.workspace_layout(cfg, 2, 3072, "fold")
    ws = np.zeros(lay["bytes"], np.uint8)
    raw = {name: ws[off:off + nb] for name, (off, nb) in lay["buffers"].items()}
    t, pad, tp = lay["convs"][1]
    b = raw["cbuf1"].view(np.float16).reshape(2, tp, 64)
    b[1, pad + 5, 3] = 7.0
    assert X.cbuf_padding_nonzero(cfg, lay, raw, 1) == 0
    inp = X.logical_inputs(cfg, lay, raw, "fold")
    assert inp["conv1"].shape == (2, t, 64) and inp["conv1"][1, 5, 3] == 7.0
    b[0, pad - 1, 0] = 1.0
    b[1, pad + t, 0] = 1.0
    assert X.cbuf_padding_nonzero(cfg, lay, raw, 1) == 2


def test_attention_bound_holds_for_fp16_weights():
    """The attention bound admits a kernel that rounds every weight exp(s - max) to fp16 before P V (its largest error
    source), normalises by the unrounded sum and rounds the output to fp16, with a peaked and a flat softmax."""
    rng = np.random.default_rng(8)
    N, T, H, win = 2, 300, 2, (127, 128)
    for qk_scale in (1.0, 3.0):
        qkv = _q16(rng.standard_normal((N * T, 3 * H * 64)))
        qkv[:, :2 * H * 64] = _q16(qkv[:, :2 * H * 64] * qk_scale)
        ref, bound = X.attention(qkv, N, T, H, win)
        x = qkv.reshape(N, T, 3, H, 64)
        i, j = np.arange(T)[:, None], np.arange(T)[None, :]
        mask = (j - i >= -win[0]) & (j - i <= win[1])
        sim = np.empty((N, T, H, 64))
        for n in range(N):
            for h in range(H):
                s = np.where(mask, x[n, :, 0, h] @ x[n, :, 1, h].T / 8.0, -np.inf)
                p = np.exp(s - s.max(axis=1, keepdims=True))
                sim[n, :, h] = (_q16(p) @ x[n, :, 2, h]) / p.sum(axis=1, keepdims=True)
        r = X.worst_ratio(_q16(sim.reshape(N * T, -1)), ref, bound)
        print(f"\n[q k x {qk_scale}] fp16 weights: {r:.3f} of the bound")
        assert r <= 1.0
