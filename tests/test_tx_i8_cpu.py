"""The int8_qkv_fp8_ffn transformer precision without a GPU: the numpy quantiser of tests/tx_i8_ref.py against the
reference's quantize_tensor run by torch on fp16 tensors and against the engine's host quantize_rows_f16, the weight
preparation against a torch restatement of the reference's, the int8 restatement against the fp8_ffn one, the
launch-by-launch reference's plan and its sensitivity, the Python interface and the build's ptxas report of the new kernel
instantiations.  The GPU side is tests/test_tx_i8_gpu.py."""
import pathlib
import re

import numpy as np
import pytest
import torch

from conftest import CONFIG_DIR
from test_tx1536_cpu import config_variant
import tx_fp8_ref
import tx_i8_ref
import tx_layer_ref as X

ROOT = pathlib.Path(__file__).resolve().parents[1]
BUILD = ROOT / "dorado_b200" / "csrc" / "build"
SUP = CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0"


def _lib():
    from dorado_b200 import lib as L
    try:
        L.load_library()
    except FileNotFoundError:
        pytest.skip("libb200call.so not built")
    return L


def _torch_quantize(x16, dim):
    """utils::quantize_tensor(t, dim) (torch_utils/tensor_utils.cpp:293-300) on an fp16 CPU tensor, then the callers'
    scale.reciprocal_() on the float scale (TxModules.cpp:500, 958): (int8 q, fp16 scale, fp32 inv)."""
    t = torch.from_numpy(np.ascontiguousarray(x16, np.float16))
    fp_range = t.abs().amax(dim)
    quant_scale = (256 / 2) / fp_range
    t_quant = (t * quant_scale.unsqueeze(dim)).round().clip(-127, 127)
    return t_quant.to(torch.int8).numpy(), quant_scale.numpy(), quant_scale.to(torch.float32).reciprocal_().numpy()


def _edge_rows(cols, rng):
    """Rows of every kind the quantiser meets: random, exact .5 products (ties to even), all zero, tiny absmax (scale +inf,
    with and without zero elements), and scales that round in fp16."""
    rows = [rng.standard_normal(cols) * s for s in (0.05, 1.0, 7.0, 300.0)]
    # absmax 1 -> scale 128: (k + 0.5) / 128 lands exactly on a tie
    r = np.zeros(cols)
    r[:2] = [1.0, -1.0]
    r[2:] = (np.arange(cols - 2) % 60 - 30 + 0.5) / 128.0
    rows.append(r)
    # absmax 0.5 -> scale 256; odd multiples of 1 / 512 are ties
    r = np.zeros(cols)
    r[:2] = [0.5, -0.5]
    r[2:] = (2 * (np.arange(cols - 2) % 60 - 30) + 1) / 512.0
    rows.append(r)
    for amax in (0.3, 0.7371, 1.337, 3.1, 250.0):
        rows.append(np.concatenate([[amax, -amax], rng.uniform(-amax, amax, cols - 2)]))
    rows.append(np.zeros(cols))                                         # all zero
    rows.append(rng.uniform(-1e-3, 1e-3, cols))                         # 128 / absmax overflows fp16: scale +inf
    r = np.zeros(cols)
    r[::3] = rng.uniform(-1e-3, 1e-3, len(r[::3]))                      # ... with zero elements (0 * inf = NaN)
    rows.append(r)
    r = np.zeros(cols)
    r[7] = 128.0 / 65504.0                                              # the last absmax whose scale is finite
    rows.append(r)
    return np.asarray(rows, np.float16)


def test_quantiser_matches_quantize_tensor_and_the_host():
    """Bit for bit: q and the fp16 scale of torch's quantize_tensor wherever torch's result is defined (a finite product),
    inv = float32(scale).reciprocal_(); the defined values elsewhere; and the engine's host quantize_rows_f16 everywhere."""
    rng = np.random.default_rng(11)
    for cols in (128, 512, 1536):
        x = _edge_rows(cols, rng)
        q, scale, inv = tx_i8_ref.quantize_act(x)
        tq, tscale, tinv = _torch_quantize(x, 1)
        np.testing.assert_array_equal(scale.view(np.uint16), tscale.view(np.uint16))
        np.testing.assert_array_equal(inv.view(np.uint32), tinv.view(np.uint32))
        with np.errstate(invalid="ignore", over="ignore"):
            defined = np.isfinite(x.astype(np.float32) * scale.astype(np.float32)[:, None]) | np.isinf(scale)[:, None] & (x != 0)
        np.testing.assert_array_equal(q[defined], tq[defined])
        zero = ~x.any(axis=1)
        tiny = np.isinf(scale)
        assert zero.sum() == 1 and tiny.sum() == 3
        assert (q[zero] == 0).all() and (inv[tiny] == 0).all()
        assert (np.abs(q[tiny & ~zero][x[tiny & ~zero] != 0]) == 127).all()
        assert (q[tiny & ~zero][x[tiny & ~zero] == 0] == -127).all()   # NaN product clipped as quantize_rows_f16 does
        assert np.isfinite(scale[-1]) and q[-1, 7] == 127
        # ties go to even
        np.testing.assert_array_equal(q[4, 2:6], np.rint(np.arange(-30, -26) + 0.5).astype(np.int8))
        L = _lib()
        hq, hscale = L.quantize_rows(x)
        np.testing.assert_array_equal(hq, q)
        np.testing.assert_array_equal(hscale.view(np.uint16), scale.view(np.uint16))


def _torch_prepare(cfg, w):
    """TxModules.cpp:481-506 and 560-589 on a model moved to half (CudaCaller.cpp:167), koi_use_f8 = koi_use_i8 = 1: Wqkv
    quantised per output row (quantize_tensor(w, -1)) BEFORE remove_bits(), which then rounds out_proj and both gains;
    fc1 / fc2 cast to E4M3.  Values only: the Q / K row interleave and the tiling are permutations."""
    out = {}
    for l in range(cfg.tx.depth):
        p = f"transformer_encoder.{l}."
        half = {k: torch.from_numpy(np.asarray(w[p + k + ".tensor"], np.float32)).half()
                for k in ("self_attn.Wqkv.weight", "self_attn.out_proj.weight", "norm1.weight", "norm2.weight",
                          "ff.fc1.weight", "ff.fc2.weight")}
        q, _, inv = _torch_quantize(half["self_attn.Wqkv.weight"].numpy(), -1)
        out[p + "self_attn.Wqkv.q"], out[p + "self_attn.Wqkv.inv"] = q, inv
        for k in ("self_attn.Wqkv.weight", "self_attn.out_proj.weight", "norm1.weight", "norm2.weight"):
            t = half[k].clone()
            t.view(torch.int16).add_(1 << 3)
            t.view(torch.int16).bitwise_and_(0x10000 - (1 << 4))
            out[p + k] = t.float().numpy()
        out[p + "ff.fc1.weight"] = half["ff.fc1.weight"].to(torch.float8_e4m3fn).float().numpy()
        out[p + "ff.fc2.weight"] = half["ff.fc2.weight"].to(torch.float8_e4m3fn).float().numpy()
    return out


@pytest.mark.parametrize("model", ["sup", "tx1536"])
def test_weight_preparation_matches_torch(model, tmp_path):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    d = SUP if model == "sup" else config_variant(tmp_path, depth=2, name="d2")
    cfg = load_model_config(d)
    w = synthetic_weights(cfg, 42)
    mine = tx_i8_ref.prepare_weights(cfg, w)
    ref = _torch_prepare(cfg, w)
    for k, v in ref.items():
        if k.endswith("Wqkv.weight"):
            assert k not in mine   # the int8 rows replace the fp16 Wqkv
            continue
        np.testing.assert_array_equal(mine[k], v, err_msg=k)
    # the order matters: quantising the remove_bits-rounded weights would give other int8 rows
    p = "transformer_encoder.0.self_attn.Wqkv."
    rq, _, _ = tx_i8_ref.quantize_act(ref[p + "weight"].astype(np.float16))
    assert (rq != mine[p + "q"]).any()
    assert np.abs(mine[p + "q"]).max(axis=1).min() == 127   # every row uses the range: the quantiser is per output row
    L = _lib()   # the engine's host quantisation of the same fp16 weights
    hq, hscale = L.quantize_rows(np.asarray(w[p + "weight.tensor"], np.float16))
    np.testing.assert_array_equal(hq, mine[p + "q"])
    np.testing.assert_array_equal((np.float32(1) / hscale.astype(np.float32)).view(np.uint32), mine[p + "inv"].view(np.uint32))


def test_s8_product_rounds_beyond_2_24():
    """float32(acc) rounds once |acc| passes 2^24 (tx1536: up to 1536 127^2, about 2.5e7); the restatement does the same."""
    qa = np.full((1, 1536), 127, np.int8)
    qw = np.full((2, 1536), 127, np.int8)
    qw[1, 0] = 126                                       # acc = 1536 127^2 - 127 = 24774017: odd, above 2^24
    v = tx_i8_ref.s8_product(qa, np.ones(1, np.float32), qw, np.ones(2, np.float32))
    assert v[0, 1] == np.float32(24774017) == 24774016.0 and v[0, 0] == 1536 * 127 * 127


# int8 restatement against the fp8_ffn restatement on the same weights and signal, N = 1, 1920 samples, weights seed 42,
# signal seed 5: how far the int8 QKV rounding points move the scores, a statistic, not a bound on the engine.
# Measured: sup (18 layers) relative L2 0.008, max 0.009 x max|ref|; tx1536 at depth 2 0.002, max 0.003.
I8_VS_FP8 = {"sup": 0.03, "tx1536_d2": 0.01}


@pytest.mark.parametrize("model", ["sup", "tx1536_d2"])
def test_int8_restatement_against_fp8_restatement(model, tmp_path):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    d = SUP if model == "sup" else config_variant(tmp_path, depth=2, name="d2")
    cfg = load_model_config(d)
    w = synthetic_weights(cfg, 42)
    sig = np.random.default_rng(5).standard_normal((1, 1920)).astype(np.float16).astype(np.float32)
    i8 = tx_i8_ref.forward(cfg, w, sig)
    f8 = tx_fp8_ref.forward(cfg, w, sig)
    assert i8.shape == f8.shape and np.isfinite(i8).all()
    rel_l2 = float(np.linalg.norm(i8 - f8) / np.linalg.norm(f8))
    mx = float(np.abs(i8 - f8).max() / np.abs(f8).max())
    print(f"\n[{model}] int8_qkv_fp8_ffn restatement vs fp8_ffn restatement: relative L2 {rel_l2:.3f}, max {mx:.3f} x max|ref|")
    assert 0 < rel_l2 <= I8_VS_FP8[model]


# ---- the launch-by-launch reference -----------------------------------------------------------------------------------
def _sup(tmp_path, depth):
    from dorado_b200.config import load_model_config
    text = (SUP / "config.toml").read_text()
    d = tmp_path / f"sup_d{depth}"
    d.mkdir()
    (d / "config.toml").write_text(text.replace("depth = 18\n", f"depth = {depth}\n"))
    return load_model_config(d)


def test_plan_and_layout(tmp_path):
    cfg = _sup(tmp_path, 2)
    names = tx_i8_ref.launches(cfg)
    assert len(names) == tx_i8_ref.launch_count(cfg) == 1 + 4 + 1 + 14 + 2
    assert [n for n, _, _ in names[5:13]] == ["quantize_i8", "qkv_gemm", "tx_attention", "out_proj_gemm", "rmsnorm_e4m3",
                                              "fc1_swiglu_gemm", "fc2_gemm", "rmsnorm_i8"]
    lay = tx_i8_ref.workspace_layout(cfg, 2, 3072)
    fp8 = X.workspace_layout(cfg, 2, 3072, "fp8_ffn")
    rows, dm = lay["rows"], cfg.tx.d_model
    assert rows == 512
    assert lay["buffers"]["x8"] == (fp8["bytes"], rows * dm)
    assert lay["buffers"]["x_inv"] == (fp8["bytes"] + rows * dm, rows * 4)
    assert lay["bytes"] == fp8["bytes"] + rows * dm + rows * 4


def test_chain_matches_restatement(tmp_path):
    """The per-launch references chained, the int8 copies quantised as the engine does, against tx_i8_ref.forward."""
    from dorado_b200.weights import synthetic_weights
    cfg = _sup(tmp_path, 2)
    w = synthetic_weights(cfg, 42)
    N, T_in = 2, 3072
    sig = np.random.default_rng(5).standard_normal((N, T_in)).astype(np.float16)
    ref = tx_i8_ref.I8LayerRef(cfg, w, N, T_in)
    inp = {"signal": sig.astype(np.float64)}
    for _, kind, idx in tx_i8_ref.launches(cfg):
        if kind == "quantize":
            inp["x"] = inp["x"].astype(np.float16).astype(np.float64)
            q, _, inv = tx_i8_ref.quantize_act(inp["x"])
            inp["x8"], inp["x_inv"] = q, inv
            continue
        for out, (r, _) in ref.reference(kind, idx, inp).items():
            if out == "hid8":
                inp[out] = tx_fp8_ref.e4m3_sat(r).astype(np.float64)
            elif out == "att" and kind == "norm1":
                inp[out] = r.astype(np.float16).astype(np.float64)
                inp["a8"] = tx_fp8_ref.e4m3(inp[out]).astype(np.float64)
            else:
                inp[out] = r.astype(np.float16).astype(np.float64) if out != "scores" else r
            if kind == "norm2":
                q, _, inv = tx_i8_ref.quantize_act(inp["x"])
                inp["x8"], inp["x_inv"] = q, inv
    want = tx_i8_ref.forward(cfg, w, sig.astype(np.float32)).astype(np.float64)
    got = inp["scores"]
    rel_l2 = np.linalg.norm(got - want) / np.linalg.norm(want)
    print(f"\nchain vs tx_i8_ref.forward: relative L2 {rel_l2:.2e}")
    assert rel_l2 < 0.02


@pytest.mark.parametrize("mutation", list(tx_i8_ref.MUTATIONS))
def test_checks_flag_each_mistake(tmp_path, mutation):
    """Each simulated mistake moves the launch's reference at least 3 bounds away from the correct one (at the worst
    element) on plausible inputs, so the GPU check of that launch would fail a kernel that made it."""
    from dorado_b200.weights import synthetic_weights
    cfg = _sup(tmp_path, 2)
    w = synthetic_weights(cfg, 42)
    ref = tx_i8_ref.I8LayerRef(cfg, w, 1, 3072)
    rows, dm = ref.lay["rows"], cfg.tx.d_model
    rng = np.random.default_rng(3)
    x = rng.standard_normal((rows, dm)).astype(np.float16).astype(np.float64)
    q, _, inv = tx_i8_ref.quantize_act(x)
    inp = {"x": x, "x8": q, "x_inv": inv, "y": rng.standard_normal((rows, dm)).astype(np.float16).astype(np.float64) * 3}
    kind = tx_i8_ref.MUTATIONS[mutation]
    (out, (r, bnd)), = ref.reference(kind, 1, inp).items()
    (_, (rm, _)), = ref.reference(kind, 1, inp, mutation=mutation).items()
    engine = r.astype(np.float16).astype(np.float64)   # a correctly rounded kernel
    assert X.worst_ratio(engine, r, bnd) <= 1.0
    ratio = X.worst_ratio(engine, rm, np.abs(bnd))
    print(f"\n[{mutation}] a correct kernel against the mistaken reference: worst ratio {ratio:.1f}")
    assert ratio >= 3.0


# ---- interface ---------------------------------------------------------------------------------------------------------
def test_python_and_header_names():
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    assert L.PRECISIONS["int8_qkv_fp8_ffn"] == (2, 0)
    d = L.model_desc_from_config(load_model_config(SUP), "int8_qkv_fp8_ffn")
    assert (d.tx_precision, d.lstm_precision) == (2, 0)
    header = (ROOT / "include" / "b200call.h").read_text()
    assert "B200_TX_I8_QKV_FP8_FFN = 2" in header
    assert "koi_use_i8" in (ROOT / "include" / "B200ModelRunner.h").read_text()


def _ptxas(log, pattern):
    out = {}
    for block in re.split(r"ptxas info\s*: Compiling entry function ", (BUILD / log).read_text())[1:]:
        m = re.search(pattern, block.split("'")[1])
        if not m:
            continue
        frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        out[m.group(1)] = (int(re.search(r"Used (\d+) registers", block).group(1)), *(int(v) for v in frame.groups()))
    return out


def test_ptxas_reports_no_spills_in_the_row_factor_forms():
    """The GEMM's int8 instantiations with row factors (template ROWS: the RoPE and the plain epilogue), the quantise
    kernel and rmsnorm_kernel with its int8 form: no stack, no spills, and the GEMMs within the 168 registers one 384-thread
    CTA per SM allows."""
    if not (BUILD / "gemm.ptxas.log").is_file() or not (BUILD / "tx_model.ptxas.log").is_file():
        pytest.skip("the ptxas logs are not built")
    gemm = _ptxas("gemm.ptxas.log", r"(gemm_wgmma_kernelIL\w+ELb1EE)")
    tx = _ptxas("tx_model.ptxas.log", r"(quantize_i8_kernel|rmsnorm_kernel)")
    assert set(gemm) == {"gemm_wgmma_kernelILi5ELNS_8GemmTypeE2ELS2_0ELb1EE", "gemm_wgmma_kernelILin1ELNS_8GemmTypeE2ELS2_0ELb1EE"}
    assert set(tx) == {"quantize_i8_kernel", "rmsnorm_kernel"}
    for name, (regs, stack, st, ld) in {**gemm, **tx}.items():
        print(f"\n[{name}] {regs} registers, {stack} B stack, {st} / {ld} B spills")
        assert stack == 0 and st == 0 and ld == 0
    assert all(regs * 384 <= 65536 for regs, *_ in gemm.values())
