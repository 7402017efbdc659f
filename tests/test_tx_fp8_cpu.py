"""The fp8_ffn transformer precision without a GPU: the engine's host E4M3 cast and remove_bits (through the C ABI, no device
needed), the FP8 oracle's weight preparation against a torch restatement of the reference's, the FP8 oracle against the fp16
one, and the build's ptxas report of the E4M3 GEMM instantiations.  The GPU side is tests/test_tx_fp8_gpu.py."""
import pathlib
import re

import numpy as np
import pytest
import torch

from conftest import CONFIG_DIR
from test_tx1536_cpu import config_variant
import tx_fp8_ref

ROOT = pathlib.Path(__file__).resolve().parents[1]
PTXAS_LOG = ROOT / "dorado_b200" / "csrc" / "build" / "gemm.ptxas.log"
SUP = CONFIG_DIR / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0"


def _lib():
    from dorado_b200 import lib as L
    try:
        L.load_library()
    except FileNotFoundError:
        pytest.skip("libb200call.so not built")
    return L


ALL_F16 = np.arange(65536, dtype=np.uint32).astype(np.uint16).view(np.float16)


def test_host_e4m3_cast_matches_torch_on_every_fp16():
    """Every fp16 bit pattern (NaN and inf included) cast to E4M3 by the engine's host code and by torch."""
    L = _lib()
    mine = L.to_e4m3(ALL_F16)
    ref = torch.from_numpy(ALL_F16.copy()).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    np.testing.assert_array_equal(mine, ref)


def test_torch_e4m3_beyond_448():
    """What torch (and so the engine's weight cast) does past the largest E4M3 value: round to nearest even up to 464, then
    NaN (0x7f) -- no saturation.  The device's activation casts saturate to 448 instead (tx_fp8_ref.e4m3_sat)."""
    L = _lib()
    v = np.array([448, 456, 464, 464.5, 472, 480, 65504, np.inf, -464, -465], np.float16)
    want = np.array([0x7e, 0x7e, 0x7e, 0x7f, 0x7f, 0x7f, 0x7f, 0x7f, 0xfe, 0xff], np.uint8)
    np.testing.assert_array_equal(torch.from_numpy(v).to(torch.float8_e4m3fn).view(torch.uint8).numpy(), want)
    np.testing.assert_array_equal(L.to_e4m3(v), want)
    assert (tx_fp8_ref.e4m3_sat(np.array([470.0, 1e4, -1e4], np.float32)) == [448, 448, -448]).all()


def _ref_remove_bits(h, bits=4):
    """TxModules.cpp:104-111 in torch: add_ on the int16 view, bitwise_and_ with 0x10000 - 2^bits."""
    t = torch.from_numpy(np.ascontiguousarray(h, np.float16).copy())
    t.view(torch.int16).add_(1 << (bits - 1))
    t.view(torch.int16).bitwise_and_(0x10000 - (1 << bits))
    return t.numpy()


def test_remove_bits_hand_cases():
    L = _lib()
    f = lambda bits: np.array(bits, np.uint16).view(np.float16)
    cases = {
        0x3c00: 0x3c00,   # 1.0: low bits already clear
        0x3c07: 0x3c00,   # below the tie: down
        0x3c08: 0x3c10,   # tie: up (the trick rounds ties away from zero, not to even)
        0x3c18: 0x3c20,   # tie above an odd kept mantissa: up
        0x3c28: 0x3c30,   # tie above an even kept mantissa: also up
        0x3c09: 0x3c10,
        0xbc08: 0xbc10,   # negative tie: away from zero too
        0x3ff8: 0x4000,   # mantissa carry into the exponent
        0x7bf7: 0x7bf0,   # 65280 stays finite
        0x7bf8: 0x7c00,   # 65408 -> inf (the reference's TODO)
        0x7bff: 0x7c00,   # 65504 -> inf
        0xfbff: 0xfc00,   # -65504 -> -inf
        0x0001: 0x0000,   # subnormals round like any other pattern
        0x0008: 0x0010,
    }
    src = f(list(cases))
    want = f(list(cases.values()))
    np.testing.assert_array_equal(_ref_remove_bits(src).view(np.uint16), want.view(np.uint16))
    np.testing.assert_array_equal(tx_fp8_ref.remove_bits(src).view(np.uint16), want.view(np.uint16))
    np.testing.assert_array_equal(L.remove_bits(src).view(np.uint16), want.view(np.uint16))


def test_remove_bits_every_finite_fp16():
    L = _lib()
    fin = ALL_F16[np.isfinite(ALL_F16)]
    ref = _ref_remove_bits(fin).view(np.uint16)
    np.testing.assert_array_equal(L.remove_bits(fin).view(np.uint16), ref)
    np.testing.assert_array_equal(tx_fp8_ref.remove_bits(fin).view(np.uint16), ref)


def _torch_prepare(cfg, w):
    """TxModules.cpp:560-575 and remove_bits() on a model moved to half (CudaCaller.cpp:167): per layer, the values (the
    tiling permutations are layout) of the rounded QKV / out_proj weights and gains and of the E4M3 fc1 / fc2 weights."""
    out = {}
    for l in range(cfg.tx.depth):
        p = f"transformer_encoder.{l}."
        half = {k: torch.from_numpy(np.asarray(w[p + k + ".tensor"], np.float32)).half()
                for k in ("self_attn.Wqkv.weight", "self_attn.out_proj.weight", "norm1.weight", "norm2.weight",
                          "ff.fc1.weight", "ff.fc2.weight")}
        for k in ("self_attn.Wqkv.weight", "self_attn.out_proj.weight", "norm1.weight", "norm2.weight"):
            t = half[k].clone()
            t.view(torch.int16).add_(1 << 3)
            t.view(torch.int16).bitwise_and_(0x10000 - (1 << 4))
            out[p + k] = t.float().numpy()
        fc1 = half["ff.fc1.weight"].unflatten(0, (2, -1, 16)).transpose(0, 1).contiguous()   # (y, gate) interleave
        fc1 = fc1.to(torch.float8_e4m3fn).transpose(0, 1).reshape(half["ff.fc1.weight"].shape)
        out[p + "ff.fc1.weight"] = fc1.float().numpy()
        out[p + "ff.fc2.weight"] = half["ff.fc2.weight"].to(torch.float8_e4m3fn).float().numpy()
    return out


@pytest.mark.parametrize("model", ["sup", "tx1536"])
def test_oracle_weight_preparation_matches_torch(model, tmp_path):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    d = SUP if model == "sup" else config_variant(tmp_path, depth=2, name="d2")
    cfg = load_model_config(d)
    w = synthetic_weights(cfg, 42)
    mine = tx_fp8_ref.prepare_weights(cfg, w)
    ref = _torch_prepare(cfg, w)
    for k, v in ref.items():
        np.testing.assert_array_equal(mine[k], v, err_msg=k)
    # the engine's host conversions give the same values (fc2 of layer 0 and the rounded gains)
    L = _lib()
    p = "transformer_encoder.0."
    np.testing.assert_array_equal(tx_fp8_ref.decode_e4m3(L.to_e4m3(np.asarray(w[p + "ff.fc2.weight.tensor"], np.float16))),
                                  ref[p + "ff.fc2.weight"])
    np.testing.assert_array_equal(L.remove_bits(np.asarray(w[p + "norm1.weight.tensor"], np.float16)).astype(np.float32),
                                  ref[p + "norm1.weight"])
    changed = float((mine[p + "self_attn.Wqkv.weight"] != _q16(w[p + "self_attn.Wqkv.weight.tensor"])).mean())
    assert changed > 0.5   # remove_bits does round most weights


def _q16(a):
    return np.asarray(a, np.float16).astype(np.float32)


# FP8 oracle against the fp16-emulating oracle (oracle/nn_oracle.py) on the same weights and signal, N = 1, 1920 samples
# (160 tokens), weights seed 42, signal seed 5.  A record of how far the rounding points move the scores, not a bound on the
# engine.  Measured: sup (18 layers) relative L2 0.026, max 0.032 x max|ref|; tx1536 at depth 2 relative L2 0.009, max 0.011.
FP8_VS_FP16 = {"sup": (0.04, 0.06), "tx1536_d2": (0.015, 0.02)}


@pytest.mark.parametrize("model", ["sup", "tx1536_d2"])
def test_fp8_oracle_against_fp16_oracle(model, tmp_path):
    from oracle import nn_oracle
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    d = SUP if model == "sup" else config_variant(tmp_path, depth=2, name="d2")
    cfg = load_model_config(d)
    w = synthetic_weights(cfg, 42)
    sig = np.random.default_rng(5).standard_normal((1, 1920)).astype(np.float16).astype(np.float32)
    f8 = tx_fp8_ref.forward(cfg, w, sig)
    f16 = nn_oracle.forward(cfg, w, sig, emulate_fp16=True)
    assert f8.shape == f16.shape and np.isfinite(f8).all()
    rel_l2 = float(np.linalg.norm(f8 - f16) / np.linalg.norm(f16))
    mx = float(np.abs(f8 - f16).max() / np.abs(f16).max())
    print(f"\n[{model}] FP8 oracle vs fp16 oracle: relative L2 {rel_l2:.3f}, max {mx:.3f} x max|ref|")
    assert 0 < rel_l2 <= FP8_VS_FP16[model][0] and mx <= FP8_VS_FP16[model][1]


def _ptxas_entries():
    text = PTXAS_LOG.read_text()
    out = {}
    for block in re.split(r"ptxas info\s*: Compiling entry function ", text)[1:]:
        name = block.split("'")[1]
        m = re.search(r"gemm_wgmma_kernelILi(n?\d+)ELNS_8GemmTypeE(\d)E", name)   # activation, operand type
        if not m:
            continue
        frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        out[(m.group(1).replace("n", "-"), m.group(2) == "1")] = (regs, *(int(x) for x in frame.groups()))
    return out


def test_ptxas_reports_no_spills_in_the_e4m3_forms():
    """The E4M3 instantiations (plain and SwiGLU epilogues; one kernel serves sup's and tx1536's shapes, the shapes are
    run-time parameters): no stack, no spills, and within the 168 registers one 384-thread CTA per SM allows."""
    if not PTXAS_LOG.is_file():
        pytest.skip("dorado_b200/csrc/build/gemm.ptxas.log not built")
    e = _ptxas_entries()
    for key in (("-1", True), ("4", True)):
        assert key in e, f"no E4M3 gemm_wgmma_kernel<{key[0]}> in the ptxas log"
        regs, stack, st, ld = e[key]
        print(f"\n[gemm_wgmma_kernel<{key[0]}, fp8>] {regs} registers, {stack} B stack, {st} / {ld} B spills")
        assert stack == 0 and st == 0 and ld == 0
        assert regs * 384 <= 65536
    assert sorted(k for k in e if k[1]) == [("-1", True), ("4", True)]   # no other E4M3 instantiation is built
