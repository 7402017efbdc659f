"""The int8_lstm precision without a device: the host weight quantisation against the reference's quantize_tensor
arithmetic run by torch on fp16 tensors, the numpy restatement (tests/lstm_int8_ref.py) against the fp16-emulating oracle,
the Python interface, and the compiler's report for the new kernels."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

import lstm_int8_ref
from conftest import ROOT, model_dir
from test_lstm128_256_cpu import model_dir as synthetic_model_dir

BUILD = ROOT / "dorado_b200" / "csrc" / "build"


def _cfg_w(kind):
    from dorado_b200.config import load_model_config
    from dorado_b200.weights import synthetic_weights
    cfg = load_model_config(model_dir("hac") if kind == "hac" else synthetic_model_dir(kind))
    return cfg, synthetic_weights(cfg, 42)


def _torch_quantize(w16):
    """utils::quantize_tensor(t, 1) (torch_utils/tensor_utils.cpp:293-300) on an fp16 CPU tensor; the scale as the callers
    store it (.to(kF16))."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(w16, np.float16))
    fp_range = t.abs().amax(1)
    quant_scale = (256 / 2) / fp_range
    t_quant = (t * quant_scale.unsqueeze(1)).round().clip(-127, 127)
    return t_quant.to(torch.int8).numpy(), quant_scale.to(torch.float32).to(torch.float16).numpy()


def _check_against_torch(w16):
    from dorado_b200 import lib as L
    q, scale = L.quantize_rows(w16)
    tq, tscale = _torch_quantize(w16)
    np.testing.assert_array_equal(scale.view(np.uint16), tscale.view(np.uint16))
    np.testing.assert_array_equal(q, tq)
    rq, rscale, _ = lstm_int8_ref.quantize_rows(w16)
    np.testing.assert_array_equal(q, rq)
    np.testing.assert_array_equal(scale.view(np.uint16), rscale.view(np.uint16))
    return q


@pytest.mark.parametrize("kind", ["hac", "lstm256"])
def test_quantize_rows_matches_quantize_tensor_on_model_weights(kind):
    cfg, w = _cfg_w(kind)
    for l in range(cfg.lstm_layers):
        p = f"{len(cfg.convs) + l + 1}.rnn."
        both = np.concatenate([w[p + "weight_ih_l0.tensor"], w[p + "weight_hh_l0.tensor"]], axis=1).astype(np.float16)
        assert both.shape == (4 * cfg.lstm_size, 2 * cfg.lstm_size)
        q = _check_against_torch(both)
        assert np.abs(q).max(axis=1).min() >= 126   # every row uses the range: the quantiser is per row
    layer = len(cfg.convs) + cfg.lstm_layers + 1
    _check_against_torch(np.asarray(w[f"{layer}.linear.weight.tensor"], np.float16))


def test_quantize_rows_ties_extremes_and_zero_row():
    from dorado_b200 import lib as L
    rng = np.random.default_rng(3)
    rows = []
    # absmax 1 -> scale 128: w = (k + 0.5) / 128 lands exactly on a rounding tie, +-1 on +-128 before the clip
    rows.append(np.concatenate([[1.0, -1.0], (np.arange(-30, 30) + 0.5) / 128.0]))
    # absmax 0.5 -> scale 256; odd multiples of 1 / 512 are ties
    rows.append(np.concatenate([[0.5, -0.5], (2 * np.arange(-30, 30) + 1) / 512.0]))
    # scales that are not powers of two, where 128 / absmax and w * scale both round in fp16
    for amax in (0.3, 0.7371, 1.337, 3.1, 1e-3, 250.0):
        rows.append(np.concatenate([[amax, -amax], rng.uniform(-amax, amax, 60)]))
    w16 = np.asarray(rows, np.float16)
    q = _check_against_torch(w16)
    assert (q[:, 0] == 127).all() and (q[:, 1] == -127).all()   # +-absmax * scale is about 128 and is clipped
    np.testing.assert_array_equal(q[0, 2:6], np.rint((np.arange(-30, -26) + 0.5)).astype(np.int8))   # ties go to even
    # an all-zero row: the reference divides by zero; the engine gives q = 0, scale = inf and a dequantisation factor of 0
    z = np.zeros((2, 64), np.float16)
    z[1, 5] = 0.25
    qz, sz = L.quantize_rows(z)
    assert (qz[0] == 0).all() and np.isinf(sz[0]) and qz[1, 5] == 127
    rq, _, rinv = lstm_int8_ref.quantize_rows(z)
    assert (rq[0] == 0).all() and rinv[0] == 0 and rinv[1] == np.float32(1) / (np.float32(127) * np.float32(512))


def test_quantize_rows_rejects_bad_arguments():
    from dorado_b200 import lib as L
    lib = L.load_library()
    assert lib.b200_test_quantize_rows(None, 1, 1, None, None) == L.B200_ERR_INVALID


# int8 restatement against the fp16-emulating oracle (oracle/nn_oracle.py), N = 2, 1200 samples, weights seed 42, signal
# seed 5: how far the int8 rounding points move the scores of these synthetic models, not a bound on the engine.
# Measured: hac relative L2 0.034, lstm256 0.035.
INT8_VS_FP16 = {"hac": 0.09, "lstm256": 0.07}


@pytest.mark.parametrize("kind", ["hac", "lstm256"])
def test_int8_restatement_against_the_fp16_oracle(kind):
    from oracle import nn_oracle
    cfg, w = _cfg_w(kind)
    sig = np.random.default_rng(5).standard_normal((2, 1200)).astype(np.float16).astype(np.float32)
    i8, inter = lstm_int8_ref.forward(cfg, w, sig, return_intermediates=True)
    f16, inter16 = nn_oracle.forward(cfg, w, sig, emulate_fp16=True, return_intermediates=True)
    assert i8.shape == f16.shape and np.isfinite(i8).all()
    # conv3's int8 output is the fp16 path's output to within half a level and the fp16 rounding
    conv = inter16["conv2"].transpose(0, 2, 1)
    assert np.abs(inter["conv2"].astype(np.float32) / 127.0 - conv).max() <= 0.5 / 127 + 2.0 ** -11
    rel = float(np.linalg.norm(i8 - f16) / np.linalg.norm(f16))
    print(f"\n[{kind}] int8 restatement vs fp16 oracle: score relative L2 {rel:.3f}")
    assert 0 < rel <= INT8_VS_FP16[kind]


def test_model_desc_precision_strings():
    from dorado_b200 import lib as L
    cfg, _ = _cfg_w("hac")
    d = L.model_desc_from_config(cfg, "int8_lstm")
    assert (d.lstm_precision, d.tx_precision) == (1, 0)
    assert L.model_desc_from_config(cfg).lstm_precision == 0
    assert L.model_desc_from_config(cfg, "fp8_ffn").lstm_precision == 0
    for bad in ("fp8", "int8", "INT8_LSTM", ""):
        with pytest.raises(ValueError):
            L.model_desc_from_config(cfg, bad)
    assert L.ModelDesc._fields_[-1][0] == "lstm_precision"


def test_model_desc_size_matches_the_header(tmp_path):
    from dorado_b200 import lib as L
    src = tmp_path / "size.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200call.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(b200_model_desc), offsetof(b200_model_desc, lstm_precision),'
                   ' offsetof(b200_model_desc, tx_precision)); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run(["cc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    size, off_lstm, off_tx = (int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    assert size == C.sizeof(L.ModelDesc)
    assert off_lstm == L.ModelDesc.lstm_precision.offset == size - 4   # the last field
    assert off_tx == L.ModelDesc.tx_precision.offset


def test_descriptor_size_rules():
    """b200_engine_create_sized reads what the caller's header declares; the exported b200_engine_create is for binaries built
    before lstm_precision and never looks at the bytes behind tx_precision.  All of this is decided before a device is needed."""
    from dorado_b200 import lib as L
    from dorado_b200.runner import _weight_array
    lib = L.load_library()
    cfg, _ = _cfg_w("hac")
    arr, keep = _weight_array({"x": np.zeros(1, np.float32)})
    full, old = C.sizeof(L.ModelDesc), L.ModelDesc.lstm_precision.offset
    assert old == L.ModelDesc.tx_precision.offset + 4
    buf = (C.c_ubyte * (full + 16))()
    desc = L.model_desc_from_config(cfg)
    desc.lstm_precision = 7
    C.memmove(buf, C.byref(desc), full)
    p = C.cast(buf, C.POINTER(L.ModelDesc))
    handle = C.c_void_p()
    create = lambda size: (lib.b200_engine_create_sized(p, size, arr, 1, 0, C.byref(handle)), lib.b200_last_error().decode())
    status, msg = create(full)
    assert status == L.B200_ERR_INVALID and "lstm_precision must be" in msg
    status, msg = create(old - 4)
    assert status == L.B200_ERR_INVALID and "desc_size" in msg
    # declared without the field, or through the earlier symbol, the bad value is never read: creation gets as far as the
    # device (no device here: B200_ERR_CUDA) or the weights (a device: the tensor "x" is not a model's)
    for status, msg in (create(old), (lib.b200_engine_create(p, arr, 1, 0, C.byref(handle)), lib.b200_last_error().decode())):
        assert status != 0 and "lstm_precision" not in msg and "desc_size" not in msg, msg
    # a longer descriptor, from a later header: fine while the fields this library does not know are zero
    desc.lstm_precision = 0
    C.memmove(buf, C.byref(desc), full)
    assert "does not know" not in create(full + 16)[1]
    buf[full + 3] = 1
    status, msg = create(full + 16)
    assert status == L.B200_ERR_UNSUPPORTED and "does not know" in msg


def _entries(log, pattern):
    out = {}
    for block in re.split(r"ptxas info\s*: Compiling entry function ", (BUILD / log).read_text())[1:]:
        m = re.search(pattern, block.split("'")[1])
        if not m:
            continue
        frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        out[m.groups()] = (regs, *(int(x) for x in frame.groups()))
    return out


def test_ptxas_reports_no_spills_in_the_int8_kernel_forms():
    """The int8 instantiations: no stack, no spills, within the registers one CTA per SM of their block size allows."""
    if not (BUILD / "gemm.ptxas.log").is_file() or not (BUILD / "lstm_model.ptxas.log").is_file():
        pytest.skip("the ptxas logs are not built")
    forms = _entries("gemm.ptxas.log", r"gemm_wgmma_kernelILi(n?\d+)ELNS_8GemmTypeE(\d)ELS\d+_(\d)ELb([01])EE")
    # (activation, operand type, output type, row factors), GemmType 0 fp16, 2 int8: int8 operands with the plain and
    # tanh x 5 epilogues, fp16 operands with the int8 tanh store
    gemm = {k: v for k, v in forms.items() if (k[1] == "2" and k[3] == "0") or k[2] == "2"}
    assert sorted(gemm) == [("2", "0", "2", "0"), ("3", "2", "0", "0"), ("n1", "2", "0", "0")]
    for key, (regs, stack, st, ld) in gemm.items():
        print(f"\n[gemm_wgmma_kernel<{key}>] {regs} registers, {stack} B stack, {st} / {ld} B spills")
        assert stack == 0 and st == 0 and ld == 0 and regs * 384 <= 65536
    rec = _entries("lstm_model.ptxas.log", r"lstm_rec_kernelILb1ELi(\d+)ELi(\d+)ELi(\d+)EE")
    assert sorted(rec) == sorted((str(c), "8", str(nb)) for c in (256, 384) for nb in (16, 32, 64))
    for (c, cl, nb), (regs, stack, st, ld) in sorted(rec.items()):
        threads = 32 * (4 * int(c) // int(cl)) // 16
        print(f"[lstm_rec_kernel<true, {c}, {cl}, {nb}>] {regs} registers, {stack} B stack, {st} / {ld} B spills")
        assert stack == 0 and st == 0 and ld == 0 and regs * threads <= 65536
