"""TEST INFRASTRUCTURE ONLY: numpy restatement of the conv_lstm_v3 modified-base forward.

ModBaseConvLSTMV3Model::forward (dorado/modbase/nn/ModBaseModel.cpp:354-401):
  signal [N,1,T] -> sig_conv1..3, k-mer one-hot [N,T_seq,4k] -> [N,4k,T_seq] -> seq_conv1..2 (every ModsConv pads by
  winlen // 2, :91-97), concatenate along channels, merge_conv1, permute to TNC, lstm1, flip, lstm2, linear, flip back
  (so lstm2 runs reversed in time), optional LinearUpsample (dorado/nn/LinearUpsample.cpp:17-23), softmax over the
  classes, flattened to [N, T_out * num_out].
Checked against the compiled reference in tests/test_modbase_cpu.py.

emulate_fp16 rounds where libb200call.so rounds (dorado_b200/csrc/modbase_model.cu): fp16 weights of the GEMM
convolutions (sig_conv3, seq_conv2, merge_conv1), of the LSTMs and of the head (whose biases are fp16 too); fp32 weights of
sig_conv1/2 and seq_conv1; every activation tensor stored as fp16 except sig_conv1's output, which conv12_kernel keeps in
fp32; gx (W_ih x + b_ih + b_hh) rounded once; the linear and upsample outputs and the probabilities rounded to fp16.
"""
from __future__ import annotations

import ctypes as C
import pathlib
import shutil

import numpy as np

from dorado_b200.config import ModBaseModelConfig
from oracle.nn_oracle import conv1d, lstm_layer


def _q16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def modbase_forward(cfg: ModBaseModelConfig, w: dict, sig: np.ndarray, seq: np.ndarray, emulate_fp16: bool = False,
                    return_intermediates: bool = False):
    """sig [N, chunk_size] (any float dtype), seq [N, T_seq, 4 kmer_len] int8 -> probabilities [N, T_out * num_out]
    float32.  With return_intermediates, also a dict of the merge conv output and both LSTM outputs, [T][N][C]."""
    q = _q16 if emulate_fp16 else (lambda a: np.asarray(a, np.float32))
    wq = q  # weights the engine holds in fp16
    f32 = lambda name: np.asarray(w[name], np.float32)
    m = cfg.modules

    x = np.asarray(sig, np.float32)[:, None, :]
    if emulate_fp16:
        x = _q16(x)
    for i, c in enumerate(m.signal_convs):
        name = f"sig_conv{i + 1}"
        gemm = i == 2
        x = conv1d(x, wq(f32(name + ".weight.tensor")) if gemm else f32(name + ".weight.tensor"), f32(name + ".bias.tensor"),
                   c.stride, c.activation)
        if i > 0:
            x = q(x)
    y = np.asarray(seq, np.float32).transpose(0, 2, 1)
    for i, c in enumerate(m.sequence_convs):
        name = f"seq_conv{i + 1}"
        y = q(conv1d(y, wq(f32(name + ".weight.tensor")) if i == 1 else f32(name + ".weight.tensor"),
                     f32(name + ".bias.tensor"), c.stride, c.activation))
    z = np.concatenate([x, y], axis=1)
    mc = m.merge_conv
    z = q(conv1d(z, wq(f32("merge_conv1.weight.tensor")), f32("merge_conv1.bias.tensor"), mc.stride, mc.activation))
    z = z.transpose(0, 2, 1)  # NTC
    inter = {"merge": z.transpose(1, 0, 2).copy()}
    for l in range(2):
        p = f"lstm{l + 1}."
        z = lstm_layer(z, wq(f32(p + "weight_ih_l0.tensor")), wq(f32(p + "weight_hh_l0.tensor")), f32(p + "bias_ih_l0.tensor"),
                       f32(p + "bias_hh_l0.tensor"), reverse=l == 1, quant=q)
        inter[f"lstm{l + 1}"] = z.transpose(1, 0, 2).copy()
    out = q(z @ wq(f32("fc.weight.tensor")).T + wq(f32("fc.bias.tensor")))
    N, T, K = out.shape
    if m.upsample is not None:
        sf = m.upsample[1]
        out = q(out @ wq(f32("linear_up.linear.weight.tensor")).T + wq(f32("linear_up.linear.bias.tensor")))
        out = out.reshape(N, sf * T, K)
    e = np.exp(out - out.max(axis=-1, keepdims=True))
    p = q(e / e.sum(axis=-1, keepdims=True))
    p = p.reshape(N, -1).astype(np.float32)
    return (p, inter) if return_intermediates else p


class ModBaseReference:
    """The reference's own CPU model and config parser through oracle/_ref/libmodbase_ref.so (modbase_ref_driver.cpp)."""

    PATH = pathlib.Path(__file__).resolve().parent / "_ref" / "libmodbase_ref.so"

    @classmethod
    def available(cls) -> bool:
        return cls.PATH.exists()

    def __init__(self):
        import torch  # noqa: F401  (loads the libtorch the library links against)
        self.lib = lib = C.CDLL(str(self.PATH))
        lib.ref_modbase_last_error.restype = C.c_char_p
        lib.ref_modbase_save_tensor.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.POINTER(C.c_int64)]
        lib.ref_modbase_config.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]
        lib.ref_modbase_create.argtypes = [C.c_char_p]
        lib.ref_modbase_create.restype = C.c_void_p
        lib.ref_modbase_destroy.argtypes = [C.c_void_p]
        lib.ref_modbase_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                            C.c_void_p, C.POINTER(C.c_int)]

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.ref_modbase_last_error().decode())

    def config(self, model_dir) -> list:
        """load_modbase_model_config, flattened as ref_modbase_config documents."""
        out = (C.c_int * 256)()
        n = C.c_int()
        self._check(self.lib.ref_modbase_config(str(model_dir).encode(), out, 256, C.byref(n)))
        return list(out[:n.value])

    def write_model_dir(self, config_dir, weights: dict, work_dir) -> pathlib.Path:
        """A model directory as dorado reads it: config_dir's config.toml and one *.tensor file per weight."""
        work_dir = pathlib.Path(work_dir)
        work_dir.mkdir(parents=True, exist_ok=True)
        shutil.copy(pathlib.Path(config_dir) / "config.toml", work_dir / "config.toml")
        for name, w in weights.items():
            w = np.ascontiguousarray(w, np.float32)
            dims = (C.c_int64 * w.ndim)(*w.shape)
            self._check(self.lib.ref_modbase_save_tensor(str(work_dir / name).encode(), w.ctypes.data, w.ndim, dims))
        return work_dir

    def forward(self, config_dir, weights: dict, work_dir, sig: np.ndarray, seq: np.ndarray) -> np.ndarray:
        """ModBaseConvLSTMV3Model::forward in fp32 on `weights`, through load_modbase_model: the config and the weights are
        written to work_dir as a model directory."""
        self.write_model_dir(config_dir, weights, work_dir)
        h = self.lib.ref_modbase_create(str(work_dir).encode())
        if not h:
            raise RuntimeError(self.lib.ref_modbase_last_error().decode())
        try:
            s = np.ascontiguousarray(sig, np.float32)
            q = np.ascontiguousarray(seq, np.int8)
            N, T = s.shape
            n = C.c_int()
            self._check(self.lib.ref_modbase_forward(h, s.ctypes.data, N, T, q.ctypes.data, q.shape[1], q.shape[2], None,
                                                     C.byref(n)))
            out = np.empty((N, n.value), np.float32)
            self._check(self.lib.ref_modbase_forward(h, s.ctypes.data, N, T, q.ctypes.data, q.shape[1], q.shape[2],
                                                     out.ctypes.data, C.byref(n)))
            return out
        finally:
            self.lib.ref_modbase_destroy(h)
