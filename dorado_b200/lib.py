"""ctypes binding of libb200call.so (the C ABI in include/b200call.h).

The product path is: this binding -> C ABI -> C++ host (engine.cu) -> sm_90a kernels.  There is no
CPU fallback: if the shared library is missing, or there is no sm_90 (H100) device, calls raise.
"""
from __future__ import annotations

import ctypes as C
import pathlib
import subprocess

import numpy as np

from .config import BasecallModelConfig

HERE = pathlib.Path(__file__).resolve().parent
import os as _os
# B200CALL_LIB: load another build of the library (A/B comparisons of two builds)
LIB_PATH = pathlib.Path(_os.environ["B200CALL_LIB"]) if _os.environ.get("B200CALL_LIB") else HERE / "libb200call.so"

B200_OK, B200_ERR_INVALID, B200_ERR_CUDA, B200_ERR_UNSUPPORTED, B200_ERR_INTERNAL = 0, -1, -2, -3, -4


class B200Error(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"b200call error {status}: {msg}")
        self.status = status


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("insize", "size", "winlen", "stride", "activation")]


class ModelDesc(C.Structure):
    _fields_ = [
        ("model_type", C.c_int32), ("num_convs", C.c_int32), ("convs", ConvDesc * 8),
        ("state_len", C.c_int32), ("outsize", C.c_int32), ("stride", C.c_int32), ("clamp", C.c_int32),
        ("qscale", C.c_float), ("qbias", C.c_float),
        ("lstm_size", C.c_int32), ("lstm_layers", C.c_int32), ("linear_bias", C.c_int32),
        ("out_features", C.c_int32), ("crf_scale", C.c_float),
        ("d_model", C.c_int32), ("nhead", C.c_int32), ("dim_feedforward", C.c_int32), ("depth", C.c_int32),
        ("attn_window_upper", C.c_int32), ("attn_window_lower", C.c_int32),
        ("upsample_scale", C.c_int32), ("max_seq_len", C.c_int32),
        ("deepnorm_alpha", C.c_float), ("theta", C.c_float), ("tx_crf_scale", C.c_float),
        ("lstm_inner_dim", C.c_int32),
    ]


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("ndim", C.c_int32), ("dims", C.c_int64 * 4)]


class DecoderOptions(C.Structure):
    _fields_ = [("beam_width", C.c_int32), ("beam_cut", C.c_float), ("blank_score", C.c_float),
                ("q_shift", C.c_float), ("q_scale", C.c_float), ("temperature", C.c_float), ("move_pad", C.c_int32)]


class Result(C.Structure):
    _fields_ = [("moves", C.POINTER(C.c_uint8)), ("sequence", C.POINTER(C.c_char)), ("qstring", C.POINTER(C.c_char)),
                ("n_bases", C.POINTER(C.c_int32)), ("t_out", C.c_int32), ("num_chunks", C.c_int32),
                ("n_moves", C.POINTER(C.c_int32))]


class RawChunk(C.Structure):
    """b200_raw_chunk"""
    _fields_ = [("raw", C.c_void_p), ("num_samples", C.c_uint64), ("input_offset", C.c_uint64), ("shift", C.c_float),
                ("scale", C.c_float)]


class CalledChunk(C.Structure):
    """b200_called_chunk"""
    _fields_ = [("input_offset", C.c_uint64), ("raw_chunk_size", C.c_uint64), ("moves", C.c_void_p),
                ("n_moves", C.c_uint64), ("sequence", C.c_void_p), ("qstring", C.c_void_p), ("n_bases", C.c_uint64)]


class Stats(C.Structure):
    _fields_ = [("batches_called", C.c_int64), ("model_decode_ms", C.c_double), ("h2d_ms", C.c_double),
                ("d2h_ms", C.c_double), ("gpu_launches", C.c_int64), ("arena_bytes", C.c_int64)]


EXPORTS = [
    "b200_last_error", "b200_version", "b200_device_count", "b200_default_decoder_options", "b200_engine_create",
    "b200_engine_destroy", "b200_engine_get_stats", "b200_runner_create", "b200_runner_destroy",
    "b200_runner_set_decoder_options", "b200_runner_batch_size", "b200_runner_chunk_size", "b200_runner_out_len",
    "b200_runner_accept_chunk_f16", "b200_runner_accept_chunk_f32", "b200_runner_input", "b200_runner_call_chunks",
    "b200_runner_upload", "b200_runner_step_device", "b200_runners_step_device", "b200_runner_forward_scores", "b200_runner_profile", "b200_runner_plan_info", "b200_runner_debug_read_workspace", "b200_decode_scores",
    "b200_test_gemm", "b200_generate_chunks", "b200_stitch_chunks", "b200_runner_accept_raw_chunk",
    "b200_runner_debug_read_input", "b200_engine_runner_bytes", "b200_engine_benchmark_batch_sizes",
    "b200_select_batch_size", "b200_generate_variable_chunks", "b200_engine_terminate", "b200_engine_restart",
    "b200_engine_set_low_latency", "b200_engine_is_low_latency", "b200_engine_batch_timeouts_ms",
    "b200_engine_set_num_runners", "b200_engine_num_runners",
    "b200_pool_create", "b200_pool_destroy", "b200_pool_num_runners", "b200_pool_runner", "b200_pool_out_len",
    "b200_pool_runner_info", "b200_pool_call_chunks", "b200_runner_variable_chunk_sizes",
    "b200_runner_accept_chunk_var_f16", "b200_chunk_benchmarks_lookup", "b200_engine_gpu_name",
]

_lib = None


def build_library(verbose: bool = False) -> None:
    """Compile every CUDA source for sm_90a into dorado_b200/libb200call.so (nvcc cross-compiles)."""
    subprocess.run(["make", "-j8", "-C", str(HERE / "csrc")], check=True,
                   stdout=None if verbose else subprocess.DEVNULL)


def load_library() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise FileNotFoundError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`; "
                                "there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    vp, i32, f32 = C.c_void_p, C.c_int32, C.c_float
    lib.b200_last_error.restype = C.c_char_p
    lib.b200_version.restype = C.c_char_p
    lib.b200_default_decoder_options.argtypes = [C.POINTER(DecoderOptions)]
    lib.b200_pool_create.argtypes = [C.POINTER(ModelDesc), C.POINTER(Tensor), i32, C.POINTER(i32), i32, i32, i32, i32,
                                     C.POINTER(vp)]
    lib.b200_pool_destroy.argtypes = [vp]
    lib.b200_pool_num_runners.argtypes = [vp]
    lib.b200_pool_out_len.argtypes = [vp]
    lib.b200_pool_runner.argtypes = [vp, i32]
    lib.b200_pool_runner.restype = vp
    lib.b200_pool_runner_info.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(C.c_int64)]
    lib.b200_pool_call_chunks.argtypes = [vp, vp, C.c_int64, vp, vp, vp, vp, C.POINTER(C.c_double)]
    lib.b200_chunk_benchmarks_lookup.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(i32), C.POINTER(f32), i32, C.POINTER(i32)]
    lib.b200_engine_gpu_name.argtypes = [vp, C.c_char_p, C.c_uint64]
    lib.b200_runner_variable_chunk_sizes.argtypes = [vp]
    lib.b200_runner_variable_chunk_sizes.restype = i32
    lib.b200_runner_accept_chunk_var_f16.argtypes = [vp, i32, vp, C.c_int64]
    lib.b200_engine_terminate.argtypes = [vp]
    lib.b200_engine_restart.argtypes = [vp]
    lib.b200_engine_set_low_latency.argtypes = [vp, i32]
    lib.b200_engine_set_num_runners.argtypes = [vp, i32]
    lib.b200_engine_num_runners.argtypes = [vp]
    lib.b200_engine_num_runners.restype = i32
    lib.b200_engine_is_low_latency.argtypes = [vp]
    lib.b200_engine_is_low_latency.restype = i32
    lib.b200_engine_batch_timeouts_ms.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
    lib.b200_engine_create.argtypes = [C.POINTER(ModelDesc), C.POINTER(Tensor), i32, i32, C.POINTER(vp)]
    lib.b200_engine_destroy.argtypes = [vp]
    lib.b200_engine_get_stats.argtypes = [vp, C.POINTER(Stats)]
    lib.b200_runner_create.argtypes = [vp, i32, i32, C.POINTER(vp)]
    lib.b200_runner_destroy.argtypes = [vp]
    lib.b200_runner_set_decoder_options.argtypes = [vp, C.POINTER(DecoderOptions)]
    for fn in ("b200_runner_batch_size", "b200_runner_chunk_size", "b200_runner_out_len"):
        getattr(lib, fn).argtypes = [vp]
        getattr(lib, fn).restype = i32
    lib.b200_runner_accept_chunk_f16.argtypes = [vp, i32, vp, C.c_int64]
    lib.b200_runner_accept_chunk_f32.argtypes = [vp, i32, vp, C.c_int64]
    lib.b200_runner_input.argtypes = [vp]
    lib.b200_runner_input.restype = C.POINTER(C.c_uint16)
    lib.b200_runner_call_chunks.argtypes = [vp, i32, C.POINTER(Result)]
    lib.b200_runner_upload.argtypes = [vp]
    lib.b200_runner_step_device.argtypes = [vp, i32, i32, C.POINTER(f32), C.POINTER(f32), C.POINTER(f32)]
    lib.b200_runners_step_device.argtypes = [C.POINTER(vp), i32, i32, i32, C.POINTER(f32)]
    lib.b200_runner_forward_scores.argtypes = [vp, i32, vp]
    lib.b200_decode_scores.argtypes = [i32, vp, i32, i32, i32, f32, C.POINTER(DecoderOptions), vp, vp, vp, vp]
    lib.b200_runner_profile.argtypes = [vp, i32, C.c_char_p, C.c_uint64]
    lib.b200_runner_plan_info.argtypes = [vp, C.c_char_p, C.c_uint64]
    lib.b200_runner_debug_read_workspace.argtypes = [vp, C.c_uint64, C.c_uint64, vp]
    lib.b200_test_gemm.argtypes = [i32, vp, vp, vp, i32, i32, i32, i32, vp]
    u64 = C.c_uint64
    lib.b200_generate_chunks.argtypes = [u64, u64, u64, u64, C.POINTER(u64), u64, C.POINTER(u64)]
    lib.b200_generate_variable_chunks.argtypes = [u64, u64, u64, u64, C.POINTER(u64), u64, C.POINTER(u64)]
    lib.b200_stitch_chunks.argtypes = [C.POINTER(CalledChunk), u64, u64, i32, vp, vp, vp, C.POINTER(u64), C.POINTER(u64)]
    lib.b200_runner_accept_raw_chunk.argtypes = [vp, i32, C.POINTER(RawChunk)]
    lib.b200_runner_debug_read_input.argtypes = [vp, i32, vp]
    lib.b200_engine_runner_bytes.argtypes = [vp, i32, i32, C.POINTER(u64)]
    lib.b200_engine_benchmark_batch_sizes.argtypes = [vp, i32, i32, i32, C.POINTER(i32), C.POINTER(f32), i32, C.POINTER(i32)]
    lib.b200_select_batch_size.argtypes = [C.POINTER(i32), C.POINTER(f32), i32, i32, i32, f32, C.POINTER(i32)]
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != B200_OK:
        raise B200Error(status, load_library().b200_last_error().decode())


def model_desc_from_config(cfg: BasecallModelConfig) -> ModelDesc:
    d = ModelDesc()
    d.model_type = 1 if cfg.is_tx_model else 0
    d.num_convs = len(cfg.convs)
    for i, c in enumerate(cfg.convs):
        d.convs[i] = ConvDesc(c.insize, c.size, c.winlen, c.stride, c.activation)
    d.state_len, d.outsize, d.stride, d.clamp = cfg.state_len, cfg.outsize, cfg.stride, int(cfg.clamp)
    d.qscale, d.qbias = cfg.qscale, cfg.qbias
    d.lstm_size, d.lstm_layers = cfg.lstm_size, cfg.lstm_layers
    d.lstm_inner_dim = cfg.lstm_inner_dim or 0
    d.linear_bias, d.out_features, d.crf_scale = int(cfg.bias), cfg.out_features or 0, cfg.scale
    if cfg.tx:
        t = cfg.tx
        d.d_model, d.nhead, d.dim_feedforward, d.depth = t.d_model, t.nhead, t.dim_feedforward, t.depth
        d.attn_window_upper, d.attn_window_lower = t.attn_window
        d.upsample_scale, d.max_seq_len = t.upsample_scale, t.max_seq_len
        d.deepnorm_alpha, d.theta, d.tx_crf_scale = t.deepnorm_alpha, t.theta, t.crf_scale
    return d


def default_decoder_options() -> DecoderOptions:
    o = DecoderOptions()
    load_library().b200_default_decoder_options(C.byref(o))
    return o


def decode_scores(scores: np.ndarray, clamp_val: float = 0.0, opts: DecoderOptions | None = None, device: int = 0):
    """Stage-level entry: fp16 scores [N,T,C] (host) -> (moves u8 [N,T], seq u8 [N,T], qstr u8 [N,T], n_bases)."""
    lib = load_library()
    assert scores.dtype == np.float16 and scores.ndim == 3
    s = np.ascontiguousarray(scores)
    N, T, Cc = s.shape
    opts = opts or default_decoder_options()
    moves = np.zeros((N, T), np.uint8)
    seq = np.zeros((N, T), np.uint8)
    qstr = np.zeros((N, T), np.uint8)
    nb = np.zeros(N, np.int32)
    check(lib.b200_decode_scores(device, s.ctypes.data, N, T, Cc, clamp_val, C.byref(opts), moves.ctypes.data,
                                 seq.ctypes.data, qstr.ctypes.data, nb.ctypes.data))
    return moves, seq, qstr, nb


def test_gemm(a: np.ndarray, b: np.ndarray, bias: np.ndarray | None, activation: int = -1, device: int = 0):
    lib = load_library()
    a = np.ascontiguousarray(a, np.float16)
    b = np.ascontiguousarray(b, np.float16)
    M, K = a.shape
    N = b.shape[0]
    c = np.empty((M, N // 2 if activation == 4 else N), np.float16)
    bias_p = None
    if bias is not None:
        bias = np.ascontiguousarray(bias, np.float32)
        bias_p = bias.ctypes.data
    check(lib.b200_test_gemm(device, a.ctypes.data, b.ctypes.data, bias_p, M, N, K, activation, c.ctypes.data))
    return c
