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
        ("lstm_inner_dim", C.c_int32), ("tx_precision", C.c_int32), ("lstm_precision", C.c_int32),
    ]


# precision name -> (b200_model_desc.tx_precision, b200_model_desc.lstm_precision)
PRECISIONS = {"fp16": (0, 0), "fp8_ffn": (1, 0), "int8_qkv_fp8_ffn": (2, 0), "int8_lstm": (0, 1)}


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


class ModBaseDesc(C.Structure):
    """b200_modbase_desc"""
    _fields_ = [("sig_convs", ConvDesc * 3), ("seq_convs", ConvDesc * 2), ("merge_conv", ConvDesc),
                ("lstm_size", C.c_int32), ("num_out", C.c_int32), ("upsample_scale", C.c_int32),
                ("kmer_len", C.c_int32), ("chunk_size", C.c_int32)]


class GemmTestDesc(C.Structure):
    """b200_gemm_test_desc"""
    _fields_ = [
        ("a", C.c_void_p), ("a_len", C.c_int64), ("w", C.c_void_p), ("w_len", C.c_int64),
        ("bias", C.c_void_p), ("bias_len", C.c_int64), ("residual", C.c_void_p), ("residual_len", C.c_int64),
        ("res_gain", C.c_void_p), ("res_gain_len", C.c_int64), ("a_ss", C.c_void_p), ("a_ss_len", C.c_int64),
        ("res_ss", C.c_void_p), ("res_ss_len", C.c_int64), ("out", C.c_void_p), ("out_len", C.c_int64),
        ("out_ss", C.c_void_p), ("out_ss_len", C.c_int64),
        ("batches", C.c_int32), ("rows_per_batch", C.c_int32), ("a_row_stride", C.c_int64), ("a_batch_stride", C.c_int64),
        ("a_inner", C.c_int32), ("K", C.c_int32), ("N", C.c_int32), ("act", C.c_int32),
        ("out_offset", C.c_int64), ("out_m1", C.c_int64), ("out_s0", C.c_int64), ("out_s1", C.c_int64),
        ("alpha", C.c_float), ("a_ss_parts", C.c_int32), ("res_ss_parts", C.c_int32), ("norm_dim", C.c_int32),
        ("norm_eps", C.c_float), ("max_ctas", C.c_int32), ("theta", C.c_float),
        ("max_seq_len", C.c_int32), ("rope_T", C.c_int32), ("rope_cols", C.c_int32),
        ("in_type", C.c_int32), ("out_type", C.c_int32), ("col_scale", C.c_void_p), ("col_scale_len", C.c_int64),
        ("row_scale", C.c_void_p), ("row_scale_len", C.c_int64),
    ]


# GemmType (dorado_b200/csrc/gemm.h): the element types of b200_gemm_test_desc's in_type and out_type, and their numpy types
GEMM_F16, GEMM_E4M3, GEMM_S8 = 0, 1, 2
GEMM_DTYPES = {GEMM_F16: np.float16, GEMM_E4M3: np.uint8, GEMM_S8: np.int8}


class Stats(C.Structure):
    _fields_ = [("batches_called", C.c_int64), ("model_decode_ms", C.c_double), ("h2d_ms", C.c_double),
                ("d2h_ms", C.c_double), ("gpu_launches", C.c_int64), ("arena_bytes", C.c_int64)]


EXPORTS = [
    "b200_last_error", "b200_version", "b200_device_count", "b200_default_decoder_options", "b200_engine_create", "b200_engine_create_sized",
    "b200_engine_destroy", "b200_engine_get_stats", "b200_runner_create", "b200_runner_destroy",
    "b200_runner_set_decoder_options", "b200_runner_batch_size", "b200_runner_chunk_size", "b200_runner_out_len",
    "b200_runner_accept_chunk_f16", "b200_runner_accept_chunk_f32", "b200_runner_input", "b200_runner_call_chunks",
    "b200_runner_upload", "b200_runner_step_device", "b200_runners_step_device", "b200_runner_forward_scores", "b200_runner_profile", "b200_runner_plan_info", "b200_runner_debug_read_workspace", "b200_decode_scores",
    "b200_test_gemm_desc", "b200_test_quantize_act_rows", "b200_test_quantize_rows", "b200_test_to_e4m3", "b200_test_remove_bits", "b200_test_attention", "b200_generate_chunks", "b200_stitch_chunks", "b200_runner_accept_raw_chunk",
    "b200_runner_debug_read_input", "b200_engine_runner_bytes", "b200_engine_benchmark_batch_sizes",
    "b200_select_batch_size", "b200_generate_variable_chunks", "b200_engine_terminate", "b200_engine_restart",
    "b200_engine_set_low_latency", "b200_engine_is_low_latency", "b200_engine_batch_timeouts_ms",
    "b200_engine_set_num_runners", "b200_engine_num_runners",
    "b200_pool_create", "b200_pool_create_sized", "b200_pool_destroy", "b200_pool_num_runners", "b200_pool_runner", "b200_pool_out_len",
    "b200_pool_runner_info", "b200_pool_call_chunks", "b200_runner_variable_chunk_sizes",
    "b200_runner_accept_chunk_var_f16", "b200_chunk_benchmarks_lookup", "b200_engine_gpu_name",
    "b200_modbase_engine_create", "b200_modbase_engine_destroy", "b200_modbase_runner_create", "b200_modbase_runner_destroy",
    "b200_modbase_runner_batch_size", "b200_modbase_runner_sig_len", "b200_modbase_runner_seq_len",
    "b200_modbase_runner_out_len", "b200_modbase_runner_num_out", "b200_modbase_runner_accept_chunk",
    "b200_modbase_runner_call_chunks", "b200_modbase_runner_profile", "b200_modbase_runner_debug_read_workspace",
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
    lib.b200_pool_create_sized.argtypes = [C.POINTER(ModelDesc), C.c_size_t, C.POINTER(Tensor), i32, C.POINTER(i32), i32, i32, i32,
                                           i32, C.POINTER(vp)]
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
    lib.b200_engine_create_sized.argtypes = [C.POINTER(ModelDesc), C.c_size_t, C.POINTER(Tensor), i32, i32, C.POINTER(vp)]
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
    lib.b200_test_gemm_desc.argtypes = [i32, C.POINTER(GemmTestDesc)]
    lib.b200_test_attention.argtypes = [i32, vp, i32, i32, i32, i32, i32, vp]
    lib.b200_test_quantize_rows.argtypes = [vp, i32, i32, vp, vp]
    lib.b200_test_quantize_act_rows.argtypes = [i32, vp, i32, i32, vp, vp]
    lib.b200_test_to_e4m3.argtypes = [vp, C.c_int64, vp]
    lib.b200_test_remove_bits.argtypes = [vp, C.c_int64, i32, vp]
    u64 = C.c_uint64
    lib.b200_generate_chunks.argtypes = [u64, u64, u64, u64, C.POINTER(u64), u64, C.POINTER(u64)]
    lib.b200_generate_variable_chunks.argtypes = [u64, u64, u64, u64, C.POINTER(u64), u64, C.POINTER(u64)]
    lib.b200_stitch_chunks.argtypes = [C.POINTER(CalledChunk), u64, u64, i32, vp, vp, vp, C.POINTER(u64), C.POINTER(u64)]
    lib.b200_runner_accept_raw_chunk.argtypes = [vp, i32, C.POINTER(RawChunk)]
    lib.b200_runner_debug_read_input.argtypes = [vp, i32, vp]
    lib.b200_engine_runner_bytes.argtypes = [vp, i32, i32, C.POINTER(u64)]
    lib.b200_engine_benchmark_batch_sizes.argtypes = [vp, i32, i32, i32, C.POINTER(i32), C.POINTER(f32), i32, C.POINTER(i32)]
    lib.b200_select_batch_size.argtypes = [C.POINTER(i32), C.POINTER(f32), i32, i32, i32, f32, C.POINTER(i32)]
    lib.b200_modbase_engine_create.argtypes = [C.POINTER(ModBaseDesc), C.POINTER(Tensor), i32, i32, C.POINTER(vp)]
    lib.b200_modbase_engine_destroy.argtypes = [vp]
    lib.b200_modbase_runner_create.argtypes = [vp, i32, C.POINTER(vp)]
    lib.b200_modbase_runner_destroy.argtypes = [vp]
    for fn in ("batch_size", "sig_len", "seq_len", "out_len", "num_out"):
        getattr(lib, "b200_modbase_runner_" + fn).argtypes = [vp]
        getattr(lib, "b200_modbase_runner_" + fn).restype = i32
    lib.b200_modbase_runner_accept_chunk.argtypes = [vp, i32, vp, C.c_int64, vp, C.c_int64]
    lib.b200_modbase_runner_call_chunks.argtypes = [vp, i32, C.POINTER(C.POINTER(C.c_uint16))]
    lib.b200_modbase_runner_profile.argtypes = [vp, C.c_char_p, C.c_uint64]
    lib.b200_modbase_runner_debug_read_workspace.argtypes = [vp, C.c_uint64, C.c_uint64, vp]
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != B200_OK:
        raise B200Error(status, load_library().b200_last_error().decode())


def model_desc_from_config(cfg: BasecallModelConfig, precision: str = "fp16") -> ModelDesc:
    """precision: "fp16" (default), "fp8_ffn" (transformer models: E4M3 feed-forward GEMMs), "int8_qkv_fp8_ffn"
    (transformer models: fp8_ffn with an int8 QKV projection, the reference's default on an H100) or "int8_lstm" (LSTM
    models of lstm_size 256 / 384: int8 LSTM layers and CRF linear); see tx_precision and lstm_precision in b200call.h."""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {precision!r}")
    d = ModelDesc()
    d.tx_precision, d.lstm_precision = PRECISIONS[precision]
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


def modbase_desc_from_config(cfg) -> ModBaseDesc:
    """b200_modbase_desc of a conv_lstm_v3 ModBaseModelConfig (dorado_b200.config.load_modbase_config)."""
    if len(cfg.modules.signal_convs) != 3 or len(cfg.modules.sequence_convs) != 2 or len(cfg.modules.lstms) != 2:
        # the reference's constructor checks (ModBaseModel.cpp:306-315)
        raise ValueError("ModBaseConvLSTMV3Model expects 3 signal convolutions, 2 sequence convolutions and 2 lstms")
    d = ModBaseDesc()
    conv = lambda c: ConvDesc(c.insize, c.size, c.winlen, c.stride, c.activation)
    for i, c in enumerate(cfg.modules.signal_convs):
        d.sig_convs[i] = conv(c)
    for i, c in enumerate(cfg.modules.sequence_convs):
        d.seq_convs[i] = conv(c)
    d.merge_conv = conv(cfg.modules.merge_conv)
    d.lstm_size, d.num_out, d.upsample_scale = cfg.lstm_size, cfg.num_out, cfg.upsample_scale
    d.kmer_len, d.chunk_size = cfg.kmer_len, cfg.chunk_size
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


def test_gemm_desc(a: np.ndarray, w: np.ndarray, out: np.ndarray, *, rows_per_batch: int, a_row_stride: int, out_s0: int,
                   batches: int = 1, a_batch_stride: int = 0, a_inner: int = 0, act: int = -1, out_offset: int = 0,
                   out_m1: int = 1, out_s1: int = 0, bias=None, residual=None, alpha: float = 0.0, res_gain=None,
                   a_ss=None, a_ss_parts: int = 0, res_ss=None, res_ss_parts: int = 0, norm_dim: int = 0,
                   norm_eps: float = 1e-5, max_ctas: int = 0, theta: float = 0.0, max_seq_len: int = 0, rope_T: int = 0,
                   rope_cols: int = 0, out_ss: bool = False, in_type: int = GEMM_F16, out_type: int = GEMM_F16,
                   col_scale=None, row_scale=None, device: int = 0):
    """The GEMM launched from a full descriptor (b200_test_gemm_desc): a is any flat buffer and w [N, K] of in_type, out the
    whole output buffer of out_type with the caller's sentinel in it (GEMM_DTYPES gives the numpy types).  Returns (the
    output buffer after the GEMM, the [rows, N / 32] partial sums of squares or None)."""
    lib = load_library()
    flat = lambda x, t: None if x is None else np.ascontiguousarray(np.ravel(x), t)
    a, res, outb = flat(a, GEMM_DTYPES[in_type]), flat(residual, np.float16), flat(out, GEMM_DTYPES[out_type]).copy()
    w = np.ascontiguousarray(w, GEMM_DTYPES[in_type])
    bias, res_gain, a_ss, res_ss, col_scale, row_scale = (flat(x, np.float32) for x in (bias, res_gain, a_ss, res_ss,
                                                                                         col_scale, row_scale))
    N, K = w.shape
    ss = np.empty((batches * rows_per_batch, N // 32), np.float32) if out_ss else None
    d = GemmTestDesc()
    for name, arr in (("a", a), ("w", w), ("bias", bias), ("residual", res), ("res_gain", res_gain), ("a_ss", a_ss),
                      ("res_ss", res_ss), ("out", outb), ("out_ss", ss), ("col_scale", col_scale), ("row_scale", row_scale)):
        if arr is not None:
            setattr(d, name, arr.ctypes.data)
            setattr(d, name + "_len", arr.size)
    d.batches, d.rows_per_batch, d.a_row_stride, d.a_batch_stride = batches, rows_per_batch, a_row_stride, a_batch_stride
    d.a_inner, d.K, d.N, d.act = a_inner, K, N, act
    d.out_offset, d.out_m1, d.out_s0, d.out_s1 = out_offset, out_m1, out_s0, out_s1
    d.alpha, d.a_ss_parts, d.res_ss_parts, d.norm_dim, d.norm_eps = alpha, a_ss_parts, res_ss_parts, norm_dim, norm_eps
    d.max_ctas, d.theta, d.max_seq_len, d.rope_T, d.rope_cols = max_ctas, theta, max_seq_len, rope_T, rope_cols
    d.in_type, d.out_type = in_type, out_type
    check(lib.b200_test_gemm_desc(device, C.byref(d)))
    return outb, ss


def _test_gemm_dense(a, b, activation, in_type, out_type=GEMM_F16, device=0, **inputs):
    """test_gemm_desc on dense operands a [M, K] and b [N, K] of in_type, K zero-padded to a whole K block (64 fp16 or
    128 one-byte elements): out_type [M, N] (N / 2 with SwiGLU)."""
    a = np.ascontiguousarray(a, GEMM_DTYPES[in_type])
    b = np.ascontiguousarray(b, GEMM_DTYPES[in_type])
    (M, K), N = a.shape, b.shape[0]
    kb = 64 if in_type == GEMM_F16 else 128
    Kp = (K + kb - 1) // kb * kb
    pad = lambda x: np.pad(x, ((0, 0), (0, Kp - K)))
    n_out = N // 2 if activation == 4 else N
    out = np.zeros(M * n_out, GEMM_DTYPES[out_type])
    c, _ = test_gemm_desc(pad(a), pad(b), out, rows_per_batch=M, a_row_stride=Kp, out_s0=n_out, act=activation,
                          in_type=in_type, out_type=out_type, device=device, **inputs)
    return c.reshape(M, n_out)


def test_gemm(a: np.ndarray, b: np.ndarray, bias: np.ndarray | None, activation: int = -1, device: int = 0):
    """The fp16 GEMM on host data: a [M, K], b [N, K] fp16 -> fp16 [M, N] (N / 2 with SwiGLU) of act(a b^T + bias)."""
    return _test_gemm_dense(a, b, activation, GEMM_F16, bias=bias, device=device)


def test_gemm_fp8(a: np.ndarray, b: np.ndarray, activation: int = -1, residual: np.ndarray | None = None,
                  alpha: float = 0.0, device: int = 0):
    """The E4M3 GEMM on host data: a [M, K], b [N, K] E4M3 bytes (uint8) -> fp16 [M, N] (activation -1, optionally
    + alpha * residual [M, N] fp16) or E4M3 bytes [M, N / 2] (activation 4, SwiGLU)."""
    if residual is not None:
        residual = np.ascontiguousarray(residual, np.float16)
        assert residual.shape == (np.shape(a)[0], np.shape(b)[0])
    return _test_gemm_dense(a, b, activation, GEMM_E4M3, GEMM_E4M3 if activation == 4 else GEMM_F16, residual=residual,
                            alpha=alpha, device=device)


def test_gemm_s8(a: np.ndarray, b: np.ndarray, col_scale: np.ndarray, bias: np.ndarray | None = None, activation: int = -1,
                 device: int = 0):
    """The int8 GEMM on host data: a [M, K], b [N, K] int8 -> fp16 [M, N] of act(float(a b^T) * col_scale + bias)."""
    col_scale = np.ascontiguousarray(col_scale, np.float32)
    assert col_scale.shape == (np.shape(b)[0],)
    return _test_gemm_dense(a, b, activation, GEMM_S8, col_scale=col_scale, bias=bias, device=device)


def test_gemm_s8_scaled(a: np.ndarray, b: np.ndarray, row_scale: np.ndarray, col_scale: np.ndarray, activation: int = -1,
                        theta: float = 0.0, max_seq_len: int = 0, rope_T: int = 0, rope_cols: int = 0, device: int = 0):
    """The int8 GEMM with per-row and per-column factors on host data: a [M, K], b [N, K] int8 -> fp16 [M, N] of
    (float(a b^T) * row_scale[m]) * col_scale[n], with RoPE at position m % rope_T on the first rope_cols columns when
    activation is 5."""
    row_scale = np.ascontiguousarray(row_scale, np.float32)
    col_scale = np.ascontiguousarray(col_scale, np.float32)
    assert row_scale.shape == (np.shape(a)[0],) and col_scale.shape == (np.shape(b)[0],)
    return _test_gemm_dense(a, b, activation, GEMM_S8, row_scale=row_scale, col_scale=col_scale, theta=theta,
                            max_seq_len=max_seq_len, rope_T=rope_T, rope_cols=rope_cols, device=device)


def quantize_act_rows(x: np.ndarray, device: int = 0):
    """The int8_qkv_fp8_ffn device quantiser on host fp16 rows [rows, cols] (cols a multiple of 128): (int8 [rows, cols],
    fp32 inv [rows])."""
    h = np.ascontiguousarray(x, np.float16)
    q = np.empty(h.shape, np.int8)
    inv = np.empty(h.shape[0], np.float32)
    check(load_library().b200_test_quantize_act_rows(device, h.ctypes.data, h.shape[0], h.shape[1], q.ctypes.data,
                                                      inv.ctypes.data))
    return q, inv


def quantize_rows(w: np.ndarray):
    """The engine's host quantisation of fp16 values [rows, cols] (no device needed): (int8 [rows, cols], fp16 scale [rows])."""
    h = np.ascontiguousarray(w, np.float16)
    q = np.empty(h.shape, np.int8)
    scale = np.empty(h.shape[0], np.float16)
    check(load_library().b200_test_quantize_rows(h.ctypes.data, h.shape[0], h.shape[1], q.ctypes.data, scale.ctypes.data))
    return q, scale


def to_e4m3(x: np.ndarray) -> np.ndarray:
    """The engine's host cast of fp16 values to E4M3 bytes (no device needed)."""
    h = np.ascontiguousarray(x, np.float16)
    out = np.empty(h.shape, np.uint8)
    check(load_library().b200_test_to_e4m3(h.ctypes.data, h.size, out.ctypes.data))
    return out


def remove_bits(x: np.ndarray, bits: int = 4) -> np.ndarray:
    """The engine's host remove_bits on fp16 values (no device needed); returns fp16."""
    h = np.ascontiguousarray(x, np.float16)
    out = np.empty(h.shape, np.float16)
    check(load_library().b200_test_remove_bits(h.ctypes.data, h.size, bits, out.ctypes.data))
    return out


def test_attention(qkv: np.ndarray, win_upper: int, win_lower: int, device: int = 0):
    """The model's attention kernel on host data: qkv [N, T, 3, H, 64] fp16 -> out [N, T, H * 64] fp16."""
    lib = load_library()
    qkv = np.ascontiguousarray(qkv, np.float16)
    N, T, three, H, D = qkv.shape
    assert three == 3 and D == 64
    out = np.empty((N, T, H * 64), np.float16)
    check(lib.b200_test_attention(device, qkv.ctypes.data, N, T, H, win_upper, win_lower, out.ctypes.data))
    return out
