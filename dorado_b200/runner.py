"""Python mirror of the reference runner interface on top of the C ABI.

``B200ModelRunner`` has the methods of ``dorado::basecall::ModelRunnerBase``
(dorado/basecall/include/basecall/ModelRunnerBase.h:20-38) with numpy arrays where the reference takes
``at::Tensor``: ``accept_chunk(idx, chunk)``, ``call_chunks(n) -> [DecodedChunk]``, ``config()``,
``chunk_size()``, ``batch_size()``, ``batch_timeouts_ms()``, ``terminate()``, ``restart()``,
``get_name()``, ``sample_stats()``.  ``B200Caller`` is the per-device engine (the reference's
``CudaCaller``); several runners may share one caller and are serialised per GPU like
``CudaCaller::call_chunks`` (dorado/basecall/CudaCaller.cpp:224-271).

The C++ adapter a dorado maintainer would use is include/B200ModelRunner.h; this module is the same
thing for the Python tests and bench.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import itertools
from typing import List

import numpy as np

from . import lib as L
from .config import BasecallModelConfig


@dataclasses.dataclass
class DecodedChunk:
    """decode::DecodedChunk (dorado/basecall/include/basecall/DecodedChunk.h:9-13)."""
    sequence: str
    qstring: str
    moves: np.ndarray


class B200Caller:
    """One model replica on one GPU (CudaCaller, dorado/basecall/CudaCaller.cpp:149-202)."""

    def __init__(self, cfg: BasecallModelConfig, weights: dict, device: int = 0, low_latency: bool = False,
                 num_runners: int = 2, precision: str = "fp16"):
        """precision: "fp16", "fp8_ffn" (transformer models: fc1 / fc2 on E4M3 operands), "int8_qkv_fp8_ffn" (transformer
        models: fp8_ffn with the QKV projection on int8 operands) or "int8_lstm" (LSTM models of lstm_size 256 / 384: int8
        LSTM layers and CRF linear); include/b200call.h."""
        self.cfg = cfg
        self.device = device
        self.precision = precision
        lib = L.load_library()
        desc = L.model_desc_from_config(cfg, precision)
        self._keep = []
        arr = (L.Tensor * len(weights))()
        for i, (name, w) in enumerate(weights.items()):
            w = np.ascontiguousarray(w, np.float32)
            self._keep.append(w)
            arr[i].name = name.encode()
            arr[i].data = w.ctypes.data_as(C.POINTER(C.c_float))
            arr[i].ndim = w.ndim
            for k, dim in enumerate(w.shape):
                arr[i].dims[k] = dim
        self.handle = C.c_void_p()
        L.check(lib.b200_engine_create_sized(C.byref(desc), C.sizeof(desc), arr, len(weights), device, C.byref(self.handle)))
        self._keep = None  # the engine copied everything to the device
        L.check(lib.b200_engine_set_low_latency(self.handle, int(low_latency)))
        # api::create_basecall_runners' num_runners (api/runner_creation.cpp:46-130): shapes launch plans only
        L.check(lib.b200_engine_set_num_runners(self.handle, int(num_runners)))

    def terminate(self) -> None:
        """CudaCaller::terminate (CudaCaller.cpp:273-280): refuse new batches, wait for the ones in flight."""
        L.check(L.load_library().b200_engine_terminate(self.handle))

    def restart(self) -> None:
        """CudaCaller::restart (CudaCaller.cpp:282-287); idempotent."""
        L.check(L.load_library().b200_engine_restart(self.handle))

    def is_low_latency(self) -> bool:
        return bool(L.load_library().b200_engine_is_low_latency(self.handle))

    def batch_timeouts_ms(self):
        a, b = C.c_int32(), C.c_int32()
        L.check(L.load_library().b200_engine_batch_timeouts_ms(self.handle, C.byref(a), C.byref(b)))
        return a.value, b.value

    def runner_bytes(self, batch_size: int, chunk_size: int) -> int:
        """Device bytes a runner of this shape allocates (exact; CudaCaller::calculate_memory_requirements estimates it)."""
        n = C.c_uint64()
        L.check(L.load_library().b200_engine_runner_bytes(self.handle, batch_size, chunk_size, C.byref(n)))
        return int(n.value)

    def benchmark_batch_sizes(self, chunk_size: int, granularity: int, max_batch_size: int):
        """determine_batch_dims' timing loop (CudaCaller.cpp:530-557): [(batch_size, ms per chunk), ...]."""
        cap = max(1, max_batch_size // max(1, granularity))
        bs = (C.c_int32 * cap)()
        ms = (C.c_float * cap)()
        n = C.c_int32()
        L.check(L.load_library().b200_engine_benchmark_batch_sizes(self.handle, chunk_size, granularity, max_batch_size, bs, ms, cap,
                                                            C.byref(n)))
        return [(int(bs[i]), float(ms[i])) for i in range(min(cap, n.value))]

    def stats(self) -> dict:
        s = L.Stats()
        L.check(L.load_library().b200_engine_get_stats(self.handle, C.byref(s)))
        return {k: getattr(s, k) for k, _ in L.Stats._fields_}

    def close(self):
        if self.handle:
            L.load_library().b200_engine_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _weight_array(weights: dict):
    keep = []
    arr = (L.Tensor * len(weights))()
    for i, (name, w) in enumerate(weights.items()):
        w = np.ascontiguousarray(w, np.float32)
        keep.append(w)
        arr[i].name = name.encode()
        arr[i].data = w.ctypes.data_as(C.POINTER(C.c_float))
        arr[i].ndim = w.ndim
        for k, dim in enumerate(w.shape):
            arr[i].dims[k] = dim
    return arr, keep


class B200Pool:
    """Several devices in one process: api::create_basecall_runners + BasecallerNode's worker loop
    (dorado/api/runner_creation.cpp:46-130, read_pipeline/nodes/BasecallerNode.cpp:300-352) -- one engine per device,
    `runners_per_device` runners each, one pinned host thread per runner, batches taken from one shared cursor."""

    def __init__(self, cfg: BasecallModelConfig, weights: dict, devices, runners_per_device: int, batch_size: int,
                 chunk_size: int, precision: str = "fp16"):
        self.cfg = cfg
        self._lib = lib = L.load_library()
        desc = L.model_desc_from_config(cfg, precision)
        arr, keep = _weight_array(weights)
        devs = (C.c_int32 * len(devices))(*devices)
        self.chunk_size = cfg.normalise_chunk_size(chunk_size)
        self.batch_size = batch_size
        self.handle = C.c_void_p()
        L.check(lib.b200_pool_create_sized(C.byref(desc), C.sizeof(desc), arr, len(weights), devs, len(devices),
                                           runners_per_device, batch_size, self.chunk_size, C.byref(self.handle)))
        del keep
        self.t_out = lib.b200_pool_out_len(self.handle)

    def num_runners(self) -> int:
        return self._lib.b200_pool_num_runners(self.handle)

    def runner_info(self, i: int):
        node, batches = C.c_int32(), C.c_int64()
        L.check(self._lib.b200_pool_runner_info(self.handle, i, C.byref(node), C.byref(batches)))
        return {"numa_node": node.value, "batches": batches.value}

    def call_chunks(self, chunks: np.ndarray, want_output: bool = True):
        """chunks: fp16 [n, chunk_size].  Returns (seconds, moves, sequence, qstring, n_bases)."""
        c = np.ascontiguousarray(chunks, np.float16)
        n = c.shape[0]
        assert c.shape[1] == self.chunk_size
        secs = C.c_double()
        if not want_output:
            L.check(self._lib.b200_pool_call_chunks(self.handle, c.ctypes.data, n, None, None, None, None, C.byref(secs)))
            return secs.value, None, None, None, None
        moves, seq, qs = (np.zeros((n, self.t_out), np.uint8) for _ in range(3))
        nb = np.zeros(n, np.int32)
        L.check(self._lib.b200_pool_call_chunks(self.handle, c.ctypes.data, n, moves.ctypes.data, seq.ctypes.data,
                                                qs.ctypes.data, nb.ctypes.data, C.byref(secs)))
        return secs.value, moves, seq, qs, nb

    def close(self):
        if self.handle:
            self._lib.b200_pool_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200ModelRunner:
    _ids = itertools.count()

    def __init__(self, caller: B200Caller, batch_size: int, chunk_size: int):
        self.caller = caller
        self._lib = L.load_library()
        self.handle = C.c_void_p()
        chunk_size = caller.cfg.normalise_chunk_size(chunk_size)
        L.check(self._lib.b200_runner_create(caller.handle, batch_size, chunk_size, C.byref(self.handle)))
        self._name = f"B200ModelRunner_{caller.device}_{next(self._ids)}"
        self._N, self._T = batch_size, chunk_size
        self._t_out = self._lib.b200_runner_out_len(self.handle)
        buf = self._lib.b200_runner_input(self.handle)
        self._input = np.ctypeslib.as_array(buf, shape=(batch_size, chunk_size)).view(np.float16)

    # --- ModelRunnerBase ---------------------------------------------------------------------
    def accept_chunk(self, chunk_idx: int, chunk: np.ndarray) -> None:
        """chunk: [1, chunk_size] or [chunk_size], float16 (CUDA dtype) or float32."""
        c = np.ascontiguousarray(chunk).reshape(-1)
        if c.dtype == np.float16:
            L.check(self._lib.b200_runner_accept_chunk_f16(self.handle, chunk_idx, c.ctypes.data, c.size))
        else:
            c = c.astype(np.float32, copy=False)
            L.check(self._lib.b200_runner_accept_chunk_f32(self.handle, chunk_idx, c.ctypes.data, c.size))

    def accept_chunk_var(self, chunk_idx: int, chunk: np.ndarray) -> None:
        """Variable chunk sizes (CudaModelRunner::accept_chunk, CudaModelRunner.cpp:21-31): fp16 chunk of any length that is
        a positive multiple of the stride and <= chunk_size."""
        c = np.ascontiguousarray(chunk, np.float16).reshape(-1)
        L.check(self._lib.b200_runner_accept_chunk_var_f16(self.handle, chunk_idx, c.ctypes.data, c.size))

    def accept_raw_chunk(self, chunk_idx: int, raw: np.ndarray, input_offset: int, shift: float, scale: float) -> None:
        """One chunk of a read given as its whole RAW int16 signal: ScalerNode's (x - shift) / scale
        (ScalerNode.cpp:226-229), BasecallerNode's slice + repeat-padding (BasecallerNode.cpp:395-440) run on the
        device at the next call_chunks.  `raw` is only read during this call."""
        r = np.ascontiguousarray(raw, np.int16).reshape(-1)
        c = L.RawChunk(r.ctypes.data, r.size, int(input_offset), float(shift), float(scale))
        L.check(self._lib.b200_runner_accept_raw_chunk(self.handle, chunk_idx, C.byref(c)))

    def debug_read_input(self, num_chunks: int) -> np.ndarray:
        """Run only the input stage and read the device-side fp16 batch input back: [num_chunks, chunk_size]."""
        out = np.empty((num_chunks, self._T), np.float16)
        L.check(self._lib.b200_runner_debug_read_input(self.handle, num_chunks, out.ctypes.data))
        return out

    def call_chunks_raw(self, num_chunks: int):
        """The bare C-ABI call (what the C++ adapter makes): H2D, forward, decode, D2H; returns views of the runner's
        pinned result buffers (moves [N,T], sequence [N,T], qstring [N,T], n_bases [N]), valid until the next call."""
        r = L.Result()
        L.check(self._lib.b200_runner_call_chunks(self.handle, num_chunks, C.byref(r)))
        T = r.t_out
        moves = np.ctypeslib.as_array(r.moves, shape=(self._N, T))
        seq = np.ctypeslib.as_array(C.cast(r.sequence, C.POINTER(C.c_uint8)), shape=(self._N, T))
        qs = np.ctypeslib.as_array(C.cast(r.qstring, C.POINTER(C.c_uint8)), shape=(self._N, T))
        nb = np.ctypeslib.as_array(r.n_bases, shape=(self._N,))
        self._n_moves = np.ctypeslib.as_array(r.n_moves, shape=(self._N,))   # == t_out unless variable chunk sizes are in use
        return moves, seq, qs, nb

    def call_chunks(self, num_chunks: int) -> List[DecodedChunk]:
        moves, seq, qs, nb = self.call_chunks_raw(num_chunks)
        out = []
        for i in range(num_chunks):
            n = int(nb[i])
            out.append(DecodedChunk(bytes(seq[i, :n]).decode("ascii"), bytes(qs[i, :n]).decode("ascii"),
                                    moves[i, :int(self._n_moves[i])].copy()))
        return out

    def config(self) -> BasecallModelConfig:
        return self.caller.cfg

    def chunk_size(self) -> int:
        return self._T

    def batch_size(self) -> int:
        return self._N

    def variable_chunk_sizes(self) -> bool:
        return bool(self._lib.b200_runner_variable_chunk_sizes(self.handle))

    def batch_timeouts_ms(self):
        return self.caller.batch_timeouts_ms()  # CudaCaller.cpp:216-222

    def is_low_latency(self) -> bool:
        return self.caller.is_low_latency()

    def terminate(self) -> None:
        self.caller.terminate()  # CudaModelRunner::terminate -> CudaCaller::terminate (CudaModelRunner.cpp:62)

    def restart(self) -> None:
        self.caller.restart()

    def get_name(self) -> str:
        return self._name

    def sample_stats(self) -> dict:
        s = self.caller.stats()
        return {"batches_called": float(s["batches_called"]), "model_decode_ms": float(s["model_decode_ms"])}

    # --- stage-level / measurement hooks -------------------------------------------------------
    def input_view(self) -> np.ndarray:
        """Pinned fp16 [batch, chunk_size] input buffer (asking for it turns raw slots back into fp16 slots)."""
        self._lib.b200_runner_input(self.handle)
        return self._input

    def forward_scores(self, num_chunks: int) -> np.ndarray:
        out = np.empty((num_chunks, self._t_out, self.caller.cfg.outsize), np.float16)
        L.check(self._lib.b200_runner_forward_scores(self.handle, num_chunks, out.ctypes.data))
        return out

    def profile(self, num_chunks: int):
        """One forward+decode pass timed per launch: [(kernel name, ms), ...] in launch order."""
        buf = C.create_string_buffer(8192)
        L.check(self._lib.b200_runner_profile(self.handle, num_chunks, buf, len(buf)))
        out = []
        for item in buf.value.decode().split(";"):
            if item:
                k, v = item.split("=")
                out.append((k, float(v)))
        return out

    def plan_info(self) -> dict:
        """Launch-plan facts (grid sizes of kernels sized for a share of the SMs): {"lstm_layer.ctas": 32, ...}."""
        buf = C.create_string_buffer(1024)
        L.check(self._lib.b200_runner_plan_info(self.handle, buf, len(buf)))
        return {k: int(v) for k, v in (item.split("=") for item in buf.value.decode().split(";") if item)}

    def debug_read_workspace(self, offset: int, nbytes: int) -> np.ndarray:
        out = np.empty(nbytes, np.uint8)
        L.check(self._lib.b200_runner_debug_read_workspace(self.handle, offset, nbytes, out.ctypes.data))
        return out

    def upload(self) -> None:
        L.check(self._lib.b200_runner_upload(self.handle))

    def step_device(self, num_chunks: int, iters: int = 1):
        tot, fwd, dec = C.c_float(), C.c_float(), C.c_float()
        L.check(self._lib.b200_runner_step_device(self.handle, num_chunks, iters, C.byref(tot), C.byref(fwd),
                                                  C.byref(dec)))
        return tot.value, fwd.value, dec.value

    @staticmethod
    def step_device_runners(runners, num_chunks: int, iters: int = 1) -> float:
        """`iters` device-resident passes round-robin over several runners of one caller, all in flight at once
        (dorado keeps num_runners = 2 per device, api/runner_creation.cpp:91-123).  Returns device milliseconds."""
        arr = (C.c_void_p * len(runners))(*[r.handle if isinstance(r.handle, int) else r.handle.value for r in runners])
        tot = C.c_float()
        L.check(runners[0]._lib.b200_runners_step_device(arr, len(runners), num_chunks, iters, C.byref(tot)))
        return tot.value

    def out_len(self) -> int:
        return self._t_out

    def close(self):
        if self.handle:
            self._lib.b200_runner_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
