"""Modified-base calling (conv_lstm_v3 models) on top of the C ABI.

``B200ModBaseCaller`` is one model on one GPU (the model data of the reference's ``ModBaseCaller``,
dorado/modbase/ModBaseCaller.cpp); ``B200ModBaseRunner`` is one batch in flight with the calls of
``ModBaseRunner`` (dorado/modbase/ModBaseRunner.cpp:36-95) for a single model: ``accept_chunk(idx, signal, kmers)``
and ``call_chunks(n)``, which returns the fp16 probabilities ``[n, out_len * num_out]`` that the reference's CUDA path
returns (ModBaseCaller.cpp:125, 193).  Several runners may share one caller.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import lib as L
from .config import ModBaseModelConfig


class B200ModBaseCaller:
    def __init__(self, cfg: ModBaseModelConfig, weights: dict, device: int = 0):
        self.cfg = cfg
        self.device = device
        lib = L.load_library()
        desc = L.modbase_desc_from_config(cfg)
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
        self.handle = C.c_void_p()
        L.check(lib.b200_modbase_engine_create(C.byref(desc), arr, len(weights), device, C.byref(self.handle)))

    def close(self) -> None:
        if self.handle:
            L.check(L.load_library().b200_modbase_engine_destroy(self.handle))
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200ModBaseRunner:
    def __init__(self, caller: B200ModBaseCaller, batch_size: int):
        self.caller = caller
        lib = L.load_library()
        self.handle = C.c_void_p()
        L.check(lib.b200_modbase_runner_create(caller.handle, batch_size, C.byref(self.handle)))
        self.batch_size = batch_size
        self.sig_len = lib.b200_modbase_runner_sig_len(self.handle)
        self.seq_len = lib.b200_modbase_runner_seq_len(self.handle)
        self.out_len = lib.b200_modbase_runner_out_len(self.handle)
        self.num_out = lib.b200_modbase_runner_num_out(self.handle)

    def accept_chunk(self, idx: int, signal: np.ndarray, kmers: np.ndarray) -> None:
        """signal: fp16 [sig_len]; kmers: int8 [seq_len, kmer_len * 4] (the one-hot k-mer encoding)."""
        s = np.ascontiguousarray(signal, np.float16)
        k = np.ascontiguousarray(kmers, np.int8)
        L.check(L.load_library().b200_modbase_runner_accept_chunk(self.handle, idx, s.ctypes.data, s.size, k.ctypes.data,
                                                                   k.size))

    def call_chunks(self, num_chunks: int) -> np.ndarray:
        """fp16 [num_chunks, out_len * num_out]: softmax over the num_out classes at every output step."""
        p = C.POINTER(C.c_uint16)()
        L.check(L.load_library().b200_modbase_runner_call_chunks(self.handle, num_chunks, C.byref(p)))
        n = num_chunks * self.out_len * self.num_out
        return np.ctypeslib.as_array(p, (n,)).view(np.float16).reshape(num_chunks, -1).copy()

    def profile(self) -> list:
        """One forward with device milliseconds per kernel launch, in launch order: [(name, ms), ...]."""
        buf = C.create_string_buffer(8192)
        L.check(L.load_library().b200_modbase_runner_profile(self.handle, buf, len(buf)))
        return [(kv.split("=")[0], float(kv.split("=")[1])) for kv in buf.value.decode().split(";") if kv]

    def debug_read_workspace(self, offset: int, nbytes: int) -> np.ndarray:
        out = np.empty(nbytes, np.uint8)
        L.check(L.load_library().b200_modbase_runner_debug_read_workspace(self.handle, offset, nbytes, out.ctypes.data))
        return out

    def read_sequence_buffer(self) -> np.ndarray:
        """The LSTM sequence buffer, fp16 [T][batch_size][lstm_size], at the start of the workspace."""
        T, N, Cc = self.caller.cfg.lstm_steps(), self.batch_size, self.caller.cfg.lstm_size
        return self.debug_read_workspace(0, T * N * Cc * 2).view(np.float16).reshape(T, N, Cc).copy()

    def close(self) -> None:
        if self.handle:
            L.check(L.load_library().b200_modbase_runner_destroy(self.handle))
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
