#!/usr/bin/env python
"""Throughput of a conv_lstm_v3 modified-base model on one GPU.

usage: python tools/bench_modbase.py --model DIR|mb384|mb192 [--batch 1024] [--runners 2] [--steps 50] [--warmup 3]

Each of R runners (R threads, each runner on its own stream) calls call_chunks on full batches, steps batches in all,
after `warmup` batches per runner; the rate is end to end (H2D of signal and k-mers, forward, D2H of the probabilities)
over the wall time of the timed batches.  Then one profiled forward on one runner with an event after every launch.
Prints one JSON line: chunks/s, samples/s, the per-kernel times of the profiled forward, and FLOP computed from the
config's shapes -- per kernel and per chunk -- over the measured times.  The card's name, power limit and SM clock limit
are read in the same run.
"""
import argparse
import json
import pathlib
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def kernel_flop(cfg):
    """Multiply-adds x 2 per chunk of every launch of the forward, by the names the profile uses."""
    m = cfg.modules
    s1, s2, s3 = m.signal_convs
    q1, q2 = m.sequence_convs
    mc = m.merge_conv
    L, Ts, T, te = cfg.chunk_size, cfg.chunked_sequence_input_TC()[0], cfg.lstm_steps(), cfg.encoder_steps()
    C = cfg.lstm_size
    head = 2.0 * T * C * cfg.num_out + (2.0 * T * cfg.upsample_scale * cfg.num_out * cfg.num_out if m.upsample else 0.0)
    return {
        "sig_conv12": 2.0 * L * (s1.size * s1.winlen + s2.size * s2.insize * s2.winlen),
        "sig_conv3_gemm": 2.0 * te * s3.size * s3.insize * s3.winlen,
        "seq_conv1": 2.0 * Ts * q1.size * q1.insize * q1.winlen,
        "seq_conv2_gemm": 2.0 * te * q2.size * q2.insize * q2.winlen,
        "merge_conv_gemm": 2.0 * T * mc.size * mc.insize * mc.winlen,
        "lstm_gx_gemm": 2.0 * T * 4 * C * C,         # per layer
        "lstm_rec": 2.0 * T * 4 * C * C,             # per layer (W_hh h)
        "lstm_grid_rec": 2.0 * T * 4 * C * C,
        "head": head,
    }


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    from test_modbase_cpu import MODBASE, modbase_dir, modbase_inputs
    from dorado_b200.config import load_modbase_config
    from dorado_b200.modbase import B200ModBaseCaller, B200ModBaseRunner
    from dorado_b200.weights import synthetic_modbase_weights
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", required=True, help="model directory, or mb384 / mb192 for the test fixtures")
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--runners", type=int, default=2)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    cfg = load_modbase_config(modbase_dir(args.model) if args.model in MODBASE else args.model)
    N, R = args.batch, max(1, args.runners)
    caller = B200ModBaseCaller(cfg, synthetic_modbase_weights(cfg, 42))
    runners = [B200ModBaseRunner(caller, N) for _ in range(R)]
    sig, seq = modbase_inputs(cfg, N, 1234)
    for r in runners:
        for i in range(N):
            r.accept_chunk(i, sig[i], seq[i])

    def work(r, n):
        for _ in range(n):
            r.call_chunks(N)

    def run_all(counts):
        ts = [threading.Thread(target=work, args=(r, k)) for r, k in zip(runners, counts)]
        t0 = time.perf_counter()
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        return time.perf_counter() - t0

    run_all([max(1, args.warmup)] * R)
    counts = [args.steps // R + (1 if i < args.steps % R else 0) for i in range(R)]
    wall = run_all(counts)
    chunks_s = N * args.steps / wall

    prof = {}
    for name, t in runners[0].profile():
        k, tot = prof.get(name, (0, 0.0))
        prof[name] = (k + 1, tot + t)
    fl = kernel_flop(cfg)
    kernels = {}
    for name, (k, ms) in prof.items():
        if name == "begin":
            continue
        f = fl.get(name, 0.0) * k * N
        kernels[name] = {"launches": k, "ms": round(ms, 4), "tflops": round(f / (ms * 1e-3) / 1e12, 2) if ms > 0 else None}
    per_chunk = sum(v for k, v in fl.items() if k not in ("lstm_gx_gemm", "lstm_rec", "lstm_grid_rec")) + 4 * fl["lstm_rec"]
    fwd_ms = sum(ms for name, (k, ms) in prof.items() if name != "begin")
    print(json.dumps({
        "metric": "modbase_chunks_per_s", "model": cfg.name, "card": card(), "batch": N, "runners": R, "steps": args.steps,
        "chunks_per_s": round(chunks_s, 1), "samples_per_s": round(chunks_s * cfg.chunk_size, 1),
        "gflop_per_chunk": round(per_chunk / 1e9, 4), "end_to_end_tflops": round(per_chunk * chunks_s / 1e12, 2),
        "profiled_forward_ms": round(fwd_ms, 4), "profiled_forward_tflops": round(per_chunk * N / (fwd_ms * 1e-3) / 1e12, 2),
        "kernels": kernels,
    }))


if __name__ == "__main__":
    main()
