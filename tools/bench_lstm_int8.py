#!/usr/bin/env python
"""Throughput of the LSTM models that have the int8_lstm precision, in either precision, on one GPU: hac@v5 (lstm_size 384)
and the synthetic 256-wide fixture.

usage: python tools/bench_lstm_int8.py --model hac|lstm256 [--precision fp16|int8_lstm] [--batch 512] [--chunksize 9996]
       [--runners 2] [--steps 20] [--warmup 3]

Device-resident steps as bench.py times them (b200_runners_step_device: step i on runner i % R, each runner on its own
stream), then one profiled forward + decode of one runner with an event after every launch.  Prints one JSON line:
samples/s, the card (name, power limit, SM clocks, read in the same run), the per-kernel times of the profiled pass, the
time per recurrence step, and the device bytes of one runner.  There is no CPU fallback: without a GPU the tool fails.
"""
import argparse
import json
import pathlib
import subprocess
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

CONFIGS = ROOT / "tests" / "data" / "model_configs"
MODELS = {"hac": CONFIGS / "dna_r10.4.1_e8.2_400bps_hac@v5.0.0", "lstm256": CONFIGS / "synthetic_lstm256@v0"}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         check=True, capture_output=True, text=True).stdout.splitlines()[0]
    name, power, sm, sm_max = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def main():
    from dorado_b200 import lib as L
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", required=True, choices=list(MODELS))
    ap.add_argument("--precision", default="fp16", choices=["fp16", "int8_lstm"])
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--chunksize", type=int, default=9996)
    ap.add_argument("--runners", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if L.load_library().b200_device_count() < 1:
        raise SystemExit("bench_lstm_int8: no CUDA device; this tool only measures on the GPU")

    cfg = load_model_config(MODELS[args.model])
    N, R = args.batch, max(1, args.runners)
    caller = B200Caller(cfg, synthetic_weights(cfg, 42), num_runners=R, precision=args.precision)
    runner_bytes = caller.runner_bytes(N, args.chunksize)
    runners = [B200ModelRunner(caller, N, args.chunksize) for _ in range(R)]
    T = runners[0].chunk_size()
    rng = np.random.default_rng(1234)
    for r in runners:
        r.input_view()[:] = rng.standard_normal((N, T)).astype(np.float16)
        r.upload()
    B200ModelRunner.step_device_runners(runners, N, max(1, args.warmup) * R)
    ms = B200ModelRunner.step_device_runners(runners, N, args.steps)
    gpu = card()

    prof = {}
    for name, t in runners[0].profile(N):
        k, tot = prof.get(name, (0, 0.0))
        prof[name] = (k + 1, tot + t)
    rec = prof.get("lstm_rec_i8") or prof["lstm_rec"]
    out = {"model": args.model, "precision": args.precision, "lstm_size": cfg.lstm_size, "batch": N, "chunk_samples": T,
           "runners": R, "steps": args.steps, "runner_bytes": runner_bytes, "card": gpu,
           "samples_per_s": N * T * args.steps / (ms * 1e-3), "ms_per_step": ms / args.steps,
           "plan": runners[0].plan_info(),
           "kernels_ms": {k: {"launches": n, "ms": round(t, 4)} for k, (n, t) in prof.items()},
           "recurrence_us_per_step": rec[1] / rec[0] * 1e3 / (T // cfg.stride)}
    print(json.dumps(out))
    for r in runners:
        r.close()
    caller.close()


if __name__ == "__main__":
    main()
