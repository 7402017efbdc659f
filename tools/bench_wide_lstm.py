#!/usr/bin/env python
"""Throughput of the lstm_size 128 / 256 models (lstm_rec_kernel) and 768 / 1024 models (lstm_grid_rec_kernel) on one GPU.

usage: python tools/bench_wide_lstm.py --model lstm128|lstm256|lstm768|lstm1024 [--batch 512] [--chunksize 10000]
       [--runners 2] [--steps 50] [--warmup 3]

Device-resident steps as bench.py times them (step i on runner i % R, each runner on its own stream), then one profiled
forward + decode with an event after every launch.  Prints one JSON line: samples/s, the per-kernel times of the profiled
pass, the x-projection GEMM and recurrence times per layer, the recurrence time per step, and the recurrence's W_hh FLOP
over its time against the dense fp16 peak of the H100 SXM data sheet (989 TFLOP/s, a 700 W card; not a measured peak).
FLOP per sample come from the config's shapes: per output step 16 C^2 per LSTM layer, conv3 and the CRF linear.
"""
import argparse
import json
import pathlib
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

PEAK_TFLOPS = 989.0


def main():
    import test_lstm128_256_cpu
    import test_wide_lstm_cpu
    from dorado_b200.config import load_model_config
    from dorado_b200.runner import B200Caller, B200ModelRunner
    from dorado_b200.weights import synthetic_weights
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", required=True, choices=["lstm128", "lstm256", "lstm768", "lstm1024"])
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--chunksize", type=int, default=10000)
    ap.add_argument("--runners", type=int, default=2)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    cluster = args.model in test_lstm128_256_cpu.MODELS   # lstm_rec_kernel, else lstm_grid_rec_kernel
    cfg = load_model_config((test_lstm128_256_cpu if cluster else test_wide_lstm_cpu).model_dir(args.model))
    C, c3 = cfg.lstm_size, cfg.convs[2]
    flop_per_sample = (cfg.lstm_layers * 16.0 * C * C + 2.0 * c3.winlen * c3.insize * C + 2.0 * C * cfg.outsize) / cfg.stride
    N, R = args.batch, max(1, args.runners)
    caller = B200Caller(cfg, synthetic_weights(cfg, 42), num_runners=R)
    runners = [B200ModelRunner(caller, N, args.chunksize) for _ in range(R)]
    T = runners[0].chunk_size()
    T_out = runners[0].out_len()
    rng = np.random.default_rng(1234)
    for r in runners:
        r.input_view()[:] = rng.standard_normal((N, T)).astype(np.float16)
        r.upload()
    B200ModelRunner.step_device_runners(runners, N, max(1, args.warmup) * R)
    ms = B200ModelRunner.step_device_runners(runners, N, args.steps)
    value = N * T * args.steps / (ms * 1e-3)

    prof = {}
    for name, t in runners[0].profile(N):
        k, tot = prof.get(name, (0, 0.0))
        prof[name] = (k + 1, tot + t)
    plan = runners[0].plan_info()
    mark, key = ("lstm_rec", "lstm_rec.ctas") if cluster else ("lstm_grid_rec", "lstm_grid.ctas")
    launches, rec_ms = prof[mark]
    layer_ms = rec_ms / cfg.lstm_layers
    rec_tflops = 8.0 * C * C * T_out * N * cfg.lstm_layers / (rec_ms * 1e-3) / 1e12
    out = {"model": args.model, "lstm_size": C, "batch": N, "chunk_samples": T, "runners": R, "steps": args.steps,
           "samples_per_s": value, "ms_per_step": ms / args.steps,
           "flop_per_sample": flop_per_sample, "forward_tflops_per_s": flop_per_sample * value / 1e12,
           "plan": plan,
           "kernels_ms": {k: {"launches": n, "ms": round(t, 4)} for k, (n, t) in prof.items()},
           "gx_gemm_ms_per_layer": prof["lstm_gx_gemm"][1] / cfg.lstm_layers,
           mark: {"ms_per_layer": layer_ms, "ms_per_launch": rec_ms / launches,
                  "us_per_step": rec_ms / launches / T_out * 1e3, "tflops": rec_tflops,
                  "frac_of_peak": rec_tflops / PEAK_TFLOPS,
                  "frac_of_sms_used": rec_tflops / PEAK_TFLOPS * 132 / min(132, plan[key])}}
    print(json.dumps(out))
    for r in runners:
        r.close()
    caller.close()


if __name__ == "__main__":
    main()
