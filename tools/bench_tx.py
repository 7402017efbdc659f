#!/usr/bin/env python
"""Throughput of the transformer models on one GPU: sup@v5 (d_model 512, window (127, 128)) and the synthetic 1536-wide
fixture (d_model 1536, 24 heads, window (255, 256), feed-forward 6144; see tests/test_tx1536_cpu.py).

usage: python tools/bench_tx.py --model sup|tx1536 [--precision fp16|fp8_ffn|int8_qkv_fp8_ffn] [--batch 128] [--chunksize 12288]
       [--runners 2] [--steps 10] [--warmup 3]

--precision fp8_ffn runs fc1 + SwiGLU and fc2 on E4M3 operands behind an explicit norm1 pass (include/b200call.h); their
FLOP rates are then to be read against the data sheet's dense FP8 figure (1,979 TFLOP/s), also printed.  --precision
int8_qkv_fp8_ffn also runs the QKV projection on int8 operands (the data sheet's dense INT8 figure is 1,979 TOPS), behind a
quantise pass of the stack's input and an explicit norm2 pass that writes the int8 copy.

Device-resident steps as bench.py times them (step i on runner i % R, each runner on its own stream), then one profiled
forward + decode with an event after every launch.  Prints one JSON line: samples/s, the card (name, power limit, SM
clocks, read in the same run), the per-kernel times of the profiled pass, each GEMM's and the attention kernel's FLOP over
its time, and the whole forward's FLOP rate against the dense fp16 figure of the H100 SXM data sheet (989 TFLOP/s, a
700 W card; not a measured peak).  FLOP come from the config's shapes (flop_per_token_layer, flop_per_sample below).
There is no CPU fallback: without a GPU the tool fails.
"""
import argparse
import json
import pathlib
import subprocess
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

DATASHEET_FP16_TFLOPS = 989.0
DATASHEET_FP8_TFLOPS = 1979.0
CONFIGS = ROOT / "tests" / "data" / "model_configs"
MODELS = {"sup": CONFIGS / "dna_r10.4.1_e8.2_400bps_sup@v5.0.0", "tx1536": CONFIGS / "synthetic_tx1536@v0"}


def gemm_flop_per_token(cfg):
    """FLOP per token of every GEMM of one encoder layer, and of the upsample and CRF GEMMs (per encoder token)."""
    tx = cfg.tx
    d, ff = tx.d_model, tx.dim_feedforward
    return {"qkv_gemm": 2 * d * 3 * d, "out_proj_gemm": 2 * d * d, "fc1_swiglu_gemm": 2 * d * 2 * ff,
            "fc2_gemm": 2 * ff * d, "upsample_gemm": 2 * d * tx.upsample_scale * d,
            "crf_gemm": tx.upsample_scale * 2 * d * cfg.outsize}


def attention_flop_per_token(cfg):
    """Q K^T and P V over the keys a query sees (win_upper + win_lower + 1), all heads."""
    keys = cfg.tx.attn_window[0] + cfg.tx.attn_window[1] + 1
    return 2 * 2 * cfg.tx.d_model * keys


def flop_per_token_layer(cfg):
    g = gemm_flop_per_token(cfg)
    return sum(g[k] for k in ("qkv_gemm", "out_proj_gemm", "fc1_swiglu_gemm", "fc2_gemm")) + attention_flop_per_token(cfg)


def flop_per_sample(cfg):
    """Whole forward per input sample: convolutions, depth encoder layers, upsample, CRF linear."""
    samples_per_token = cfg.stride * cfg.tx.upsample_scale
    conv, step = 0.0, 1
    for c in cfg.convs:
        step *= c.stride
        conv += 2.0 * c.insize * c.size * c.winlen / step
    g = gemm_flop_per_token(cfg)
    return conv + (cfg.tx.depth * flop_per_token_layer(cfg) + g["upsample_gemm"] + g["crf_gemm"]) / samples_per_token


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
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp8_ffn", "int8_qkv_fp8_ffn"])
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--chunksize", type=int, default=12288)
    ap.add_argument("--runners", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if L.load_library().b200_device_count() < 1:
        raise SystemExit("bench_tx: no CUDA device; this tool only measures on the GPU")

    cfg = load_model_config(MODELS[args.model])
    N, R = args.batch, max(1, args.runners)
    caller = B200Caller(cfg, synthetic_weights(cfg, 42), num_runners=R, precision=args.precision)
    runner_bytes = caller.runner_bytes(N, args.chunksize)
    runners = [B200ModelRunner(caller, N, args.chunksize) for _ in range(R)]
    T = runners[0].chunk_size()
    tokens = T // (cfg.stride * cfg.tx.upsample_scale)
    rng = np.random.default_rng(1234)
    for r in runners:
        r.input_view()[:] = rng.standard_normal((N, T)).astype(np.float16)
        r.upload()
    B200ModelRunner.step_device_runners(runners, N, max(1, args.warmup) * R)
    ms = B200ModelRunner.step_device_runners(runners, N, args.steps)
    value = N * T * args.steps / (ms * 1e-3)
    gpu = card()

    prof = {}
    for name, t in runners[0].profile(N):
        k, tot = prof.get(name, (0, 0.0))
        prof[name] = (k + 1, tot + t)
    rows = N * tokens
    rates = {}
    for k, f in list(gemm_flop_per_token(cfg).items()) + [("tx_attention", attention_flop_per_token(cfg))]:
        if k in prof:
            launches, t = prof[k]
            rates[k] = {"ms_per_launch": t / launches, "tflops": f * rows * launches / (t * 1e-3) / 1e12}
    # bytes per element: rmsnorm_e4m3 reads the fp16 row, writes it in fp16 and E4M3; rmsnorm_i8 also reads its fp16 output
    # back and writes int8; quantize_i8 reads fp16 and writes int8
    for k, per_elem in (("rmsnorm_e4m3", 5), ("rmsnorm_i8", 7), ("quantize_i8", 3)):
        if k in prof:
            launches, t = prof[k]
            rates[k] = {"ms_per_launch": t / launches, "gb_per_s": rows * cfg.tx.d_model * per_elem * launches / (t * 1e-3) / 1e9}
    att_launches, att_ms = prof["tx_attention"]
    fps = flop_per_sample(cfg)
    out = {"model": args.model, "precision": args.precision, "d_model": cfg.tx.d_model, "nhead": cfg.tx.nhead, "attn_window": list(cfg.tx.attn_window),
           "batch": N, "chunk_samples": T, "tokens": tokens, "runners": R, "steps": args.steps,
           "runner_bytes": runner_bytes, "card": gpu,
           "samples_per_s": value, "ms_per_step": ms / args.steps,
           "flop_per_sample": fps, "flop_per_token_layer": flop_per_token_layer(cfg),
           "forward_tflops_per_s": fps * value / 1e12,
           "frac_of_datasheet_fp16": fps * value / 1e12 / DATASHEET_FP16_TFLOPS,
           "datasheet_tflops": {"fp16": DATASHEET_FP16_TFLOPS, "fp8": DATASHEET_FP8_TFLOPS},
           "kernels_ms": {k: {"launches": n, "ms": round(t, 4)} for k, (n, t) in prof.items()},
           "kernel_rates": rates,
           "attention_ms_per_layer": att_ms / att_launches,
           "attention_ns_per_query_key": att_ms / att_launches * 1e6 / (rows * cfg.tx.nhead *
                                                                        (cfg.tx.attn_window[0] + cfg.tx.attn_window[1] + 1))}
    print(json.dumps(out))
    for r in runners:
        r.close()
    caller.close()


if __name__ == "__main__":
    main()
