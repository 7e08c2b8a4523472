#!/usr/bin/env python
"""Per-layer times of the FP16 Generator: bv2_generator at config-5 size under torch.profiler (CUDA activities), every k_g2_conv launch
attributed to its layer by its order on its stream, printed as us and TFLOP/s per (level, resblock kernel size, conv).

Launch order (engine.cu g2_windows): the main stream runs conv_pre, then per level the ConvTranspose and resblock 0; side stream j runs
resblock j of every level (side streams are told apart by creation order, which is the order of their stream ids).  Each resblock is
nd x (c1, c2) convs in dilation order.  Numbers taken under the profiler are per-kernel times, not a bench value.

  python tools/gen_layer_times.py [--frames 1024] [--runs 5] [--out profiles/h100_generator_layers.json --label after]

--out merges the result into the file under --label, so runs of two builds can sit side by side."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.engine import Engine  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402


def layer_table(cfg, F):
    """[(stream, name, flops)] in launch order per stream: stream 0 = main, j = side stream of resblock j."""
    nk, nd = len(cfg.resblock_kernel_sizes), len(cfg.resblock_dilation_sizes[0])
    C0 = cfg.upsample_initial_channel
    rows = {j: [] for j in range(nk)}
    rows[0].append(("conv_pre", 2.0 * F * C0 * cfg.inter_channels * 7))
    T, C = F, C0
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        rows[0].append((f"L{i} ups C{C}->{C // 2} k{k}", 2.0 * T * C * (C // 2) * k))  # T input frames x Cin x Cout x k
        T, C = T * u, C // 2
        for j, (ks, ds) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
            for d in range(nd):
                for c in (1, 2):
                    rows[j].append((f"L{i} C{C} rb k{ks} d{ds[d]} c{c}", 2.0 * T * C * C * ks))
    return rows


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5, help="profiled Generator runs; each layer reports the median")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--label", default="run")
    a = ap.parse_args()

    cfg = ModelConfig()
    eng = Engine(cfg, synth.synthetic_state_dict(cfg, 0), "cuda:0", "fp16")
    z, g = synth.synthetic_generator_inputs(cfg, 1, a.frames)
    z, g = z.cuda(), g.cuda()
    for _ in range(a.warmup):
        eng.generator(z, g)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.runs):
            eng.generator(z, g)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kern = [e for e in trace["traceEvents"] if e.get("cat") == "kernel" and "k_g2_conv" in e.get("name", "")]
    by_stream = {}
    for e in sorted(kern, key=lambda e: e["ts"]):
        by_stream.setdefault(e["args"]["stream"], []).append(e)

    table = layer_table(cfg, a.frames)
    per_run = {j: len(r) for j, r in table.items()}
    main_ids = [s for s, ev in by_stream.items() if len(ev) == per_run[0] * a.runs]
    side_ids = sorted(s for s in by_stream if s not in main_ids)
    if len(main_ids) != 1 or len(side_ids) != len(table) - 1 or any(len(by_stream[s]) != per_run[j + 1] * a.runs for j, s in enumerate(side_ids)):
        sys.exit(f"unexpected k_g2_conv launch pattern: {{stream: launches}} = { {s: len(v) for s, v in by_stream.items()} }")
    streams = {0: main_ids[0], **{j + 1: s for j, s in enumerate(side_ids)}}

    layers = []
    for j, rows in table.items():
        ev = by_stream[streams[j]]
        n = len(rows)
        for idx, (name, flops) in enumerate(rows):
            us = statistics.median(ev[r * n + idx]["dur"] for r in range(a.runs))
            layers.append({"layer": name, "stream": j, "us": round(us, 2), "tflops": round(flops / (us * 1e-6) / 1e12, 1)})
    total_us = sum(l["us"] for l in layers)
    total_flops = sum(f for rows in table.values() for _, f in rows)
    name, q = card()
    res = {"gpu": name, "power_limit_max_sm_clock": q, "frames": a.frames, "runs": a.runs, "k_g2_conv_launches": len(layers),
           "sum_us": round(total_us, 1), "sum_tflops": round(total_flops / (total_us * 1e-6) / 1e12, 1),
           "note": "per-kernel durations under torch.profiler (median over runs); side-stream kernels overlap main-stream ones, so sum_us is "
                   "kernel time, not wall time",
           "layers": layers}
    for l in layers:
        print(f"{l['layer']:34s} stream {l['stream']}  {l['us']:9.1f} us  {l['tflops']:6.1f} TFLOP/s")
    print(f"{name} ({q}): {len(layers)} k_g2_conv launches, {total_us:.0f} us kernel time, {res['sum_tflops']} TFLOP/s")
    if a.out:
        data = {}
        if os.path.exists(a.out):
            with open(a.out) as f:
                data = json.load(f)
        data[a.label] = res
        with open(a.out, "w") as f:
            json.dump(data, f, indent=1)
            f.write("\n")


if __name__ == "__main__":
    main()
