#!/usr/bin/env python
"""Per-layer times of the FP16 transformer flow: Engine.flow_reverse at config-2 size under torch.profiler (CUDA activities), every
kernel of the flow attributed to its role by its launch order, printed as us and TFLOP/s per launch and summed per role.

Launch order (engine.cu run_flow / run_encoder), one stream: per coupling `pre`, then n_layers_trans_flow layers, then `post`; per layer
qkv, k_flow_attn, conv_o + residual + LayerNorm, FFN conv_1, FFN conv_2, k_layernorm_c4, with k_add_bvec_mask in front of layer
cond_layer_idx.  Numbers taken under the profiler are per-kernel times, not a bench value; `flow_ms` is the wall time of one
flow_reverse call between CUDA events, taken without the profiler.

  python tools/flow_layer_times.py [--frames 1023] [--batch 1] [--runs 5] [--out profiles/h100_flow_layers.json --label after]

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

# role -> kernel the role launches (substring of the profiler's kernel name)
KERNEL = {"pre": "k_tc_conv1d", "qkv": "k_tc_conv1d", "attn": "k_flow_attn", "conv_o+LN": "k_tc_conv1d", "ffn1": "k_tc_conv1d",
          "ffn2": "k_tc_conv1d", "ln2": "k_layernorm_c4", "bvec": "k_add_bvec_mask", "post": "k_tc_conv1d"}
CONV_ROLES = ("pre", "qkv", "conv_o+LN", "ffn1", "ffn2", "post")


def launch_table(cfg, B, F):
    """[(coupling, layer, role, flops)] in launch order for one flow_reverse call with y_lengths = F."""
    H, I, Fc, K = cfg.hidden_channels, cfg.inter_channels, cfg.filter_channels, cfg.flow_kernel_size
    conv = lambda cin, cout, k: 2.0 * B * F * cin * cout * k  # noqa: E731
    rows = []
    for c in range(cfg.n_flows):
        rows.append((c, None, "pre", conv(I // 2, H, 1)))
        for i in range(cfg.n_layers_trans_flow):
            if i == cfg.cond_layer_idx:
                rows.append((c, i, "bvec", 0.0))
            rows += [(c, i, "qkv", conv(H, 3 * H, 1)),
                     (c, i, "attn", 4.0 * B * F * F * H),  # Q.K^T and P.V over all keys, every head
                     (c, i, "conv_o+LN", conv(H, H, 1)),
                     (c, i, "ffn1", conv(H, Fc, K)),
                     (c, i, "ffn2", conv(Fc, H, K)),
                     (c, i, "ln2", 0.0)]
        rows.append((c, None, "post", conv(H, I // 2, 1)))
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
    ap.add_argument("--frames", type=int, default=1023)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--runs", type=int, default=5, help="profiled flow_reverse calls; each launch reports the median")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--label", default="run")
    a = ap.parse_args()

    cfg = ModelConfig()
    if not cfg.use_transformer_flow:
        sys.exit("the layer table is written for the transformer flow")
    B, F = a.batch, a.frames
    eng = Engine(cfg, synth.synthetic_state_dict(cfg, 0), "cuda:0", "fp16")
    gen = torch.Generator().manual_seed(3)
    z_p = torch.randn(B, cfg.inter_channels, F, generator=gen).cuda()
    y_lengths = torch.full((B,), F, dtype=torch.int64).cuda()
    sid = torch.zeros(B, dtype=torch.int64).cuda()
    for _ in range(a.warmup):
        eng.flow_reverse(z_p, y_lengths, sid)
    torch.cuda.synchronize()
    walls = []
    for _ in range(max(a.runs, 5)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.flow_reverse(z_p, y_lengths, sid)
        e1.record()
        torch.cuda.synchronize()
        walls.append(e0.elapsed_time(e1))
    flow_ms = statistics.median(walls)

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.runs):
            eng.flow_reverse(z_p, y_lengths, sid)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    names = set(KERNEL.values())
    kern = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel" and any(k in e.get("name", "") for k in names)),
                  key=lambda e: e["ts"])
    table = launch_table(cfg, B, F)
    n = len(table)
    got = [next(k for k in names if k in e["name"]) for e in kern]
    want = [KERNEL[r[2]] for r in table] * a.runs
    if got != want:
        counts = {k: got.count(k) for k in sorted(names)}
        expect = {k: want.count(k) for k in sorted(names)}
        sys.exit(f"unexpected flow launch pattern: launches {counts}, expected {expect} ({a.runs} runs of {n})")

    def chain(k):
        """what launch k adds to the stream's chain: its end minus the previous flow kernel's end (its own duration for the first).  With
        programmatic dependent launch a kernel starts before its predecessor ends and waits for it, so `dur` double counts that overlap;
        the chain times partition the flow's kernel span."""
        e = kern[k]
        if k % n == 0:
            return e["dur"]
        p = kern[k - 1]
        return (e["ts"] + e["dur"]) - (p["ts"] + p["dur"])

    launches = []
    for idx, (c, i, role, flops) in enumerate(table):
        us = statistics.median(kern[r * n + idx]["dur"] for r in range(a.runs))
        ch = statistics.median(chain(r * n + idx) for r in range(a.runs))
        ent = {"coupling": c, "layer": i, "role": role, "us": round(us, 2), "chain_us": round(ch, 2)}
        if flops:
            ent["tflops"] = round(flops / (us * 1e-6) / 1e12, 2)
        launches.append(ent)
    roles = {}
    for role in KERNEL:
        ents = [l for l in launches if l["role"] == role]
        us = sum(l["us"] for l in ents)
        flops = sum(r[3] for r in table if r[2] == role)
        roles[role] = {"launches": len(ents), "sum_us": round(us, 1), "us_per_launch": round(us / len(ents), 2),
                       "chain_us": round(sum(l["chain_us"] for l in ents), 1)}
        if flops:
            roles[role]["tflops"] = round(flops / (us * 1e-6) / 1e12, 2)
    total_us = sum(l["us"] for l in launches)
    chain_us = sum(l["chain_us"] for l in launches)
    conv_chain_us = sum(roles[r]["chain_us"] for r in CONV_ROLES)
    name, q = card()
    res = {"gpu": name, "power_limit_max_sm_clock": q, "batch": B, "frames": F, "runs": a.runs, "launches_per_call": n,
           "flow_ms": round(flow_ms, 3), "sum_kernel_us": round(total_us, 1),
           "chain_us": round(chain_us, 1), "conv_chain_us": round(conv_chain_us, 1), "conv_share_of_chain": round(conv_chain_us / chain_us, 3),
           "note": "us: per-kernel durations under torch.profiler (median over runs), including the time a kernel launched early by "
                   "programmatic dependent launch waits for its predecessor; chain_us: end of the launch minus end of the previous flow "
                   "kernel, which partitions the flow's kernel span; flow_ms = wall time of one flow_reverse call (CUDA events, median, "
                   "profiler off), which also holds the speaker projection and the layout copies around the flow",
           "roles": roles, "launches": launches}
    for l in launches:
        lay = "" if l["layer"] is None else f"L{l['layer']}"
        tf = f"{l['tflops']:7.2f} TFLOP/s" if "tflops" in l else ""
        print(f"c{l['coupling']} {lay:3s} {l['role']:10s} {l['us']:8.1f} us  chain {l['chain_us']:8.1f} us  {tf}")
    print("per role:")
    for role, r in roles.items():
        tf = f"{r['tflops']:7.2f} TFLOP/s" if "tflops" in r else ""
        print(f"  {role:10s} {r['launches']:3d} launches {r['sum_us']:9.1f} us ({r['us_per_launch']:7.2f} us each)  chain {r['chain_us']:9.1f} us  {tf}")
    print(f"{name} ({q}): B={B} F={F}: flow_reverse {flow_ms:.3f} ms wall, {chain_us:.0f} us kernel chain in {n} launches, "
          f"convolutions {conv_chain_us:.0f} us of it ({res['conv_share_of_chain']:.2f})")
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
