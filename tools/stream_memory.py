#!/usr/bin/env python3
"""Memory and latency of bounded streams against unbounded ones and one-shot infer(), written as JSON.

Workloads (FP16 engine, B=1, bench.py's settings): config 2 (T=256, about 1023 frames) and a long synthetic utterance (T=1024, about
4000 frames).  The one-shot run of each goes first; it is the reference every stream must equal bit for bit.  Caps: unbounded, 64 and
256, each on a fresh engine, in rounds that alternate between them.  Per case:
  workspace_bytes        both arenas after the stream opened (fresh engine, so the stream's own request sized them)
  stream_bytes           the Generator storage the engine computes for the stream (bv2_stream_bytes)
  grows_after_reserve    workspace regrowths of a second engine during the stream after reserve_stream(1, T, F, cap)
  first_chunk_ms         host clock from the start of infer_begin to the completion of chunk 0 (32 frames, then doubling up to the cap)
  stream_ms, oneshot_ms  host clock to the completion of the last chunk / around infer_begin + infer_finish + synchronise
  launches               kernels per stream / per one-shot call
Medians over --reps rounds.  The card's name and power limit are read in the same run (nvidia-smi queries only).

    python tools/stream_memory.py --out profiles/h100_stream_memory.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.engine import Engine  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402

INFER_KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.625)  # bench.py's settings
WORKLOADS = {"config2": (256, 2048, 2), "long": (1024, 8192, 4)}  # T, noise frames, seed
CAPS = [None, 64, 256]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?"])[:2] if r.returncode == 0 else ("unknown", "unknown")
    return {"name": name, "power_limit": power}


def _args(inp, nw):
    return (inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw,
            INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])


def one_shot(eng, case):
    inp, nw, nz = case
    B, T = inp["x"].shape
    torch.cuda.synchronize()
    l0, t0 = eng.launch_count, time.perf_counter()
    _, F = eng.infer_begin(*_args(inp, nw))
    o, _, _, _ = eng.infer_finish(B, T, F, nz, INFER_KW["noise_scale"], None, want_attn=False)
    torch.cuda.synchronize()
    return o, F, (time.perf_counter() - t0) * 1e3, eng.launch_count - l0


def stream(eng, case, cap):
    """(o, ms to chunk 0, ms total, launches, workspace bytes right after the stream opened)"""
    inp, nw, nz = case
    B, T = inp["x"].shape
    hop = eng.cfg.hop
    torch.cuda.synchronize()
    l0, t0 = eng.launch_count, time.perf_counter()
    _, F = eng.infer_begin(*_args(inp, nw))
    o, _, _, _ = eng.infer_finish_stream(B, T, F, nz, INFER_KW["noise_scale"], None, want_attn=False, max_chunk_frames=cap)
    ws = eng.workspace_bytes
    Fg, done, step, first = o.shape[-1] // hop, 0, 32, None
    while done < Fg:
        target = min(done + step, Fg)
        eng.stream_advance(target)
        torch.cuda.current_stream().synchronize()
        if first is None:
            first = (time.perf_counter() - t0) * 1e3
        done, step = target, 2 * step if cap is None else min(2 * step, cap)
    return o, first, (time.perf_counter() - t0) * 1e3, eng.launch_count - l0, ws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_memory.py measures on the GPU; no CUDA device found")
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    result = {"card": card(), "precision": "fp16", "infer_kw": INFER_KW, "reps": args.reps, "workloads": {}}
    for wname, (T, n_noise, seed) in WORKLOADS.items():
        inp = synth.synthetic_inputs(cfg, [T], [0], seed=seed)
        nw, nz = synth.synthetic_noise(cfg, 1, T, n_noise, seed=seed)
        case = (inp, nw, nz)
        ref_eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
        one_shot(ref_eng, case)  # warm-up
        ref, F, _, launches_1 = one_shot(ref_eng, case)
        ref = ref.clone()
        one_ms = []
        rows = {str(c): {"first_chunk_ms": [], "stream_ms": [], "launches": None, "workspace_bytes": None, "bit_identical": True} for c in CAPS}
        for _ in range(args.reps):
            for cap in CAPS:  # rounds alternate between the caps
                one_ms.append(one_shot(ref_eng, case)[2])
                eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
                o, first, total, launches, ws = stream(eng, case, cap)
                r = rows[str(cap)]
                r["bit_identical"] &= bool(torch.equal(o, ref))
                r["first_chunk_ms"].append(first)
                r["stream_ms"].append(total)
                r["launches"], r["workspace_bytes"], r["stream_bytes"] = launches, ws, eng.stream_bytes(1, o.shape[-1] // cfg.hop, cap)
                del eng, o
                eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
                eng.reserve_stream(1, T, F, cap)
                g0 = eng.workspace_grows
                o, _, _, _, _ = stream(eng, case, cap)
                r["grows_after_reserve"] = eng.workspace_grows - g0
                r["bit_identical"] &= bool(torch.equal(o, ref))
                del eng, o
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
        for r in rows.values():
            for k in ("first_chunk_ms", "stream_ms"):
                r[k] = {"median": statistics.median(r[k]), "min": min(r[k]), "max": max(r[k])}
        result["workloads"][wname] = {"T": T, "frames": F, "oneshot_ms": {"median": statistics.median(one_ms), "min": min(one_ms), "max": max(one_ms)},
                                      "oneshot_launches": launches_1, "cases": rows}
        print(json.dumps({wname: result["workloads"][wname]}), flush=True)
        del ref_eng
    text = json.dumps(result, indent=2)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
