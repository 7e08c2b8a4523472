#!/usr/bin/env python3
"""Latency of streaming synthesis against one-shot infer() on the bench workloads, written as JSON.

For the config-2 utterance (B=1, T=256 ZH, length_scale 0.625) and config 3 (B=32, T=128 mixed ZH/JA/EN), per precision:
  first_chunk_ms   host clock from the start of infer_begin to the completion of chunk 0 (first_chunk_frames=32, then doubling)
  stream_ms        host clock from the start of infer_begin to the completion of the last chunk
  oneshot_ms       host clock around infer_begin + infer_finish + device synchronise
  launches         kernels per stream / per one-shot call
Medians over --reps runs after --warmup runs.  Also the Generator launches of a config-2 stream per chunk schedule.  The card's name and
power limit are read in the same run (nvidia-smi queries only).

    python tools/stream_latency.py --out profiles/h100_stream_latency.json
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
WORKLOADS = {"config2": ([256], [0], 2), "config3": ([128] * 32, [i % 3 for i in range(32)], 3)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?"])[:2] if r.returncode == 0 else ("unknown", "unknown")
    return {"name": name, "power_limit": power}


def geometric(first):
    def f(Fg):
        out, x, step = [], 0, first
        while x < Fg:
            x = min(x + step, Fg)
            out.append(x)
            step *= 2
        return out
    return f


def run(eng, case, frontiers=None):
    """one call; frontiers None: one-shot.  Returns (ms to chunk 0 or None, ms total, launches, chunks)"""
    inp, nw, nz = case
    B, T = inp["x"].shape
    args = (inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw,
            INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
    torch.cuda.synchronize()
    l0 = eng.launch_count
    t0 = time.perf_counter()
    _, F = eng.infer_begin(*args)
    if frontiers is None:
        eng.infer_finish(B, T, F, nz, INFER_KW["noise_scale"], want_attn=False)
        torch.cuda.synchronize()
        return None, (time.perf_counter() - t0) * 1e3, eng.launch_count - l0, 1
    eng.infer_finish_stream(B, T, F, nz, INFER_KW["noise_scale"], want_attn=False)
    first = None
    fr = frontiers(F)
    for f in fr:
        eng.stream_advance(f)
        torch.cuda.current_stream().synchronize()
        if first is None:
            first = (time.perf_counter() - t0) * 1e3
    return first, (time.perf_counter() - t0) * 1e3, eng.launch_count - l0, len(fr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--precisions", default="fp16,fp16g")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stream_latency: no CUDA device (this script measures on the GPU only)")
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    cases = {}
    for name, (lens, langs, seed) in WORKLOADS.items():
        inp = synth.synthetic_inputs(cfg, lens, langs, seed=seed)
        nw, nz = synth.synthetic_noise(cfg, len(lens), max(lens), 4096, seed=seed)
        cases[name] = ({k: v.cuda() for k, v in inp.items()}, nw.cuda(), nz.cuda())
    out = {"card": card(), "first_chunk_frames": 32, "schedule": "32 frames, then doubling", "reps": a.reps, "results": {}}
    for prec in a.precisions.split(","):
        eng = Engine(cfg, sd, device="cuda:0", precision=prec)
        res = {}
        for name, case in cases.items():
            for _ in range(a.warmup):
                run(eng, case)
                run(eng, case, geometric(32))
            one, st = [], []
            for _ in range(a.reps):  # alternate the two so that both see the same host and device conditions
                one.append(run(eng, case))
                st.append(run(eng, case, geometric(32)))
            _, F = eng.infer_begin(*(case[0][k] for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")),
                                   case[1], INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
            res[name] = {"frames": F, "batch": case[0]["x"].shape[0],
                         "first_chunk_ms": statistics.median(r[0] for r in st), "stream_ms": statistics.median(r[1] for r in st),
                         "oneshot_ms": statistics.median(r[1] for r in one), "launches_stream": st[0][2], "launches_oneshot": one[0][2],
                         "chunks": st[0][3]}
            print(prec, name, json.dumps(res[name]), flush=True)
        sched = {"geometric_32": geometric(32), "chunks_of_7": lambda F: list(range(7, F, 7)) + [F], "one_chunk": lambda F: [F],
                 "every_frame": lambda F: list(range(1, F + 1))}
        res["config2_launches_per_schedule"] = {k: {"chunks": r[3], "launches": r[2]} for k, f in sched.items()
                                                for r in [run(eng, cases["config2"], f)]}
        out["results"][prec] = res
        del eng
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
