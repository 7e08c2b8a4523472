#!/usr/bin/env python
"""Ragged against padded batches through the FP16 Generator: what running each utterance at its own length saves.

Two workloads on a synthetic checkpoint at the default configuration:
  paragraph  8 sentences of one paragraph, 24 to 256 tokens (a caller batching the sentence slices it synthesizes one by one)
  config3    a config-3-like batch of 32 utterances, 32 to 128 tokens (seeded mix)
and three setups, alternated within every round so that they see the same machine state:
  padded   infer(): the Generator runs every utterance over F_max = max(y_lengths) frames
  ragged   infer(ragged=True): each utterance runs at its own length
  b1       the same utterances one by one at B=1
Durations are teacher-forced to the padded batch's (w_ceil_override), so every setup synthesizes the same frames.  Reported per setup
(median over rounds): Generator stage ms (bv2_stage_ms "generator", summed over the calls of b1), flow stage ms, whole-call ms (host
clock around infer_begin + infer_finish, ending in a device synchronise), kernel launches per call; per workload sum(L_b) against
B * F_max and the saving 1 - sum(L_b) / (B * F_max) that the Generator's work would show if its time were proportional to its frames.
The same run checks that every ragged utterance is bit-identical to a B=1 generator() call on the same z.

  python tools/ragged_batch.py [--rounds 10] [--warmup 2] [--out profiles/h100_ragged_batch.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.engine import Engine  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402

KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)


def workloads():
    r = np.random.default_rng(3)
    return {"paragraph": [24, 61, 98, 137, 170, 203, 229, 256],
            "config3": [int(v) for v in r.integers(32, 129, size=32)]}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"unavailable ({e})"
    return name, q


def _slice(inp, b, t):
    one = {k: (v[b:b + 1, ..., :t] if v.dim() >= 2 else v[b:b + 1]) for k, v in inp.items()}
    one["x_lengths"] = torch.tensor([t])
    return one


def _call(eng, inp, nw, nz, w_ceil, ragged):
    """one infer_begin + infer_finish; returns (o, z, y_lengths, generator ms, flow ms, whole-call ms, launches)"""
    B, T = inp["x"].shape
    torch.cuda.synchronize()
    l0, t0 = eng.launch_count, time.perf_counter()
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, KW["noise_scale_w"], KW["length_scale"], KW["sdp_ratio"], w_ceil_override=w_ceil)
    o, _, _, (z, _, _, _) = eng.infer_finish(B, T, F, nz, KW["noise_scale"], want_attn=False, ragged=ragged)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return o, z, ylen, eng.stage_ms("generator"), eng.stage_ms("flow"), ms, eng.launch_count - l0


def run_workload(eng, sd, cfg, lengths, rounds, warmup):
    B, T = len(lengths), max(lengths)
    inp = synth.synthetic_inputs(cfg, lengths, [i % 3 for i in range(B)], seed=B)
    nw, nz = synth.synthetic_noise(cfg, B, T, 16 * T + 64, seed=B)
    inp = {k: v.cuda() for k, v in inp.items()}
    nw, nz = nw.cuda(), nz.cuda()
    eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw,
                    KW["noise_scale_w"], KW["length_scale"], KW["sdp_ratio"])
    w_ceil = eng.debug_read("w_ceil", (B, 1, T))[:, 0].cuda()
    ylen = None
    setups = {"padded": [], "ragged": [], "b1": []}
    identical = True
    for r in range(warmup + rounds):
        rec = {}
        _, _, ylen, *m = _call(eng, inp, nw, nz, w_ceil, False)
        rec["padded"] = m
        o, z, _, *m = _call(eng, inp, nw, nz, w_ceil, True)
        rec["ragged"] = m
        if r == 0:  # every ragged utterance against a B=1 generator() call on the same z
            g = sd["emb_g.weight"].cuda()[inp["sid"]].unsqueeze(-1)
            for b, L in enumerate(ylen.tolist()):
                ref = eng.generator(z[b:b + 1, :, :L].contiguous(), g[b:b + 1])
                identical &= bool(torch.equal(o[b, :, :L * cfg.hop], ref[0])) and bool((o[b, :, L * cfg.hop:] == 0).all())
        acc = [0.0, 0.0, 0.0, 0]
        for b, t in enumerate(lengths):
            *_, gm, fm, ms, n = _call(eng, _slice(inp, b, t), nw[b:b + 1, :, :t], nz[b:b + 1], w_ceil[b:b + 1, :t], False)
            acc = [acc[0] + gm, acc[1] + fm, acc[2] + ms, acc[3] + n]
        rec["b1"] = acc
        if r >= warmup:
            for k, v in rec.items():
                setups[k].append(v)
    frames = [int(v) for v in ylen]
    out = {"B": B, "tokens": lengths, "frames": frames, "sum_L": sum(frames), "B_x_F_max": B * max(frames),
           "generator_saving_if_proportional_to_frames": round(1 - sum(frames) / (B * max(frames)), 3),
           "ragged_bit_identical_to_b1_generator": identical}
    for k, rows in setups.items():
        med = [statistics.median(row[i] for row in rows) for i in range(4)]
        out[k] = {"generator_ms": round(med[0], 3), "flow_ms": round(med[1], 3), "call_ms": round(med[2], 3), "launches": int(med[3]),
                  "flow_share_of_call": round(med[1] / med[2], 3)}
    out["measured_generator_saving_ragged_vs_padded"] = round(1 - out["ragged"]["generator_ms"] / out["padded"]["generator_ms"], 3)
    out["measured_call_saving_ragged_vs_padded"] = round(1 - out["ragged"]["call_ms"] / out["padded"]["call_ms"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ragged_batch.py measures on a CUDA device; none is available")
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    eng = Engine(cfg, sd, "cuda:0", "fp16")
    eng.set_profiling(True)
    name, q = card()
    res = {"gpu": name, "power_limit_max_sm_clock": q, "precision": "fp16", "rounds": a.rounds, "warmup": a.warmup,
           "note": "medians over rounds; setups alternate within each round; b1 sums the B=1 calls of the same utterances; "
                   "durations teacher-forced to the padded batch's; generator_saving_if_proportional_to_frames is computed, not measured",
           "workloads": {}}
    for wname, lengths in workloads().items():
        w = run_workload(eng, sd, cfg, lengths, a.rounds, a.warmup)
        res["workloads"][wname] = w
        print(f"{wname}: B={w['B']} sum(L)={w['sum_L']} B*F_max={w['B_x_F_max']} (computed saving "
              f"{w['generator_saving_if_proportional_to_frames']:.1%}), bit-identical to B=1: {w['ragged_bit_identical_to_b1_generator']}")
        for k in ("padded", "ragged", "b1"):
            s = w[k]
            print(f"  {k:7s} generator {s['generator_ms']:8.3f} ms  flow {s['flow_ms']:7.3f} ms  call {s['call_ms']:8.3f} ms  "
                  f"launches {s['launches']:5d}  flow share {s['flow_share_of_call']:.1%}")
        print(f"  measured: Generator {w['measured_generator_saving_ragged_vs_padded']:.1%}, whole call "
              f"{w['measured_call_saving_ragged_vs_padded']:.1%} less time ragged than padded")
    print(f"{name} ({q})")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
            f.write("\n")
    if not all(w["ragged_bit_identical_to_b1_generator"] for w in res["workloads"].values()):
        sys.exit("ragged outputs are not bit-identical to B=1 generator() calls")


if __name__ == "__main__":
    main()
