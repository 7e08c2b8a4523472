#!/usr/bin/env python
"""Ragged against padded streams through the FP16 Generator: what running each utterance of a streamed batch at its own length saves.

The two workloads of tools/ragged_batch.py on a synthetic checkpoint at the default configuration (paragraph: 8 sentences of 24 to 256
tokens; config3: a seeded mix of 32 utterances of 32 to 128 tokens), durations teacher-forced to the padded batch's (w_ceil_override) so
that every setup synthesizes the same frames.  Four setups, alternated within every round so that they see the same machine state:
  padded / ragged          infer_finish_stream(..., ragged=False / True), unbounded
  padded_256 / ragged_256  the same with max_chunk_frames = 256 (bounded streams)
each advanced with infer_stream()'s schedule (32 frames, then doubling; up to 256 with the cap).  Reported per setup (median over rounds):
time to the first chunk and whole-stream time (host clock from infer_begin to the chunk's completion event), Generator ms (bv2_stage_ms
"generator" of every advance, summed), kernel launches per stream; per workload sum(L_b) against B * F_max and the saving
1 - sum(L_b) / (B * F_max) that the Generator's work would show if its time were proportional to its frames (computed, not measured).
The same run checks that every ragged stream is bit-identical to infer_finish(..., ragged=True).

  python tools/ragged_stream.py [--rounds 10] [--warmup 2] [--out profiles/h100_ragged_stream.json]"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.engine import Engine  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402
from ragged_batch import KW, card, workloads  # noqa: E402

FIRST, CAP = 32, 256
SETUPS = {"padded": (False, None), "ragged": (True, None), "padded_256": (False, CAP), "ragged_256": (True, CAP)}


def _begin(eng, inp, nw, w_ceil):
    return eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"],
                           nw, KW["noise_scale_w"], KW["length_scale"], KW["sdp_ratio"], w_ceil_override=w_ceil)


def _stream(eng, inp, nw, nz, w_ceil, ragged, cap):
    """one stream: (o, first-chunk ms, whole-stream ms, Generator ms, launches, chunks)"""
    B, T = inp["x"].shape
    st = torch.cuda.current_stream()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, F = _begin(eng, inp, nw, w_ceil)
    o, _, _, _ = eng.infer_finish_stream(B, T, F, nz, KW["noise_scale"], want_attn=False, max_chunk_frames=cap, ragged=ragged)
    l0, gen, first, done, step, n = eng.launch_count, 0.0, None, 0, FIRST, 0
    while done < F:
        target = min(done + step, F)
        eng.stream_advance(target)
        ev = torch.cuda.Event()
        ev.record(st)
        ev.synchronize()
        if first is None:
            first = (time.perf_counter() - t0) * 1e3
        gen += eng.stage_ms("generator")
        done, step, n = target, 2 * step if cap is None else min(2 * step, cap), n + 1
    whole = (time.perf_counter() - t0) * 1e3
    return o, first, whole, gen, eng.launch_count - l0, n


def run_workload(eng, cfg, lengths, rounds, warmup):
    B, T = len(lengths), max(lengths)
    inp = synth.synthetic_inputs(cfg, lengths, [i % 3 for i in range(B)], seed=B)
    nw, nz = synth.synthetic_noise(cfg, B, T, 16 * T + 64, seed=B)
    inp = {k: v.cuda() for k, v in inp.items()}
    nw, nz = nw.cuda(), nz.cuda()
    _begin(eng, inp, nw, None)
    w_ceil = eng.debug_read("w_ceil", (B, 1, T))[:, 0].cuda()
    ylen, F = _begin(eng, inp, nw, w_ceil)
    ref, _, _, _ = eng.infer_finish(B, T, F, nz, KW["noise_scale"], want_attn=False, ragged=True)
    ref = ref.clone()
    rows = {k: [] for k in SETUPS}
    identical = True
    chunks = {}
    for r in range(warmup + rounds):
        for k, (ragged, cap) in SETUPS.items():
            o, *m, n = _stream(eng, inp, nw, nz, w_ceil, ragged, cap)
            chunks[k] = n
            if ragged:
                identical &= bool(torch.equal(o, ref))
            if r >= warmup:
                rows[k].append(m)
    frames = [int(v) for v in ylen]
    out = {"B": B, "tokens": lengths, "frames": frames, "F_max": F, "sum_L": sum(frames), "B_x_F_max": B * F,
           "generator_saving_if_proportional_to_frames": round(1 - sum(frames) / (B * F), 3),
           "ragged_streams_bit_identical_to_ragged_infer": identical}
    for k, rr in rows.items():
        med = [statistics.median(row[i] for row in rr) for i in range(4)]
        out[k] = {"first_chunk_ms": round(med[0], 3), "stream_ms": round(med[1], 3), "generator_ms": round(med[2], 3),
                  "launches": int(med[3]), "chunks": chunks[k]}
    for cap in ("", "_256"):
        p, g = out["padded" + cap], out["ragged" + cap]
        out["measured_saving_ragged_vs_padded" + cap] = {"generator": round(1 - g["generator_ms"] / p["generator_ms"], 3),
                                                         "stream": round(1 - g["stream_ms"] / p["stream_ms"], 3),
                                                         "first_chunk": round(1 - g["first_chunk_ms"] / p["first_chunk_ms"], 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ragged_stream.py measures on a CUDA device; none is available")
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    eng = Engine(cfg, sd, "cuda:0", "fp16")
    eng.set_profiling(True)
    name, q = card()
    res = {"gpu": name, "power_limit_max_sm_clock": q, "precision": "fp16", "rounds": a.rounds, "warmup": a.warmup,
           "schedule": f"{FIRST} frames, then doubling (up to {CAP} with the cap)",
           "note": "medians over rounds; setups alternate within each round; times on the host clock from infer_begin to the chunk's "
                   "completion event; generator_ms sums bv2_stage_ms('generator') over the advances; durations teacher-forced to the "
                   "padded batch's; generator_saving_if_proportional_to_frames is computed, not measured",
           "workloads": {}}
    for wname, lengths in workloads().items():
        w = run_workload(eng, cfg, lengths, a.rounds, a.warmup)
        res["workloads"][wname] = w
        print(f"{wname}: B={w['B']} sum(L)={w['sum_L']} B*F_max={w['B_x_F_max']} (computed saving "
              f"{w['generator_saving_if_proportional_to_frames']:.1%}), ragged bit-identical to infer(ragged=True): "
              f"{w['ragged_streams_bit_identical_to_ragged_infer']}")
        for k in SETUPS:
            s = w[k]
            print(f"  {k:10s} first chunk {s['first_chunk_ms']:8.3f} ms  stream {s['stream_ms']:8.3f} ms  generator {s['generator_ms']:8.3f} ms  "
                  f"launches {s['launches']:5d}  chunks {s['chunks']}")
        for cap in ("", "_256"):
            m = w["measured_saving_ragged_vs_padded" + cap]
            print(f"  measured{cap or ' (unbounded)'}: Generator {m['generator']:.1%}, stream {m['stream']:.1%}, first chunk "
                  f"{m['first_chunk']:.1%} less time ragged than padded")
    print(f"{name} ({q})")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
            f.write("\n")
    if not all(w["ragged_streams_bit_identical_to_ragged_infer"] for w in res["workloads"].values()):
        sys.exit("ragged streams are not bit-identical to infer(ragged=True)")


if __name__ == "__main__":
    main()
