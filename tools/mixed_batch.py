#!/usr/bin/env python
"""Per-utterance settings: one ragged call for a dialogue whose speakers each have their own settings, against what a caller had to
do before (one call per setting group) and against B=1 calls.

Workload: a 10-sentence dialogue of 3 speakers on a synthetic checkpoint at the default configuration; each speaker has its own
length_scale / sdp_ratio / noise_scale / noise_scale_w.  Three setups, alternated within every round so that they see the same
machine state, all on the FP16 engine with ragged=True:
  mixed    one call, every sentence with its speaker's settings (bv2_infer_begin_items)
  grouped  one call per speaker (its sentences, its settings as scalars): the calls a caller made before
  b1       every sentence alone at B=1
Durations are teacher-forced (w_ceil_override) to those of the mixed call, so every setup synthesizes the same frames.  Reported per
setup (median over rounds): whole-call ms (host clock around infer_begin + infer_finish of every call of the setup, ending in a
device synchronise), Generator and flow stage ms (bv2_stage_ms, summed over the setup's calls), and kernel launches.  Outside the
timed rounds, every sentence of the mixed call is checked bit for bit against the same batch called with its settings as scalars
(the grouped calls run other shapes, so they are not a bitwise reference).

  python tools/mixed_batch.py [--rounds 10] [--warmup 2] [--out profiles/h100_mixed_batch.json]"""
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
from ragged_batch import card  # noqa: E402

# speaker -> (sid, noise_scale, noise_scale_w, length_scale, sdp_ratio)
SPEAKERS = {"A": (3, 0.6, 0.8, 1.0, 0.2), "B": (41, 0.667, 0.9, 0.85, 0.5), "C": (77, 0.5, 0.7, 1.2, 0.0)}
DIALOGUE = [("A", 42), ("B", 87), ("A", 23), ("C", 131), ("B", 56), ("A", 164), ("C", 38), ("B", 112), ("C", 71), ("A", 95)]


def _slice(inp, idx):
    """the sentences idx of the padded batch, re-padded to their own longest"""
    t = max(int(inp["x_lengths"][i]) for i in idx)
    ix = torch.tensor(idx, device=inp["x"].device)
    return {k: (v[ix][..., :t] if v.dim() >= 2 else v[ix]) for k, v in inp.items()}


def _call(eng, inp, nw, nz, w, settings):
    """one ragged infer_begin + infer_finish: settings is (ns, nsw, ls, sr) of floats or of [B] tensors.
    Returns (o, y_lengths, generator ms, flow ms, launches); the caller times the calls it groups."""
    B, T = inp["x"].shape
    ns, nsw, ls, sr = settings
    l0 = eng.launch_count
    per_item = isinstance(ns, torch.Tensor)
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, nsw, ls, sr, w_ceil_override=w, item_noise_scale=ns if per_item else None)
    o, _, _, _ = eng.infer_finish(B, T, F, nz, 1.0 if per_item else ns, want_attn=False, ragged=True)
    return o, ylen, eng.stage_ms("generator"), eng.stage_ms("flow"), eng.launch_count - l0


def _timed(eng, calls):
    """[(inp, nw, nz, w, settings)] run back to back -> (whole ms, generator ms, flow ms, launches), and the outputs"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    acc, outs = [0.0, 0.0, 0], []
    for c in calls:
        o, ylen, gm, fm, n = _call(eng, *c)
        acc = [acc[0] + gm, acc[1] + fm, acc[2] + n]
        outs.append((o, ylen))
    torch.cuda.synchronize()
    return [(time.perf_counter() - t0) * 1e3] + acc, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mixed_batch.py measures on a CUDA device; none is available")
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    eng = Engine(cfg, sd, "cuda:0", "fp16")
    eng.set_profiling(True)
    name, q = card()

    lengths = [t for _, t in DIALOGUE]
    B, T = len(lengths), max(lengths)
    inp = synth.synthetic_inputs(cfg, lengths, [i % 3 for i in range(B)], seed=12)
    inp["sid"] = torch.tensor([SPEAKERS[s][0] for s, _ in DIALOGUE])
    nw, nz = synth.synthetic_noise(cfg, B, T, 16 * T + 64, seed=12)
    inp = {k: v.cuda() for k, v in inp.items()}
    nw, nz = nw.cuda(), nz.cuda()
    cols = [torch.tensor([SPEAKERS[s][j] for s, _ in DIALOGUE], dtype=torch.float32, device="cuda") for j in (1, 2, 3, 4)]
    mixed_settings = tuple(cols)  # (ns, nsw, ls, sr) per sentence
    eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw,
                    cols[1], cols[2], cols[3], item_noise_scale=cols[0])
    w = eng.debug_read("w_ceil", (B, 1, T))[:, 0].cuda()

    mixed = [(inp, nw, nz, w, mixed_settings)]
    groups = {}
    for i, (s, _) in enumerate(DIALOGUE):
        groups.setdefault(s, []).append(i)
    grouped = []
    for s, idx in groups.items():
        sub = _slice(inp, idx)
        t = sub["x"].shape[1]
        grouped.append((sub, nw[idx][..., :t].contiguous(), nz[idx].contiguous(), w[idx][:, :t].contiguous(), SPEAKERS[s][1:]))
    b1 = [(_slice(inp, [i]), nw[i:i + 1, :, :t].contiguous(), nz[i:i + 1].contiguous(), w[i:i + 1, :t].contiguous(), SPEAKERS[s][1:])
          for i, (s, t) in enumerate(DIALOGUE)]

    # every sentence of the mixed call against the same batch with its settings as scalars (outside the timed rounds)
    _, outs = _timed(eng, mixed)
    o_mix, ylen = outs[0]
    identical = True
    for s, idx in groups.items():
        _, ref = _timed(eng, [(inp, nw, nz, w, SPEAKERS[s][1:])])
        for i in idx:
            identical &= bool(torch.equal(o_mix[i], ref[0][0][i])) and int(ref[0][1][i]) == int(ylen[i])

    setups = {"mixed": mixed, "grouped": grouped, "b1": b1}
    rows = {k: [] for k in setups}
    for r in range(a.warmup + a.rounds):
        for k, calls in setups.items():
            m, _ = _timed(eng, calls)
            if r >= a.warmup:
                rows[k].append(m)
    frames = [int(v) for v in ylen]
    res = {"gpu": name, "power_limit_max_sm_clock": q, "precision": "fp16", "ragged": True, "rounds": a.rounds, "warmup": a.warmup,
           "note": "medians over rounds; setups alternate within each round; grouped = one call per speaker (setting group), b1 = one "
                   "call per sentence, summed; durations teacher-forced to the mixed call's; call_ms is the host clock around all "
                   "calls of a setup, ending in a device synchronise",
           "speakers": {s: dict(zip(("sid", "noise_scale", "noise_scale_w", "length_scale", "sdp_ratio"), v)) for s, v in SPEAKERS.items()},
           "dialogue": [{"speaker": s, "tokens": t, "frames": f} for (s, t), f in zip(DIALOGUE, frames)],
           "B": B, "setting_groups": len(groups), "mixed_bit_identical_to_uniform_calls": identical, "setups": {}}
    for k, rs in rows.items():
        med = [statistics.median(row[i] for row in rs) for i in range(4)]
        res["setups"][k] = {"calls": len(setups[k]), "call_ms": round(med[0], 3), "generator_ms": round(med[1], 3),
                            "flow_ms": round(med[2], 3), "launches": int(med[3])}
    for k, s in res["setups"].items():
        print(f"{k:8s} calls {s['calls']:3d}  call {s['call_ms']:8.3f} ms  generator {s['generator_ms']:8.3f} ms  flow {s['flow_ms']:7.3f} ms  "
              f"launches {s['launches']:5d}")
    print(f"mixed sentences bit-identical to uniform-settings calls: {identical}")
    print(f"{name} ({q})")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
            f.write("\n")
    if not identical:
        sys.exit("mixed-settings sentences are not bit-identical to the uniform-settings calls")


if __name__ == "__main__":
    main()
