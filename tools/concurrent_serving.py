#!/usr/bin/env python3
"""Concurrent config-2 requests on one GPU, written as JSON: SynthesizerTrn(concurrency=N).infer from M host threads against two
independent engines (bench.py's config2_two_workers: two engines, two host threads, two streams).

Every request is bench.py's config 2 (B=1, T=256 ZH, INFER_KW, seeded inputs and noise), followed by a synchronise of the calling
thread's stream.  Per setup:
  audio_s_per_s        valid audio seconds of all timed requests / host wall clock from the start gate to the last thread's end,
                       with the device synchronised on both sides
  latency_ms p50/p95   host clock per request, from the call to its stream synchronise (includes waiting for a free engine)
  launches_per_request kernels launched by all engines of the setup / requests
  workspace_bytes      per engine after the run
The setups run alternately, --reps rounds, so that they see the same host and device conditions; figures are medians over rounds.
memory_informational: cudaMemGetInfo deltas of creating one sibling and one independent engine (the GPU is shared, so other
processes can move these numbers).  The card's name and power limit are read in the same run (nvidia-smi queries only).

    python tools/concurrent_serving.py --out profiles/h100_concurrent_serving.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import CTOR, HOP, INFER_KW, SR, make_case  # noqa: E402
from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.models import SynthesizerTrn  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402

NAMES = ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")
POOL_SETUPS = [(1, 1), (1, 2), (2, 2), (4, 4)]  # (concurrency, host threads)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?"])[:2] if r.returncode == 0 else ("unknown", "unknown")
    return {"name": name, "power_limit": power}


def timed_threads(n_threads, per_thread, request):
    """runs request(k) per_thread times in each of n_threads threads behind a start gate; returns (wall s, latencies ms, frames)"""
    lat, frames, errors = [], [0] * n_threads, []
    gate = threading.Barrier(n_threads + 1)

    def worker(k):
        try:
            gate.wait()
            for _ in range(per_thread):
                t0 = time.perf_counter()
                frames[k] += request(k)
                lat.append((time.perf_counter() - t0) * 1e3)
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(n_threads)]
    for t in ths:
        t.start()
    torch.cuda.synchronize()
    gate.wait()
    c0 = time.perf_counter()
    for t in ths:
        t.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]
    return time.perf_counter() - c0, lat, sum(frames)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--requests", type=int, default=16, help="timed requests per host thread per round")
    ap.add_argument("--precision", default="fp16", choices=["fp32", "tf32", "fp16g", "fp16"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("concurrent_serving: no CUDA device (this script measures on the GPU only)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    inp, nw, nz = make_case(cfg)
    d = {k: v.to(dev) for k, v in inp.items()}
    d_nw, d_nz = nw.to(dev), nz.to(dev)
    B, T = d["x"].shape

    def make_net(concurrency):
        net = SynthesizerTrn(cfg.n_vocab, *CTOR, n_speakers=cfg.n_speakers, gin_channels=512, init_seed=None, precision=a.precision,
                             concurrency=concurrency)
        net.load_state_dict(sd, strict=False)
        return net.to(dev).eval()

    nets = {c: make_net(c) for c in sorted({c for c, _ in POOL_SETUPS})}
    # memory (informational): an independent engine uploads its own weight arena; a sibling allocates nothing on the device until
    # its first request sizes its workspace
    torch.cuda.synchronize()
    net_b = make_net(1)
    f0 = torch.cuda.mem_get_info(dev)[0]
    eng_b = net_b._engine(dev)
    torch.cuda.synchronize()
    f1 = torch.cuda.mem_get_info(dev)[0]
    sib = eng_b.sibling()
    torch.cuda.synchronize()
    f2 = torch.cuda.mem_get_info(dev)[0]
    del sib
    engs_indep = [nets[1]._engine(dev), eng_b]
    streams_indep = [torch.cuda.Stream(dev) for _ in engs_indep]
    for e in engs_indep:
        e.reserve(B, T, 2048)

    def net_request(net):
        def req(k):
            net.infer(*[d[n] for n in NAMES], noise_w=d_nw, noise_z=d_nz, **INFER_KW)
            torch.cuda.current_stream(dev).synchronize()
            return int(net.last_y_lengths.sum())
        return req

    def indep_request(k):
        eng, s = engs_indep[k], streams_indep[k]
        with torch.cuda.stream(s):
            yl, F = eng.infer_begin(*[d[n] for n in NAMES], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
            eng.infer_finish(B, T, F, d_nz, INFER_KW["noise_scale"], want_attn=False)
        s.synchronize()
        return int(yl.sum())

    setups = {f"pool_c{c}_t{t}": (t, net_request(nets[c]), (lambda c=c: nets[c]._pool(dev).engines)) for c, t in POOL_SETUPS}
    setups["independent_engines_2"] = (2, indep_request, lambda: engs_indep)
    # warm-up: every engine of every setup sized and its kernels loaded
    for name, (t, req, engines) in setups.items():
        timed_threads(t, 3, req)
    for c, n in nets.items():
        for e in n._pool(dev).engines:
            e.reserve(B, T, 2048)
    rounds = {name: [] for name in setups}
    for _ in range(a.reps):
        for name, (t, req, engines) in setups.items():
            l0 = sum(e.launch_count for e in engines())
            g0 = sum(e.workspace_grows for e in engines())
            dt, lat, frames = timed_threads(t, a.requests, req)
            rounds[name].append({"audio_s_per_s": frames * HOP / SR / dt, "wall_s": dt, "lat": lat,
                                 "launches_per_request": (sum(e.launch_count for e in engines()) - l0) / (t * a.requests),
                                 "workspace_grows": sum(e.workspace_grows for e in engines()) - g0})
            print(name, f"{rounds[name][-1]['audio_s_per_s']:.1f} audio-s/s", flush=True)
    results = {}
    for name, (t, req, engines) in setups.items():
        rs = rounds[name]
        lat = [x for r in rs for x in r["lat"]]
        results[name] = {"host_threads": t, "engines": len(engines()), "requests_per_round": t * a.requests,
                         "audio_s_per_s": statistics.median(r["audio_s_per_s"] for r in rs),
                         "audio_s_per_s_rounds": [r["audio_s_per_s"] for r in rs],
                         "latency_ms_p50": float(np.percentile(lat, 50)), "latency_ms_p95": float(np.percentile(lat, 95)),
                         "launches_per_request": statistics.median(r["launches_per_request"] for r in rs),
                         "workspace_grows_in_timed_rounds": sum(r["workspace_grows"] for r in rs),
                         "workspace_bytes_per_engine": [e.workspace_bytes for e in engines()]}
    _, F = engs_indep[0].infer_begin(*[d[n] for n in NAMES], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
    out = {"card": card(), "precision": a.precision, "workload": f"config 2: B={B}, T={T} ZH, {INFER_KW}, seeded (bench.py make_case)",
           "frames_per_request": int(F), "reps": a.reps, "timing": "host wall clock between device synchronisations; every request ends with a stream synchronise",
           "results": results,
           "memory_informational": {"note": "cudaMemGetInfo deltas on a shared GPU: informational only",
                                    "independent_engine_creation_bytes": int(f0 - f1), "sibling_creation_bytes": int(f1 - f2)}}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
