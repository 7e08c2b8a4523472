#!/usr/bin/env python
"""Benchmark of the SynthesizerTrn.infer hot path (BASELINE.json metric: audio-sec/s at 44.1 kHz).

    python bench.py --gpus N --steps K --warmup W            # this repo's CUDA engine
    python bench.py --impl reference --gpus N --steps K ...  # the reference algorithm on the host CPU cores (same config)

A "step" is one whole infer() over one batch of synthetic get_text() outputs.  Headline workload = BASELINE.json
configs[1] ("config 2": B=1, 256-phoneme ZH utterance, 44.1 kHz, full path enc_p -> SDP/DP -> length regulation -> flow ->
Generator), calibrated as SURVEY.md section 8d prescribes: the API's own `length_scale` is set so that the utterance comes out
at ~4 frames/token (~1022 frames = 11.9 s of audio, a trained model's speech rate); the un-calibrated run (length_scale 1,
1573 frames, round 1's workload) is reported next to it.  Synthetic seeded weights of the reference architecture (no network).

  value     whole-job audio-seconds per second, inputs resident in HBM (CUDA events, barrier + synchronize on both sides,
            max over ranks)
  e2e       the same through the public drop-in API SynthesizerTrn.infer() from pinned HOST buffers: H2D of the step's
            inputs and D2H of the waveform inside the timed region
  roofline  Generator stage (>99 % of FLOPs): algorithmic layer-boundary bytes (SURVEY.md section 8d: 6 830 852 B per frame) /
            device time of the stage measured with CUDA events inside the timed steps, against MEASURED_PEAKS.json
  cpu_baseline  the CPU oracle port of the reference (oracle/vits2_oracle.py; the reference itself does not exist on the GPU
            box) on the host cores, on the SAME utterance
  extras    config2_length_scale_1, config3_batched (B=32, per-stage ms), config5_generator (F=1024 + F/B roofline sweep),
            flow_wn (config 2 with use_transformer_flow=False), and at N>1 config4_sharded (length-bucketed ragged batches
            dealt to the ranks)

Multi-GPU (--gpus N under torchrun): utterances shard embarrassingly; every rank runs the SAME utterance (identical frame
count: clean weak scaling) and the waveforms land on rank 0 (fused peer-store epilogue by default).
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402

SR, HOP = 44100, 512
GEN_BYTES_PER_FRAME = 6_830_852      # SURVEY.md section 8d, layer-boundary algorithmic bytes, fp32 activations
GEN_FLOP_PER_FRAME = 651_608_576     # SURVEY.md section 8d (exact)
# webui defaults (webui.py:443-454) except length_scale: calibrated with the oracle so that the seeded config-2 utterance
# (256 tokens) yields ~4 frames/token (SURVEY.md section 8d "calibrate with the API's own length_scale"); 1.0 gives 6.1 frames/token
LENGTH_SCALE_CAL = 0.625
INFER_KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=LENGTH_SCALE_CAL)
WORKLOAD = dict(B=1, T=256, languages=[0], seed=2)  # BASELINE.json configs[1]
WORKLOAD_NAME = "config2: B=1, T=256 ZH phonemes, full SynthesizerTrn.infer path (transformer flow), length_scale 0.625 (~4 frames/token)"
CTOR = (1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512, [16, 16, 8, 2, 2])
DTYPES = {"tf32": "tf32", "fp16": "f16xf16+f32acc", "fp16g": "f16xf16+f32acc", "fp32": "f32"}


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        d = json.load(open(p))
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "data sheet (H100 SXM HBM3)"


def build_id(only=None):
    """Hash of the CUDA sources: profile-derived numbers (roofline.traffic) are only attached when they were captured on this build."""
    h = hashlib.sha256()
    d = os.path.join(ROOT, "bert_vits2_b200", "csrc")
    for f in sorted(os.listdir(d)):
        if f.endswith((".cu", ".cuh")) and (only is None or f in only):
            h.update(open(os.path.join(d, f), "rb").read())
    return h.hexdigest()[:16]


#: the sources the Generator's launches are compiled from (k_g2_conv, conv_post, the H8 conversion, their host code): the DRAM bytes of
#: those launches cannot change with an edit elsewhere (e.g. the attention kernel), so the traffic capture is keyed on these files
GENERATOR_SOURCES = ("common.cuh", "tc_conv.cuh", "tc_gen.cuh", "engine.cu")


def generator_build_id():
    return build_id(GENERATOR_SOURCES)


class ClockSampler:
    """nvidia-smi clocks/throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx = float(f[1])
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": mx, "samples": len(sm), "reasons": sorted(reasons)}


def host_cores():
    """Usable host threads: affinity mask capped by the cgroup CPU quota (os.cpu_count() ignores both)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = max(1, min(n, int(float(q) / float(per))))
    except Exception:
        pass
    return n


def make_case(cfg, T=None, B=None, languages=None, seed=None, fcap=4096):
    wl = WORKLOAD
    T = wl["T"] if T is None else T
    B = wl["B"] if B is None else B
    languages = (wl["languages"] * B) if languages is None else languages
    seed = wl["seed"] if seed is None else seed
    inp = synth.synthetic_inputs(cfg, [T] * B, languages, seed=seed)
    nw, nz = synth.synthetic_noise(cfg, B, T, fcap, seed=seed)
    return inp, nw, nz


def cpu_oracle_rate(cfg, sd, budget_s=25.0, max_iters=3):
    """The reference's CPU algorithm (oracle port) on the SAME config-2 utterance (same ids, features, noise, length_scale)."""
    from oracle import vits2_oracle as O
    avail = host_cores()
    # pick the thread count that serves the reference best on this host (all threads can be far slower than a subset on
    # many-core boxes because the path is ~12 k small ATen ops): probe on a 16-phoneme utterance
    pin = synth.synthetic_inputs(cfg, [16], [0], seed=3)
    pnw, pnz = synth.synthetic_noise(cfg, 1, 16, 1024, seed=3)
    best, cores = None, avail
    for n_thr in sorted({min(avail, 8), min(avail, 16), min(avail, 32), min(avail, 64), avail}):
        torch.set_num_threads(n_thr)
        c0 = time.perf_counter()
        O.infer(sd, cfg, **pin, noise_w=pnw, noise_z=pnz, **INFER_KW)
        dt = time.perf_counter() - c0
        if best is not None and dt > 3 * best:
            break  # oversubscribed: do not pay for a second, timed call
        c0 = time.perf_counter()
        O.infer(sd, cfg, **pin, noise_w=pnw, noise_z=pnz, **INFER_KW)
        dt = time.perf_counter() - c0
        if best is None or dt < best:
            best, cores = dt, n_thr
        elif dt > 1.1 * best:
            break  # more threads stopped helping
    torch.set_num_threads(cores)
    inp, nw, nz = make_case(cfg)
    secs, n, audio, frames = 0.0, 0, 0.0, 0
    t_start = time.perf_counter()
    for i in range(max_iters + 1):
        c0 = time.perf_counter()
        oo, _, ym, _ = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, **INFER_KW)
        dt = time.perf_counter() - c0
        if i:
            secs += dt; n += 1; frames = int(ym.sum()); audio += frames * HOP / SR
        if time.perf_counter() - t_start > budget_s and n >= 1:
            break
    return {"value": audio / secs, "unit": "audio-s/s", "cores": cores, "cores_available": avail, "kind": "port",
            "sample": f"{n} x the whole config-2 utterance (T=256, {frames} frames, {audio / n:.2f} s audio each) after 1 warm-up, torch CPU fp32 "
                      f"oracle port of the reference, weight-norm re-evaluated per call"}, secs / n, frames


def config_dict(frames, world=1, precision=None, parallelism="single GPU"):
    d = {"workload": WORKLOAD_NAME, "global_batch": world * WORKLOAD["B"], "T": WORKLOAD["T"], "length_scale": LENGTH_SCALE_CAL,
         "frames_per_utterance": frames, "audio_seconds_per_utterance": frames * HOP / SR, "parallelism": parallelism,
         "l2": "no explicit flush: the working set of one step (Generator activations of ~1000 frames x 512 hop) is far beyond the 50 MB L2"}
    if precision:
        d["precision"] = precision
    return d


def run_reference(args, rank, world):
    """--impl reference: the reference's CPU algorithm (oracle port) on all useful host threads, same config/metric."""
    if rank != 0:
        return
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    steps, warm = max(1, min(args.steps, 5)), 1
    cb, sec_per, frames = cpu_oracle_rate(cfg, sd, budget_s=90.0, max_iters=steps)
    v = cb["value"]
    line = {
        "impl": "reference", "metric": "audio-sec/s (real-time factor) at 44.1kHz", "value": v, "unit": "audio-s/s", "n_gpus": args.gpus,
        "steps": steps, "warmup": warm, "ms_per_step": 1e3 * sec_per, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": config_dict(frames, 1, None, "host CPU threads"),
        "cpu_baseline": cb,
        "e2e": {"value": v, "unit": "audio-s/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def build_net(cfg, sd, dev, precision, use_transformer_flow=True):
    from bert_vits2_b200.models import SynthesizerTrn
    net = SynthesizerTrn(cfg.n_vocab, *CTOR, n_speakers=cfg.n_speakers, gin_channels=512, init_seed=None, precision=precision,
                         use_transformer_flow=use_transformer_flow)
    net.load_state_dict(sd, strict=False)
    return net.to(dev).eval()


def time_resident(eng, d_inp, d_nw, d_nz, kw, steps, warmup, dev):
    """Device-resident steps of one workload on one engine; returns (ms_per_step, frames_per_step, stage means, launches, F_padded)."""
    B, T = d_inp["x"].shape
    Fm = [0]

    def step():
        ylen, F = eng.infer_begin(d_inp["x"], d_inp["x_lengths"], d_inp["sid"], d_inp["tone"], d_inp["language"], d_inp["bert"],
                                  d_inp["ja_bert"], d_inp["en_bert"], d_nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"])
        eng.infer_finish(B, T, F, d_nz, kw["noise_scale"], want_attn=False)
        Fm[0] = F
        return int(ylen.sum())
    for _ in range(warmup):
        step()
    torch.cuda.synchronize(dev)
    l0 = eng.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fr, st = 0, {"encoder_duration": [], "flow": [], "generator": []}
    for _ in range(steps):
        fr += step()
        for k in st:
            st[k].append(eng.stage_ms(k))
    e1.record(); torch.cuda.synchronize(dev)
    ms = e0.elapsed_time(e1)
    return ms / steps, fr / steps, {k: float(np.mean(v)) for k, v in st.items()}, (eng.launch_count - l0) / steps, Fm[0]


def dump_outputs(out_dir, wave, y_lengths):
    """The arrays the timed path handed its caller in the last step, as .npy files (inputs are seeded: two builds of the project can
    be compared output for output): wave.npy = the waveform batch [B, 1, samples] (float32, samples past an utterance's length are
    padding), y_samples.npy = the valid samples of each utterance (y_lengths * hop, float64)."""
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "wave.npy"), wave.detach().float().cpu().numpy())
    np.save(os.path.join(out_dir, "y_samples.npy"), np.asarray(torch.as_tensor(y_lengths).cpu(), dtype=np.float64).reshape(-1) * HOP)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--precision", default=os.environ.get("BV2_PRECISION", "fp16"), choices=["fp32", "tf32", "fp16g", "fp16"])
    ap.add_argument("--cpu-baseline-steps", type=int, default=3)
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write what the last timed step returned (waveform batch, per-utterance sample counts) as DIR/<name>.npy")
    ap.add_argument("--extras", type=int, default=1, help="0: headline line only (config2_length_scale_1, config3, config5, flow_wn, config4 skipped)")
    ap.add_argument("--exchange", default="p2p", choices=["p2p", "nccl", "none"],
                    help="N>1: how the finished waveforms reach rank 0 inside the timed region (see step_resident)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    args.warmup = max(args.warmup, 3)
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(cfg, 0)
    net = build_net(cfg, sd, dev, args.precision)
    eng = net._engine(dev)
    eng.set_profiling(True)
    inp, nw, nz = make_case(cfg)  # every rank: the same utterance (identical frame count -> clean weak scaling)
    B, T = inp["x"].shape
    d_inp = {k: v.to(dev) for k, v in inp.items()}
    d_nw, d_nz = nw.to(dev), nz.to(dev)
    h_inp = {k: v.pin_memory() for k, v in inp.items()}
    eng.reserve(B, T, 2048)  # workspace sized up front: no allocation on the hot call

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    from bert_vits2_b200.sharding import PeerWaveSlab, gather_waveforms

    # ---- multi-GPU exchange step (SURVEY.md section 8e).  Utterances shard with no data-path collective; the finished waveforms
    # are collected on rank 0.  --exchange p2p (default): the Generator's conv_post+tanh epilogue stores straight into a
    # CUDA-IPC mapped slab in rank 0's HBM over NVLink/NVSwitch (fused compute + transfer, NCCL carries a 4-byte flag);
    # --exchange nccl: padded NCCL gather of the finished tensors (baseline); --exchange none: every rank keeps its output.
    exchange = args.exchange if world > 1 else "none"
    slab = None
    step_no = [0]
    if exchange == "p2p":
        _, F0 = eng.infer_begin(d_inp["x"], d_inp["x_lengths"], d_inp["sid"], d_inp["tone"], d_inp["language"], d_inp["bert"],
                                d_inp["ja_bert"], d_inp["en_bert"], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"],
                                INFER_KW["sdp_ratio"])
        eng.infer_finish(B, T, F0, d_nz, INFER_KW["noise_scale"], want_attn=False)
        fcap = torch.tensor([F0], device=dev); dist.all_reduce(fcap, op=dist.ReduceOp.MAX)
        try:
            slab = PeerWaveSlab(dev, B, 2 * int(fcap) * HOP, dst=0, slots=2)
        except RuntimeError as ex:  # raised on every rank together (collective constructor): fall back to the NCCL gather
            if rank == 0:
                print(f"[bench] peer slab unavailable ({ex}); using the NCCL gather", file=sys.stderr, flush=True)
            exchange = "nccl"

    last_out = [None, None]  # (waveform batch, per-utterance frame counts) of the latest step_resident()

    def step_resident():
        ylen, F = eng.infer_begin(d_inp["x"], d_inp["x_lengths"], d_inp["sid"], d_inp["tone"], d_inp["language"], d_inp["bert"],
                                  d_inp["ja_bert"], d_inp["en_bert"], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"],
                                  INFER_KW["sdp_ratio"])
        if slab is not None:
            slot = step_no[0] % 2; step_no[0] += 1
            slab.wait(slot)  # slot reuse: ordered after the completion flag of the step that used it last
            if not slab.fits(B, F * HOP):
                raise RuntimeError("waveform batch exceeds the peer slab slot")
            o, attn, y_mask, aux = eng.infer_finish(B, T, F, d_nz, INFER_KW["noise_scale"], out_ptr=slab.wave_ptr(slot), want_attn=False)
            slab.publish(slot, B, F * HOP, ylen * HOP)
            slab.release(slot)  # back-pressure protocol (the root consumes nothing in this loop: see step_e2e for the consuming variant)
        else:
            o, attn, y_mask, aux = eng.infer_finish(B, T, F, d_nz, INFER_KW["noise_scale"], want_attn=False)
            if exchange == "nccl":
                gather_waveforms(o, torch.as_tensor(ylen, device=o.device) * HOP, dst=0)
        last_out[:] = [o, ylen]
        return int(ylen.sum()), o

    def step_e2e():
        dd = {k: v.to(dev, non_blocking=True) for k, v in h_inp.items()}
        o, attn, y_mask, aux = net.infer(dd["x"], dd["x_lengths"], dd["sid"], dd["tone"], dd["language"], dd["bert"], dd["ja_bert"],
                                         dd["en_bert"], **INFER_KW)
        if slab is not None:  # API-level variant: the caller holds the tensor, one peer copy puts it into rank 0's slab
            slot = step_no[0] % 2; step_no[0] += 1
            slab.wait(slot)
            slab.publish(slot, B, o.shape[-1], net.last_y_lengths * HOP, wave=o)
            if rank == 0:  # the root really consumes every rank's waveform each step: one device copy out of the slab per rank
                waves, counts = slab.collect(slot)
                keep = [w.clone() for w in waves]  # noqa: F841
            slab.release(slot)
        elif exchange == "nccl":
            gather_waveforms(o, torch.as_tensor(net.last_y_lengths, device=o.device) * HOP, dst=0)
        wav = o[:, 0].cpu()  # D2H of the step's result, as infer.py:315-318 does
        return int(net.last_y_lengths.sum()), wav

    def check_exchange():
        """After the timed loops: rank 0 reads every rank's last waveform out of the slab and compares its checksum with the
        one the producing rank computes from a local, un-exchanged run of the same inputs (bit-exact path)."""
        ylen, F = eng.infer_begin(d_inp["x"], d_inp["x_lengths"], d_inp["sid"], d_inp["tone"], d_inp["language"], d_inp["bert"],
                                  d_inp["ja_bert"], d_inp["en_bert"], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"],
                                  INFER_KW["sdp_ratio"])
        o_loc = eng.infer_finish(B, T, F, d_nz, INFER_KW["noise_scale"], want_attn=False)[0]
        eng.infer_begin(d_inp["x"], d_inp["x_lengths"], d_inp["sid"], d_inp["tone"], d_inp["language"], d_inp["bert"],
                        d_inp["ja_bert"], d_inp["en_bert"], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
        slab.wait(0)
        eng.infer_finish(B, T, F, d_nz, INFER_KW["noise_scale"], out_ptr=slab.wave_ptr(0), want_attn=False)
        slab.publish(0, B, F * HOP, ylen * HOP)
        mine = torch.stack([o_loc.double().abs().sum(), torch.tensor(float(F * HOP), device=dev, dtype=torch.float64)])
        allsum = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(allsum, mine)
        waves, counts = slab.collect(0)
        ok = True
        if rank == 0:
            for r in range(world):
                got = waves[r].double().abs().sum()
                ok &= bool(waves[r].shape[-1] == int(allsum[r][1])) and bool(torch.isfinite(waves[r]).all())
                ok &= bool(torch.allclose(got, allsum[r][0], rtol=1e-9, atol=0.0)) and float(got) > 0.0
            ok &= bool(torch.equal(waves[0], o_loc))
        return ok

    # ---------------- device-resident value
    for _ in range(args.warmup):
        step_resident()
    l0 = eng.launch_count
    g0 = eng.workspace_grows
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    frames, gen_ms, flow_l, enc_l = 0, [], [], []
    for _ in range(args.steps):
        f, o = step_resident()
        frames += f
        gen_ms.append(eng.stage_ms("generator"))  # blocks on this step's generator end event only
        flow_l.append(eng.stage_ms("flow")); enc_l.append(eng.stage_ms("encoder_duration"))
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop() if rank == 0 else None
    launches = eng.launch_count - l0
    flow_ms, enc_ms = float(np.mean(flow_l)), float(np.mean(enc_l))
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, *last_out)  # the last timed step
    # ---------------- end to end through the public API with host buffers
    for _ in range(args.warmup):
        step_e2e()
    barrier()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    frames_e = 0
    for _ in range(args.steps):
        f, wav = step_e2e()
        frames_e += f
    t1.record()
    barrier()
    ms_e = t0.elapsed_time(t1)
    grows = eng.workspace_grows - g0
    h2d = sum(v.numel() * v.element_size() for v in h_inp.values())
    d2h = wav.numel() * wav.element_size()
    exchange_ok = None
    if slab is not None:
        exchange_ok = check_exchange()
        slab.close()
    # ---------------- max over ranks (value), min/max over ranks (e2e spread)
    stats = torch.tensor([ms, ms_e, float(frames), float(frames_e)], device=dev, dtype=torch.float64)
    ms_e_min = ms_e
    if world > 1:
        mx = stats.clone(); dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        mn = stats.clone(); dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        sm = stats.clone(); dist.all_reduce(sm, op=dist.ReduceOp.SUM)
        ms, ms_e = float(mx[0]), float(mx[1]); frames, frames_e = float(sm[2]), float(sm[3]); ms_e_min = float(mn[1])

    # ---------------- config 4 (N > 1): B = 32 per rank, T ~ U{64..512}, length-bucketed and dealt to the ranks
    cfg4 = None
    if world > 1 and args.extras:
        try:
            from bert_vits2_b200.sharding import deal_buckets
            rng = np.random.Generator(np.random.Philox(key=[4, 0]))
            lengths = [int(v) for v in rng.integers(64, 513, size=32 * world)]
            plan = deal_buckets(lengths, world, 32)[rank]
            batches = []
            for bi, idxs in enumerate(plan):
                ls = [lengths[i] for i in idxs]
                inp4 = synth.synthetic_inputs(cfg, ls, [i % 3 for i in idxs], seed=400 + rank * 16 + bi)
                nw4, nz4 = synth.synthetic_noise(cfg, len(ls), max(ls), 4096, seed=400 + rank * 16 + bi)
                batches.append(({k: v.to(dev) for k, v in inp4.items()}, nw4.to(dev), nz4.to(dev)))

            def step4():
                fr = 0
                for d4, nw4, nz4 in batches:
                    yl, F4 = eng.infer_begin(d4["x"], d4["x_lengths"], d4["sid"], d4["tone"], d4["language"], d4["bert"], d4["ja_bert"],
                                             d4["en_bert"], nw4, INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
                    eng.infer_finish(d4["x"].shape[0], d4["x"].shape[1], F4, nz4, INFER_KW["noise_scale"], want_attn=False)
                    fr += int(yl.sum())
                return fr
            for _ in range(2):
                step4()
            barrier()
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record()
            fr4 = 0
            for _ in range(3):
                fr4 += step4()
            a1.record(); barrier()
            st4 = torch.tensor([a0.elapsed_time(a1), float(fr4)], device=dev, dtype=torch.float64)
            mx4 = st4.clone(); dist.all_reduce(mx4, op=dist.ReduceOp.MAX)
            sm4 = st4.clone(); dist.all_reduce(sm4, op=dist.ReduceOp.SUM)
            cfg4 = {"workload": f"config4: B={32 * world} utterances, T ~ U{{64..512}} (seeded), length-bucketed (deal_buckets) into batches of 32, one per rank",
                    "value": float(sm4[1]) * HOP / SR / (float(mx4[0]) * 1e-3), "unit": "audio-s/s", "ms_per_step": float(mx4[0]) / 3,
                    "valid_frames_per_step": float(sm4[1]) / 3}
        except Exception as ex:
            cfg4 = {"error": str(ex)[:200]}

    if rank == 0:
        audio = frames * HOP / SR
        value = audio / (ms * 1e-3)
        e2e_v = (frames_e * HOP / SR) / (ms_e * 1e-3)
        hbm, how = peaks()
        fpu = frames / (args.steps * world)  # frames per utterance-step on one GPU
        g_ms = float(np.mean(gen_ms))
        traffic, traffic_note = None, "no dram__bytes capture for this build (profiles/*_generator_traffic.json build_id mismatch or absent)"
        bid = build_id()
        pdir = os.path.join(ROOT, "profiles")
        for name in (sorted(os.listdir(pdir), reverse=True) if os.path.isdir(pdir) else []):
            if name.endswith("_generator_traffic.json"):
                tj = json.load(open(os.path.join(pdir, name)))
                if tj.get("build_id") == bid or tj.get("generator_build_id") == generator_build_id():  # dram__bytes_read+write summed over the Generator launches of one ncu capture (per frame)
                    traffic = tj["generator_dram_bytes_per_frame"] * fpu
                    traffic_note = f"profiles/{name} (" + ("same build" if tj.get("build_id") == bid else "same Generator sources") + ")"
                    break
        ach = GEN_BYTES_PER_FRAME * fpu / (g_ms * 1e-3) / 1e9
        par = (f"dp{world} (utterance sharding, identical utterance on every rank; waveforms to rank 0: " +
               {"p2p": "Generator epilogue stores into a CUDA-IPC slab over NVLink, 4-byte NCCL flag)",
                "nccl": "padded NCCL gather)", "none": "none)"}[exchange]) if world > 1 else "single GPU"
        line = {
            "metric": "audio-sec/s (real-time factor) at 44.1kHz", "value": value, "unit": "audio-s/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": DTYPES[args.precision], "data": "synthetic",
            "config": config_dict(fpu, world, args.precision, par),
            "e2e": {"value": e2e_v, "unit": "audio-s/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                    "ms_per_step": ms_e / args.steps, "ms_per_step_min_rank": ms_e_min / args.steps, "ms_per_step_max_rank": ms_e / args.steps,
                    "workspace_regrowths_in_timed_loops": int(grows)},
            "gpu_launches": int(launches),
            **({"exchange": {"kind": exchange, "verified": exchange_ok}} if world > 1 else {}),
            "clocks": clocks,
            "roofline": {"bound": "hbm", "kernel": "Generator stage (conv_pre .. conv_post+tanh, 98 convolutions)", "achieved": ach, "peak": hbm,
                         "unit": "GB/s", "frac": ach / hbm, "traffic": traffic, "traffic_source": traffic_note, "peak_source": how, "stage_ms": g_ms,
                         "tensor_tflops": GEN_FLOP_PER_FRAME * fpu / (g_ms * 1e-3) / 1e12, "build_id": bid,
                         "algorithmic_bytes_convention": "SURVEY.md 8d: fp32 layer-boundary tensors, 6 830 852 B per frame; the fp16 engine keeps the "
                                                         "Generator's tensors as 16-bit operand images, so its DRAM traffic is well below that figure",
                         "dram_gbs_actual": (traffic / (g_ms * 1e-3) / 1e9) if traffic else None},
            "stage_ms": {"encoder_duration": enc_ms, "flow": flow_ms, "generator": g_ms},
            "launches_per_step": launches / args.steps,
        }
        if cfg4 is not None:
            line["config4_sharded"] = cfg4
        if world == 1 and args.extras:
            extras(line, args, cfg, sd, eng, dev, d_inp, d_nw, d_nz, hbm)
        # CPU baseline on rank 0 at N=1 only: the same utterance on the host cores
        if world == 1 and args.cpu_baseline_steps > 0:
            line["cpu_baseline"], _, _ = cpu_oracle_rate(cfg, sd, budget_s=25.0, max_iters=args.cpu_baseline_steps)
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def extras(line, args, cfg, sd, eng, dev, d_inp, d_nw, d_nz, hbm):
    """Not the headline: the other BASELINE.json configs on the same engine (never allowed to break the contract line)."""
    # ---- config 2 without the length_scale calibration (round-1 workload: 1573 frames)
    try:
        kw = dict(INFER_KW, length_scale=1.0)
        ms1, fr1, st1, l1, _ = time_resident(eng, d_inp, d_nw, d_nz, kw, max(5, args.steps // 2), 2, dev)
        line["config2_length_scale_1"] = {"value": fr1 * HOP / SR / (ms1 * 1e-3), "unit": "audio-s/s", "ms_per_step": ms1, "frames": fr1,
                                          "stage_ms": st1, "roofline_frac": GEN_BYTES_PER_FRAME * fr1 / (st1["generator"] * 1e-3) / 1e9 / hbm,
                                          "launches_per_step": l1}
    except Exception as ex:
        line["config2_length_scale_1"] = {"error": str(ex)[:200]}
    # ---- config 3: B=32 mixed ZH/JA/EN 128-phoneme utterances
    try:
        inp3 = synth.synthetic_inputs(cfg, [128] * 32, [i % 3 for i in range(32)], seed=3)
        nw3, nz3 = synth.synthetic_noise(cfg, 32, 128, 2048, seed=3)
        d3 = {k: v.to(dev) for k, v in inp3.items()}
        ms3, fr3, st3, l3, F3 = time_resident(eng, d3, nw3.to(dev), nz3.to(dev), INFER_KW, 5, 2, dev)
        line["config3_batched"] = {"workload": "config3: B=32, T=128 mixed ZH/JP/EN, full path", "value": fr3 * HOP / SR / (ms3 * 1e-3), "unit": "audio-s/s",
                                   "ms_per_step": ms3, "valid_frames_per_step": fr3, "padded_frames": int(F3), "stage_ms": st3,
                                   "roofline_frac_padded": GEN_BYTES_PER_FRAME * 32 * F3 / (st3["generator"] * 1e-3) / 1e9 / hbm, "launches_per_step": l3}
    except Exception as ex:
        line["config3_batched"] = {"error": str(ex)[:200]}
    # ---- config 5: Generator-only, 1024-frame latent -> waveform, + the F / B roofline sweep
    try:
        def gen_time(Bg, Fg, iters):
            z, g = synth.synthetic_generator_inputs(cfg, Bg, Fg)
            z, g = z.to(dev), g.to(dev)
            out = torch.empty(Bg, 1, Fg * HOP, device=dev)
            for _ in range(2):
                eng.generator(z, g, out)
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            acc = []
            for _ in range(iters):
                eng.generator(z, g, out)
                acc.append(eng.stage_ms("generator"))
            b.record(); torch.cuda.synchronize(dev)
            return a.elapsed_time(b) / iters, float(np.mean(acc))
        ms5, st5 = gen_time(1, 1024, 10)
        sweep = []
        for Bg, Fg in ((1, 128), (1, 256), (1, 512), (1, 2048), (1, 4096), (8, 256), (8, 1024), (32, 128), (32, 512)):
            _, stg = gen_time(Bg, Fg, 3)
            sweep.append({"B": Bg, "F": Fg, "stage_ms": stg, "roofline_frac": GEN_BYTES_PER_FRAME * Bg * Fg / (stg * 1e-3) / 1e9 / hbm})
        line["config5_generator"] = {"workload": "config5: Generator-only, z[1,192,1024] -> wav[1,1,524288] through bv2_generator",
                                     "value": 1024 * HOP / SR / (ms5 * 1e-3), "unit": "audio-s/s", "ms_per_call": ms5, "stage_ms": st5,
                                     "roofline_frac": GEN_BYTES_PER_FRAME * 1024 / (st5 * 1e-3) / 1e9 / hbm,
                                     "tensor_tflops": GEN_FLOP_PER_FRAME * 1024 / (st5 * 1e-3) / 1e12, "sweep": sweep}
    except Exception as ex:
        line["config5_generator"] = {"error": str(ex)[:200]}
    # ---- config 2 served by TWO workers on one GPU (two engines, two host threads, two streams): consecutive single-utterance
    # requests overlap -- the latency-bound token-rate / flow stages of one request run under the Generator of the other.
    # Reported next to the strict one-request-at-a-time headline, never instead of it.
    try:
        import threading as _th
        net2 = build_net(cfg, sd, dev, args.precision)
        engs = [eng, net2._engine(dev)]
        for e_ in engs:
            e_.reserve(1, WORKLOAD["T"], 2048)
        nper = max(6, args.steps // 2)
        frames2 = [0, 0]

        def worker(k):
            st = torch.cuda.Stream(device=dev)
            with torch.cuda.stream(st):
                for it in range(nper + 2):
                    yl, F2 = engs[k].infer_begin(d_inp["x"], d_inp["x_lengths"], d_inp["sid"], d_inp["tone"], d_inp["language"], d_inp["bert"],
                                                 d_inp["ja_bert"], d_inp["en_bert"], d_nw, INFER_KW["noise_scale_w"], INFER_KW["length_scale"], INFER_KW["sdp_ratio"])
                    engs[k].infer_finish(1, WORKLOAD["T"], F2, d_nz, INFER_KW["noise_scale"], want_attn=False)
                    if it == 1:  # two warm-up requests per worker, then both start the timed part together
                        st.synchronize(); gate.wait()
                    if it >= 2:
                        frames2[k] += int(yl.sum())
                st.synchronize()
        gate = _th.Barrier(3)
        ths = [_th.Thread(target=worker, args=(k,)) for k in range(2)]
        for t_ in ths:
            t_.start()
        gate.wait()
        c0 = time.perf_counter()
        for t_ in ths:
            t_.join()
        torch.cuda.synchronize(dev)
        dt = time.perf_counter() - c0
        line["config2_two_workers"] = {"workload": "config 2, two engines / host threads / streams on ONE GPU, 1 utterance per request",
                                       "value": sum(frames2) * HOP / SR / dt, "unit": "audio-s/s", "requests": 2 * nper,
                                       "ms_per_request_amortised": 1e3 * dt / (2 * nper), "timing": "host wall clock between device synchronisations"}
        del net2, engs
    except Exception as ex:
        line["config2_two_workers"] = {"error": str(ex)[:200]}
    # ---- config 2 with the WN flow (use_transformer_flow=False: ResidualCouplingBlock, reference models.py:403-445)
    try:
        cfgw = ModelConfig(use_transformer_flow=False)
        sdw = synth.synthetic_state_dict(cfgw, 0)
        netw = build_net(cfgw, sdw, dev, args.precision, use_transformer_flow=False)
        engw = netw._engine(dev)
        engw.set_profiling(True)
        msw, frw, stw, lw, _ = time_resident(engw, d_inp, d_nw, d_nz, INFER_KW, max(5, args.steps // 2), 3, dev)
        line["flow_wn"] = {"workload": "config2 inputs, use_transformer_flow=False (ResidualCouplingBlock / WN flow)", "value": frw * HOP / SR / (msw * 1e-3),
                           "unit": "audio-s/s", "ms_per_step": msw, "frames": frw, "stage_ms": stw, "launches_per_step": lw}
        del engw, netw
    except Exception as ex:
        line["flow_wn"] = {"error": str(ex)[:200]}


if __name__ == "__main__":
    main()
