"""Per-utterance synthesis settings (bv2_infer_begin_items): every utterance of a batch carries its own noise_scale, noise_scale_w,
length_scale and sdp_ratio.  Utterance b of a mixed batch is bit-identical to the same batch called with b's settings as scalars,
in the durations and, with the same frames, in everything finish writes (padded, ragged, pcm16, streams); uniform arrays equal the
scalar call with the same launches and workspace; each utterance matches the CPU oracle run of it alone with its own settings; and
the error paths and concurrent serving.  Run on an H100: pytest -m gpu."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Engine
from util import model_for, rms

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "fp16g", "fp16"]
FP16 = ("fp16", "fp16g")
LENGTHS = [64, 9, 30, 21, 14, 5]
# (noise_scale, noise_scale_w, length_scale, sdp_ratio) per utterance: sdp_ratio 0 and 1, length_scale below and above 1
SETTINGS = [(0.667, 0.8, 1.0, 0.0), (0.3, 1.1, 0.7, 1.0), (0.9, 0.5, 1.3, 0.5), (0.0, 0.0, 1.05, 0.2), (1.2, 0.9, 0.85, 0.8),
            (0.5, 0.667, 1.6, 0.35)]
CTOR = (112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512, [16, 16, 8, 2, 2])
NAMES = ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")
TOL_WAV = 1e-3  # waveform RMS against the oracle: the FP16 Generator's bar (test_ragged_gpu.py)


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(precision):
        if precision not in cache:
            cfg, sd = model_for(True, 0)
            cache[precision] = Engine(cfg, sd, device="cuda:0", precision=precision)
        return cache[precision]

    yield get
    cache.clear()


@pytest.fixture(scope="module")
def case():
    """B=6 batch of spread lengths, its noise, and teacher-forced durations of 3 to 6 frames per token (item 0: over 256 frames)"""
    cfg, _ = model_for(True, 0)
    B, T = len(LENGTHS), max(LENGTHS)
    inp = synth.synthetic_inputs(cfg, LENGTHS, [b % 3 for b in range(B)], seed=71)
    inp["sid"] = torch.tensor([0, 1, 2, 1, 0, 2])
    nw, nz = synth.synthetic_noise(cfg, B, T, 6 * T + 8, seed=71)
    w = torch.zeros(B, T)
    r = np.random.default_rng(71)
    for b, t in enumerate(LENGTHS):
        w[b, :t] = torch.as_tensor(r.integers(3, 7, size=t), dtype=torch.float32)
    return inp, nw, nz, w


def _cols(i):
    return torch.tensor([s[i] for s in SETTINGS], dtype=torch.float32)


def _begin(eng, inp, nw, s, w=None):
    """s: one (noise_scale, noise_scale_w, length_scale, sdp_ratio) for every utterance (the scalar call), or None: SETTINGS per
    utterance.  Returns (y_lengths, F, the noise_scale finish takes)."""
    args = [inp[k] for k in NAMES] + [nw]
    if s is not None:
        ylen, F = eng.infer_begin(*args, s[1], s[2], s[3], w_ceil_override=w)
        return ylen, F, s[0]
    ylen, F = eng.infer_begin(*args, _cols(1), _cols(2), _cols(3), w_ceil_override=w, item_noise_scale=_cols(0))
    return ylen, F, 1.0


def _taps(eng, B, T):
    return [eng.debug_read(n, (B, 1, T)).clone() for n in ("logw_sdp", "logw_dp", "w_ceil")]


def _finish(eng, case, s, mode):
    """one teacher-forced call in `mode` -> (o, [y_mask, z, z_p, m_p, logs_p]) on the CPU"""
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    _, F, ns = _begin(eng, inp, nw, s, w)
    kind, cap = mode
    if kind in ("padded", "ragged", "pcm16", "ragged_pcm16"):
        o, _, ym, aux = eng.infer_finish(B, T, F, nz, ns, want_attn=False, pcm16=kind.endswith("pcm16"), ragged=kind.startswith("ragged"))
    else:
        o, _, ym, aux = eng.infer_finish_stream(B, T, F, nz, ns, want_attn=False, max_chunk_frames=cap, ragged=kind == "ragged_stream")
        f, step, Fg = 0, 1, o.shape[-1] // eng.cfg.hop
        while f < Fg:
            f = min(f + step, Fg)
            eng.stream_advance(f)
            step = 2 * step if cap is None else min(2 * step, cap)
    torch.cuda.synchronize()
    return o.cpu(), [ym.cpu()] + [a.cpu() for a in aux]


def _modes(precision):
    out = [("padded", None), ("pcm16", None), ("stream", None)]
    if precision in FP16:
        out += [("ragged", None), ("ragged_pcm16", None), ("stream", 7), ("stream", 256), ("ragged_stream", 7), ("ragged_stream", 256)]
    return out


# ---------------------------------------------------------------- 1. mixed against uniform, bitwise
@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_durations_equal_uniform_calls(engines, precision, case):
    eng = engines(precision)
    inp, nw, _, _ = case
    B, T = inp["x"].shape
    ylen, _, _ = _begin(eng, inp, nw, None)
    mixed = _taps(eng, B, T)
    for b, s in enumerate(SETTINGS):
        ylen_b, _, _ = _begin(eng, inp, nw, s)
        assert ylen_b[b] == ylen[b], (precision, b)
        for name, got, want in zip(("logw_sdp", "logw_dp", "w_ceil"), mixed, _taps(eng, B, T)):
            assert torch.equal(got[b], want[b]), (precision, b, name)
    assert len(set(ylen.tolist())) > 1


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_outputs_equal_uniform_calls(engines, precision, case):
    eng = engines(precision)
    for mode in _modes(precision):
        o, rest = _finish(eng, case, None, mode)
        for b, s in enumerate(SETTINGS):
            o_b, rest_b = _finish(eng, case, s, mode)
            assert torch.equal(o[b], o_b[b]), (precision, mode, b, "o")
            for name, got, want in zip(("y_mask", "z", "z_p", "m_p", "logs_p"), rest, rest_b):
                assert torch.equal(got[b], want[b]), (precision, mode, b, name)
        assert not torch.equal(o[0], o_b[0]), mode  # item 0 under item 5's noise_scale: the setting does reach the output


# ---------------------------------------------------------------- 2. uniform arrays equal the scalar call
@pytest.mark.parametrize("precision", PRECISIONS)
def test_uniform_arrays_equal_scalar_call(engines, precision, case):
    eng = engines(precision)
    inp, nw, nz, _ = case
    B, T = inp["x"].shape
    ns, nsw, ls, sr = 0.6, 0.9, 0.8, 0.4
    args = [inp[k] for k in NAMES] + [nw]
    full = lambda v: torch.full((B,), v)  # noqa: E731
    variants = {  # (begin arguments, finish noise_scale)
        "scalar": (dict(noise_scale_w=nsw, length_scale=ls, sdp_ratio=sr), ns),
        "arrays": (dict(noise_scale_w=full(nsw), length_scale=full(ls), sdp_ratio=full(sr), item_noise_scale=full(ns)), 1.0),
        "arrays_scalar_noise": (dict(noise_scale_w=full(nsw), length_scale=ls, sdp_ratio=sr), ns),
    }
    cap = 32 if precision in FP16 else None
    ylen, F = eng.infer_begin(*args, nsw, ls, sr)
    eng.reserve_stream(B, T, F, cap)
    grows, ws = eng.workspace_grows, eng.workspace_bytes
    res = {}
    for name, (kw, fin) in variants.items():
        l0 = eng.launch_count
        ylen_v, F_v = eng.infer_begin(*args, **kw)
        taps = _taps(eng, B, T)
        o, _, ym, aux = eng.infer_finish(B, T, F_v, nz, fin, want_attn=False)
        eng.infer_begin(*args, **kw)
        so, *_ = eng.infer_finish_stream(B, T, F_v, nz, fin, want_attn=False, max_chunk_frames=cap)
        f = 0
        while f < F_v:
            f = min(f + 32, F_v)
            eng.stream_advance(f)
        torch.cuda.synchronize()
        res[name] = (ylen_v.tolist(), taps, o.cpu(), ym.cpu(), [a.cpu() for a in aux], so.cpu(), eng.launch_count - l0)
        assert eng.workspace_grows == grows and eng.workspace_bytes == ws, (precision, name)
    ref = res["scalar"]
    for name, got in res.items():
        assert got[0] == ref[0] and got[6] == ref[6], (precision, name, "y_lengths / launches")
        assert all(torch.equal(a, b) for a, b in zip(got[1], ref[1])), (precision, name, "duration taps")
        assert torch.equal(got[2], ref[2]) and torch.equal(got[3], ref[3]) and torch.equal(got[5], ref[5]), (precision, name, "o / y_mask")
        assert all(torch.equal(a, b) for a, b in zip(got[4], ref[4])), (precision, name, "z / z_p / m_p / logs_p")


# ---------------------------------------------------------------- 3. each utterance against the CPU oracle run alone
@pytest.mark.parametrize("precision", FP16)
def test_items_vs_oracle_alone(engines, precision, case):
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    inp, nw, nz, _ = case
    B, T = inp["x"].shape
    alone, w_ceil = [], torch.zeros(B, T)
    for b, (t, s) in enumerate(zip(LENGTHS, SETTINGS)):
        one = {k: (v[b:b + 1, ..., :t] if v.dim() >= 2 else v[b:b + 1]) for k, v in inp.items()}
        one["x_lengths"] = torch.tensor([t])
        st = O.infer(sd, cfg, **one, noise_w=nw[b:b + 1, :, :t], noise_z=nz[b:b + 1], return_stages=True, noise_scale=s[0],
                     noise_scale_w=s[1], length_scale=s[2], sdp_ratio=s[3])
        alone.append(st)
        w_ceil[b, :t] = torch.as_tensor(st["w_ceil"]).reshape(-1)[:t]
    eng = engines(precision)
    ylen, F, ns = _begin(eng, inp, nw, None, w_ceil)
    assert ylen.tolist() == [int(st["y_lengths"][0]) for st in alone]
    o, _, _, _ = eng.infer_finish(B, T, F, nz, ns, want_attn=False, ragged=True)
    o = o.cpu()
    for b, st in enumerate(alone):
        n = int(ylen[b]) * cfg.hop
        ref = torch.as_tensor(st["o"]).reshape(-1)
        assert ref.numel() == n
        e = rms(o[b, 0, :n], ref)
        print(f"[{precision}] item {b} {SETTINGS[b]}: frames {int(ylen[b])}, waveform RMS vs oracle alone {e:.2e}")
        assert e < TOL_WAV
        assert (o[b, 0, n:] == 0).all()


# ---------------------------------------------------------------- 4. errors
def test_null_setting_array_is_rejected(engines, case):
    eng = engines("fp16")
    inp, nw, nz, _ = case
    B, T = inp["x"].shape
    dev = [eng._i64(inp[k]) for k in NAMES[:5]] + [eng._f32(inp[k]) for k in NAMES[5:]] + [eng._f32(nw)]
    ones = torch.ones(B, device=eng.device)
    ylen, fmax = (C.c_int64 * B)(), C.c_int32(0)
    p = [C.c_void_p(t.data_ptr()) for t in dev]
    for hole in range(4):
        arrays = [None if i == hole else C.c_void_p(ones.data_ptr()) for i in range(4)]
        rc = eng.lib.bv2_infer_begin_items(eng._h, B, T, *p, *arrays, None, eng._stream(), ylen, C.byref(fmax))
        assert rc == -1, (hole, rc)
    with pytest.raises(ValueError):
        eng.infer_begin(*[inp[k] for k in NAMES], nw, torch.ones(B + 1), 1.0, 0.0)
    # the engine serves the next call
    _, F, _ = _begin(eng, inp, nw, None)
    o, *_ = eng.infer_finish(B, T, F, nz, 1.0, want_attn=False)
    assert torch.isfinite(o).all()


def _net(precision="fp16", concurrency=1):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, _ = model_for(True, 0)
    return SynthesizerTrn(*CTOR, n_speakers=cfg.n_speakers, gin_channels=512, precision=precision, init_seed=0,
                          concurrency=concurrency).to("cuda")


def test_module_rejects_wrong_length_or_rank(case):
    net = _net()
    inp, nw, _, _ = case
    args = [inp[k].cuda() for k in NAMES]
    B = args[0].shape[0]
    for bad in (dict(length_scale=[1.0] * (B - 1)), dict(sdp_ratio=torch.zeros(B, 1)), dict(noise_scale=torch.ones(B + 2, device="cuda")),
                dict(noise_scale_w=[[0.8]] * B)):
        with pytest.raises(ValueError):
            net.infer(*args, **bad)
        with pytest.raises(ValueError):
            next(net.infer_stream(*args, **bad))
    assert torch.isfinite(net.infer(*args, noise_w=nw.cuda())[0]).all()


# ---------------------------------------------------------------- 5. the module, serially and concurrently
def _module_kw(case):
    inp, nw, nz, w = case
    return [inp[k].cuda() for k in NAMES], dict(noise_w=nw.cuda(), noise_z=nz.cuda(), w_ceil_override=w.cuda())


def test_module_mixed_equals_uniform_and_concurrency(case):
    """SynthesizerTrn.infer / infer_stream with per-utterance settings (a device tensor, a CPU tensor, a list and a tuple): item b
    equals the module's scalar call with b's settings; with concurrency=2, two threads with different settings get exactly the
    concurrency=1 results"""
    args, kw = _module_kw(case)
    per_item = dict(noise_scale=_cols(0).cuda(), noise_scale_w=_cols(1), length_scale=[s[2] for s in SETTINGS],
                    sdp_ratio=tuple(s[3] for s in SETTINGS))
    swapped = {k: (v.flip(0) if isinstance(v, torch.Tensor) else list(v)[::-1]) for k, v in per_item.items()}
    net1 = _net(concurrency=1)
    ref = {}
    for name, st in (("a", per_item), ("b", swapped)):
        o = net1.infer(*args, **kw, **st, ragged=True)[0].cpu()
        chunks = [c.cpu() for c in net1.infer_stream(*args, **kw, **st, first_chunk_frames=8, max_chunk_frames=32)]
        ref[name] = (o, torch.cat(chunks, -1))
    pad = net1.infer(*args, **kw, **per_item)[0].cpu()
    assert torch.equal(ref["a"][1], pad)  # the stream is the padded call
    for b, s in enumerate(SETTINGS):
        one = dict(noise_scale=s[0], noise_scale_w=s[1], length_scale=s[2], sdp_ratio=s[3])
        assert torch.equal(net1.infer(*args, **kw, **one, ragged=True)[0].cpu()[b], ref["a"][0][b]), b
        assert torch.equal(net1.infer(*args, **kw, **one)[0].cpu()[b], pad[b]), b
    net2 = _net(concurrency=2)
    got, errors = {}, []

    def run(name, st):
        try:
            for _ in range(2):
                o = net2.infer(*args, **kw, **st, ragged=True)[0]
                chunks = list(net2.infer_stream(*args, **kw, **st, first_chunk_frames=8, max_chunk_frames=32))
                torch.cuda.current_stream().synchronize()
                got[name] = (o.cpu(), torch.cat(chunks, -1).cpu())
        except Exception as e:  # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=a) for a in (("a", per_item), ("b", swapped))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for name in ("a", "b"):
        assert torch.equal(got[name][0], ref[name][0]) and torch.equal(got[name][1], ref[name][1]), name
