"""Speaker mixes (bv2_infer_begin_mix): every utterance of a batch is conditioned on its own weighted sum of emb_g rows.  The "g" tap
equals the np.float32 host mix bit for bit; a batch of mixes is bit-identical to the plain call on an engine whose emb_g holds the
host mixes as extra rows (every precision, padded, ragged, pcm16 and streams); a weight-1.0 single-entry mix is the plain call with
the same launches and workspace; the module, infer_batch and concurrent serving; each mixed utterance against the CPU oracle; and
the error paths.  Run on an H100: pytest -m gpu."""
import ctypes as C
import dataclasses
import threading

import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Engine
from bert_vits2_b200.infer_api import infer_batch
from bert_vits2_b200.models import speaker_mixes
from util import model_for, rms

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "fp16g", "fp16"]
FP16 = ("fp16", "fp16g")
LENGTHS = [64, 9, 30, 21, 14, 5]
# one mix per utterance: interpolations, a negative weight (extrapolation), a single speaker with weight != 1, unequal lengths
MIXES = [{0: 0.5, 1: 0.5}, {3: 0.7, 12: 0.6, 40: -0.3}, {849: 1.0}, {5: 0.25, 6: 0.25, 7: 0.25, 8: 0.25}, {2: 1.5, 4: -0.5},
         {10: 0.37}]
SETTINGS = [(0.667, 0.8, 1.0, 0.0), (0.3, 1.1, 0.7, 1.0), (0.9, 0.5, 1.3, 0.5), (0.0, 0.0, 1.05, 0.2), (1.2, 0.9, 0.85, 0.8),
            (0.5, 0.667, 1.6, 0.35)]
SCALARS = (0.667, 0.8, 1.0, 0.2)  # (noise_scale, noise_scale_w, length_scale, sdp_ratio) of the plain calls
CTOR = (112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512, [16, 16, 8, 2, 2])
NAMES = ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")
TOL_WAV = 1e-3  # waveform RMS against the oracle: the FP16 Generator's bar (test_item_settings_gpu.py)


def host_mix(E, ids, w):
    """the engine's arithmetic in np.float32: g = fl(w_0 E[i_0]), then g = fl(g + fl(w_k E[i_k])) in k order"""
    E, ids, w = np.asarray(E, np.float32), np.asarray(ids), np.asarray(w, np.float32)
    g = w[:, 0:1] * E[ids[:, 0]]
    for k in range(1, ids.shape[1]):
        g = g + w[:, k:k + 1] * E[ids[:, k]]
    assert g.dtype == np.float32
    return g


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


@pytest.fixture(scope="module")
def models():
    """(cfg, sd) of the base model, and of the extended model whose emb_g rows 850..855 hold the host mixes of MIXES"""
    cfg, sd = model_for(True, 0)
    ids, w = speaker_mixes(len(MIXES), MIXES)
    rows = torch.from_numpy(host_mix(sd["emb_g.weight"].numpy(), ids.numpy(), w.numpy()))
    sd_ext = dict(sd)
    sd_ext["emb_g.weight"] = torch.cat([sd["emb_g.weight"], rows])
    cfg_ext = dataclasses.replace(cfg, n_speakers=cfg.n_speakers + len(MIXES))
    return (cfg, sd), (cfg_ext, sd_ext)


@pytest.fixture(scope="module")
def engines(models):
    cache = {}

    def get(precision, extended=False):
        key = (precision, extended)
        if key not in cache:
            cfg, sd = models[int(extended)]
            cache[key] = Engine(cfg, sd, device="cuda:0", precision=precision)
        return cache[key]

    yield get
    cache.clear()


@pytest.fixture(scope="module")
def case():
    """B=6 batch of spread lengths, its noise, and teacher-forced durations of 3 to 6 frames per token (item 0: over 256 frames)"""
    cfg, _ = model_for(True, 0)
    B, T = len(LENGTHS), max(LENGTHS)
    inp = synth.synthetic_inputs(cfg, LENGTHS, [b % 3 for b in range(B)], seed=83)
    nw, nz = synth.synthetic_noise(cfg, B, T, 10 * T + 64, seed=83)  # room for free durations at length_scale 1.6
    w = torch.zeros(B, T)
    r = np.random.default_rng(83)
    for b, t in enumerate(LENGTHS):
        w[b, :t] = torch.as_tensor(r.integers(3, 7, size=t), dtype=torch.float32)
    return inp, nw, nz, w


EXT_SID = torch.arange(850, 850 + len(MIXES))


def _cols(i):
    return torch.tensor([s[i] for s in SETTINGS], dtype=torch.float32)


def _begin(eng, inp, nw, sid=None, mix=None, w=None, per_item=False):
    """the plain call (sid) or the mix call (mix: (ids, weights)), with SCALARS or SETTINGS per utterance -> (y_lengths, F, the
    noise_scale finish takes)"""
    args = [inp[k] for k in NAMES] + [nw]
    args[2] = sid
    if per_item:
        ylen, F = eng.infer_begin(*args, _cols(1), _cols(2), _cols(3), w_ceil_override=w, item_noise_scale=_cols(0), speaker_mix=mix)
        return ylen, F, 1.0
    ylen, F = eng.infer_begin(*args, *SCALARS[1:], w_ceil_override=w, speaker_mix=mix)
    return ylen, F, SCALARS[0]


def _taps(eng, B, T):
    return [eng.debug_read(n, (B, 1, T)).clone() for n in ("logw_sdp", "logw_dp", "w_ceil")]


def _finish(eng, B, T, F, nz, ns, mode):
    """finish in `mode` -> (o, [y_mask, z, z_p, m_p, logs_p]) on the CPU"""
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


def _mix_tensors():
    return speaker_mixes(len(MIXES), MIXES)


# ---------------------------------------------------------------- 1. the arithmetic, bitwise against np.float32
@pytest.mark.parametrize("precision", PRECISIONS)
def test_g_tap_equals_host_mix(engines, models, precision, case):
    eng = engines(precision)
    (cfg, sd), _ = models
    E = sd["emb_g.weight"].numpy()
    inp, nw, _, _ = case
    B, G = inp["x"].shape[0], cfg.gin_channels
    r = np.random.default_rng(5)
    dense_w = r.standard_normal((B, cfg.n_speakers)).astype(np.float32) / np.float32(cfg.n_speakers)
    cases = {
        "K=1": (np.arange(B)[:, None] * 7, r.uniform(-2, 2, (B, 1))),
        "K=3, repeated id, negative weight": (np.array([[4, 9, 4]] * B) + np.arange(B)[:, None], np.array([[0.6, -0.45, 0.85]] * B)),
        "padded, unequal lengths": tuple(t.numpy() for t in _mix_tensors()),
        "dense K=850 (CharaMix)": (np.stack([r.permutation(cfg.n_speakers) for _ in range(B)]), dense_w),
    }
    for name, (ids, w) in cases.items():
        ids, w = np.asarray(ids, np.int64), np.asarray(w, np.float32)
        _begin(eng, inp, nw, mix=(torch.from_numpy(ids), torch.from_numpy(w)))
        g = eng.debug_read("g", (B, G, 1)).numpy()[:, :, 0]
        want = host_mix(E, ids, w)
        assert np.array_equal(_bits(g), _bits(want)), (precision, name, int((_bits(g) != _bits(want)).sum()))
    # the bitwise check tells summation orders apart: the dense mix summed in float64 and rounded once has other bits
    assert not np.array_equal(_bits(want), _bits((w.astype(np.float64)[:, :, None] * E[ids].astype(np.float64)).sum(1).astype(np.float32)))
    # the plain call's tap is the row of sid
    _begin(eng, inp, nw, sid=inp["sid"])
    assert np.array_equal(eng.debug_read("g", (B, G, 1)).numpy()[:, :, 0], E[inp["sid"].numpy()])


# ---------------------------------------------------------------- 2. contract (b): the extended table
def _compare(a, b, what):
    (o, rest), (o2, rest2) = a, b
    assert torch.equal(o, o2), (what, "o")
    for name, x, y in zip(("y_mask", "z", "z_p", "m_p", "logs_p"), rest, rest2):
        assert torch.equal(x, y), (what, name)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mix_equals_extended_table(engines, precision, case):
    eng, ext = engines(precision), engines(precision, extended=True)
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    mix = _mix_tensors()
    # durations free: the durations themselves, then a padded call
    for per_item in (False, True):
        ylen, F, ns = _begin(eng, inp, nw, mix=mix, per_item=per_item)
        taps = _taps(eng, B, T)
        got = _finish(eng, B, T, F, nz, ns, ("padded", None))
        ylen2, F2, ns2 = _begin(ext, inp, nw, sid=EXT_SID, per_item=per_item)
        assert ylen.tolist() == ylen2.tolist() and F == F2, (precision, per_item)
        for name, x, y in zip(("logw_sdp", "logw_dp", "w_ceil"), taps, _taps(ext, B, T)):
            assert torch.equal(x, y), (precision, per_item, name)
        _compare(got, _finish(ext, B, T, F2, nz, ns2, ("padded", None)), (precision, "free durations", per_item))
    assert len(set(ylen.tolist())) > 1
    # teacher-forced: every finish mode, with scalar settings and with per-utterance settings
    for per_item in (False, True):
        for mode in _modes(precision):
            _, F, ns = _begin(eng, inp, nw, mix=mix, w=w, per_item=per_item)
            got = _finish(eng, B, T, F, nz, ns, mode)
            _, F2, ns2 = _begin(ext, inp, nw, sid=EXT_SID, w=w, per_item=per_item)
            _compare(got, _finish(ext, B, T, F2, nz, ns2, mode), (precision, mode, per_item))
    # the mix reaches the output: item 0 under item 1's mix differs
    outs = []
    for m in (mix, speaker_mixes(B, [MIXES[1]] + MIXES[1:])):
        _, F, ns = _begin(eng, inp, nw, mix=m, w=w)
        outs.append(_finish(eng, B, T, F, nz, ns, ("padded", None))[0])
    assert not torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1:], outs[1][1:])


# ---------------------------------------------------------------- 3. contract (a): weight-1.0 single-entry mixes
@pytest.mark.parametrize("precision", PRECISIONS)
def test_unit_mix_equals_plain_call(engines, precision, case):
    """against bv2_infer_begin_items with those sids, each on a sibling with a fresh workspace: same bits, same launches, same
    workspace"""
    base = engines(precision)
    inp, nw, nz, _ = case
    B, T = inp["x"].shape
    mix = (inp["sid"].reshape(B, 1).clone(), torch.ones(B, 1))
    res = []
    for kw in (dict(sid=inp["sid"]), dict(mix=mix)):
        eng = base.sibling()
        l0, w0 = eng.launch_count, eng.workspace_bytes
        ylen, F, ns = _begin(eng, inp, nw, per_item=True, **kw)
        taps = _taps(eng, B, T)
        g = eng.debug_read("g", (B, eng.cfg.gin_channels, 1))
        out = _finish(eng, B, T, F, nz, ns, ("padded", None))
        res.append((ylen.tolist(), taps, g, out, eng.launch_count - l0, eng.workspace_bytes - w0))
    (ylen, taps, g, out, launches, ws), (ylen2, taps2, g2, out2, launches2, ws2) = res
    assert ylen == ylen2 and launches == launches2 and ws == ws2, (precision, launches, launches2, ws, ws2)
    assert torch.equal(g, g2) and all(torch.equal(a, b) for a, b in zip(taps, taps2)), precision
    _compare(out, out2, precision)


# ---------------------------------------------------------------- 4. the module, infer_batch and concurrency
def _nets(models, concurrency=1):
    from bert_vits2_b200.models import SynthesizerTrn
    (cfg, sd), (cfg_ext, sd_ext) = models
    out = []
    for c, s in ((cfg, sd), (cfg_ext, sd_ext)):
        net = SynthesizerTrn(*CTOR, n_speakers=c.n_speakers, gin_channels=512, precision="fp16", init_seed=None, concurrency=concurrency)
        net.load_state_dict(s)
        out.append(net.to("cuda"))
    return out


def test_module_mix_equals_extended_table(models, case):
    """infer (padded, ragged), infer_stream (ragged, bounded) and infer_batch with speaker_mix reproduce the extended module's plain
    calls; with concurrency=2, two threads with different mixes get exactly their serial results"""
    inp, nw, nz, w = case
    net, ext = _nets(models)
    args = [inp[k].cuda() for k in NAMES]
    kw = dict(noise_w=nw.cuda(), noise_z=nz.cuda(), noise_scale=SCALARS[0], noise_scale_w=SCALARS[1], length_scale=SCALARS[2],
              sdp_ratio=SCALARS[3])
    plain = lambda: [*args[:2], EXT_SID.cuda(), *args[3:]]  # noqa: E731
    mixed = lambda: [*args[:2], None, *args[3:]]  # noqa: E731
    for extra in (dict(), dict(ragged=True), dict(ragged=True, w_ceil_override=w.cuda()), dict(pcm16=True)):
        o = net.infer(*mixed(), **kw, **extra, speaker_mix=MIXES)[0].cpu()
        assert torch.equal(o, ext.infer(*plain(), **kw, **extra)[0].cpu()), extra
        assert net.last_y_lengths.tolist() == ext.last_y_lengths.tolist()
    for extra in (dict(ragged=True), dict(max_chunk_frames=32), dict(ragged=True, max_chunk_frames=32)):
        a = torch.cat([c.cpu() for c in net.infer_stream(*mixed(), **kw, **extra, first_chunk_frames=8, speaker_mix=MIXES)], -1)
        b = torch.cat([c.cpu() for c in ext.infer_stream(*plain(), **kw, **extra, first_chunk_frames=8)], -1)
        assert torch.equal(a, b), extra
    # per-utterance settings in the same call
    per = dict(noise_scale=_cols(0), noise_scale_w=_cols(1), length_scale=_cols(2), sdp_ratio=_cols(3))
    kw2 = dict(noise_w=nw.cuda(), noise_z=nz.cuda(), **per)
    assert torch.equal(net.infer(*mixed(), **kw2, speaker_mix=MIXES)[0].cpu(), ext.infer(*plain(), **kw2)[0].cpu())
    # infer_batch: one mix per item in item order, buckets by length; the noise is drawn inside, so both runs seed it alike
    items = [(inp["bert"][b, :, :t], inp["ja_bert"][b, :, :t], inp["en_bert"][b, :, :t], inp["x"][b, :t], inp["tone"][b, :t],
              inp["language"][b, :t]) for b, t in enumerate(LENGTHS)]
    torch.manual_seed(3)
    got = infer_batch(net, items, batch_size=4, speaker_mix=MIXES, ragged=True)
    torch.manual_seed(3)
    want = infer_batch(ext, items, sid=EXT_SID.tolist(), batch_size=4, ragged=True)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    # concurrency=2 against the serial results
    ref = {}
    mixes = {"a": MIXES, "b": MIXES[::-1]}
    for name, m in mixes.items():
        o = net.infer(*mixed(), **kw, speaker_mix=m, ragged=True)[0].cpu()
        s = torch.cat([c.cpu() for c in net.infer_stream(*mixed(), **kw, speaker_mix=m, first_chunk_frames=8, max_chunk_frames=32)], -1)
        ref[name] = (o, s)
    assert not torch.equal(ref["a"][0], ref["b"][0])
    net2, _ = _nets(models, concurrency=2)
    got, errors = {}, []

    def run(name):
        try:
            for _ in range(2):
                o = net2.infer(*mixed(), **kw, speaker_mix=mixes[name], ragged=True)[0]
                chunks = list(net2.infer_stream(*mixed(), **kw, speaker_mix=mixes[name], first_chunk_frames=8, max_chunk_frames=32))
                torch.cuda.current_stream().synchronize()
                got[name] = (o.cpu(), torch.cat(chunks, -1).cpu())
        except Exception as e:  # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(n,)) for n in mixes]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for name in mixes:
        assert torch.equal(got[name][0], ref[name][0]) and torch.equal(got[name][1], ref[name][1]), name


# ---------------------------------------------------------------- 5. each mixed utterance against the CPU oracle
@pytest.fixture(scope="module")
def oracle_alone(models, case):
    """the CPU oracle on the extended state dict, each utterance alone with sid = its mix's row"""
    from oracle import vits2_oracle as O
    _, (cfg_ext, sd_ext) = models
    inp, nw, nz, _ = case
    out = []
    for b, t in enumerate(LENGTHS):
        one = {k: (v[b:b + 1, ..., :t] if v.dim() >= 2 else v[b:b + 1]) for k, v in inp.items()}
        one["x_lengths"], one["sid"] = torch.tensor([t]), EXT_SID[b:b + 1]
        out.append(O.infer(sd_ext, cfg_ext, **one, noise_w=nw[b:b + 1, :, :t], noise_z=nz[b:b + 1], return_stages=True,
                           noise_scale=SCALARS[0], noise_scale_w=SCALARS[1], length_scale=SCALARS[2], sdp_ratio=SCALARS[3]))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_utterances_vs_oracle(engines, models, precision, case, oracle_alone):
    (cfg, _), _ = models
    eng = engines(precision)
    inp, nw, nz, _ = case
    for b, (t, st) in enumerate(zip(LENGTHS, oracle_alone)):
        one = {k: (v[b:b + 1, ..., :t] if v.dim() >= 2 else v[b:b + 1]) for k, v in inp.items()}
        one["x_lengths"] = torch.tensor([t])
        w_ceil = torch.as_tensor(st["w_ceil"]).reshape(1, -1)[:, :t]
        ylen, F, ns = _begin(eng, one, nw[b:b + 1, :, :t], mix=speaker_mixes(1, MIXES[b]), w=w_ceil)
        assert ylen.tolist() == [int(st["y_lengths"][0])], (precision, b)
        o, _ = _finish(eng, 1, t, F, nz[b:b + 1], ns, ("padded", None))
        ref = torch.as_tensor(st["o"]).reshape(-1)
        e = rms(o.reshape(-1), ref)
        print(f"[{precision}] item {b} {MIXES[b]}: frames {F}, waveform RMS vs oracle {e:.2e}")
        assert o.numel() == ref.numel() and e < TOL_WAV


# ---------------------------------------------------------------- 6. errors
def test_errors_then_next_call_unchanged(engines, models, case):
    (cfg, sd), _ = models
    eng = engines("fp16")
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    mix = _mix_tensors()

    def good_call(e):
        ylen, F, ns = _begin(e, inp, nw, mix=mix, w=w)
        return ylen.tolist(), _taps(e, B, T), _finish(e, B, T, F, nz, ns, ("ragged", None))

    fresh = good_call(Engine(cfg, sd, device="cuda:0", precision="fp16"))

    def check_next():
        ylen, taps, out = good_call(eng)
        assert ylen == fresh[0] and all(torch.equal(a, b) for a, b in zip(taps, fresh[1]))
        _compare(out, fresh[2], "after an error")

    ids, wts = mix

    def with_entry(b, k, sid=None, weight=None):
        i, x = ids.clone(), wts.clone()
        if sid is not None:
            i[b, k] = sid
        if weight is not None:
            x[b, k] = weight
        return i, x

    for bad in (with_entry(2, 0, sid=-1), with_entry(5, 3, sid=850), with_entry(0, 1, sid=-1, weight=float("nan"))):
        with pytest.raises(IndexError, match="speaker id"):
            _begin(eng, inp, nw, mix=bad, w=w)
        check_next()
    for weight in (float("nan"), float("inf"), float("-inf")):
        with pytest.raises(ValueError) as ei:
            _begin(eng, inp, nw, mix=with_entry(3, 2, weight=weight), w=w)
        assert not isinstance(ei.value, IndexError) and "index out of range" not in str(ei.value)
        check_next()
    # at the C ABI: K = 0, a NULL array, B*K over INT32_MAX
    dev = [eng._i64(inp[k]) for k in ("x", "x_lengths", "tone", "language")] + [eng._f32(inp[k]) for k in NAMES[5:]] + [eng._f32(nw)]
    p = [C.c_void_p(t.data_ptr()) for t in dev]
    ones = torch.ones(B, device=eng.device)
    ylen, fmax = (C.c_int64 * B)(), C.c_int32(0)
    d_ids, d_w = ids.cuda(), wts.cuda()
    for K, pi, pw in ((0, d_ids, d_w), (-1, d_ids, d_w), (4, None, d_w), (4, d_ids, None), (2 ** 31 // B + 1, d_ids, d_w)):
        rc = eng.lib.bv2_infer_begin_mix(eng._h, B, T, p[0], p[1], K, None if pi is None else C.c_void_p(pi.data_ptr()),
                                         None if pw is None else C.c_void_p(pw.data_ptr()), *p[2:], *[C.c_void_p(ones.data_ptr())] * 4,
                                         None, eng._stream(), ylen, C.byref(fmax))
        assert rc == -1, (K, rc)
        check_next()
