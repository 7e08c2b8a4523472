"""Ragged streams (precision fp16 / fp16g): a batched Generator stream in which every utterance runs at its own length.  The chunks of
each utterance, joined, are bit-identical to infer(..., ragged=True) with the same noise and durations, and 0 past its end, for every
chunk schedule and cap, including the bounded streams whose slides carry the zeros after an item's end.  Also a B=1 agreement, one
streamed ragged k_g2_conv on resident storage through a kernel harness, and the error and workspace paths.
Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Engine
from util import model_for

pytestmark = pytest.mark.gpu

FP16 = ["fp16", "fp16g"]
KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)


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


def _batch(frames, seed):
    """inputs of a batch whose item b has exactly frames[b] frames: min(frames[b], 12) tokens, durations teacher-forced
    (w_ceil_override) so that they add up to frames[b]"""
    cfg, _ = model_for(True, 0)
    toks = [max(1, min(int(L), 12)) for L in frames]
    B, T = len(frames), max(toks)
    inp = synth.synthetic_inputs(cfg, toks, [b % 3 for b in range(B)], seed=seed)
    nw, nz = synth.synthetic_noise(cfg, B, T, max(frames) + 8, seed=seed)
    w = torch.zeros(B, T)
    for b, (L, t) in enumerate(zip(frames, toks)):
        q, r = divmod(int(L), t)
        w[b, :t] = q
        w[b, :r] += 1
    return inp, nw, nz, w


def _begin(eng, inp, nw, w):
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, KW["noise_scale_w"], KW["length_scale"], KW["sdp_ratio"], w_ceil_override=w)
    return ylen, F


def _one_shot(eng, case, max_len=None):
    """infer(..., ragged=True): (o, y_mask, (z, z_p, m_p, logs_p), y_lengths) on the CPU"""
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    ylen, F = _begin(eng, inp, nw, w)
    o, _, ym, aux = eng.infer_finish(B, T, F, nz, KW["noise_scale"], max_len, want_attn=False, ragged=True)
    torch.cuda.synchronize()
    return o.cpu(), ym.cpu(), [a.cpu() for a in aux], ylen


def _stream(eng, case, cap, frontiers, max_len=None, ragged=True):
    """a stream over frontiers(Fg): (chunks copied as each became final, final o, y_mask, aux, kernel launches of the advances)"""
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    _, F = _begin(eng, inp, nw, w)
    o, _, ym, aux = eng.infer_finish_stream(B, T, F, nz, KW["noise_scale"], max_len, want_attn=False, max_chunk_frames=cap, ragged=ragged)
    hop, Fg = eng.cfg.hop, o.shape[-1] // eng.cfg.hop
    chunks, prev, l0 = [], 0, eng.launch_count
    for f in frontiers(Fg):
        n = eng.stream_advance(f)
        assert n == min(f, Fg) * hop
        torch.cuda.current_stream().synchronize()
        chunks.append(o[:, :, prev * hop:n].cpu())
        prev = min(f, Fg)
    assert prev == Fg
    return chunks, o.cpu(), ym.cpu(), [a.cpu() for a in aux], eng.launch_count - l0


# chunk schedules of tests/test_stream_bounded_gpu.py; cap None: no cap
def _geometric(cap):
    def f(Fg):
        out, x, step = [], 0, 1
        while x < Fg:
            x = min(x + step, Fg)
            out.append(x)
            step = 2 * step if cap is None else min(2 * step, cap)
        return out
    return f


def _fixed(cap):
    n = 7 if cap is None else min(7, cap)
    return lambda Fg: list(range(n, Fg, n)) + [Fg]


def _random(cap):
    def f(Fg):
        c = 96 if cap is None else cap
        rng = np.random.default_rng(Fg * 7919 + c)
        out, x = [], 0
        while x < Fg:
            x = min(x + int(rng.integers(1, c + 1)), Fg)
            out.append(x)
        return out
    return f


SCHEDULES = {"geometric": _geometric, "fixed_7": _fixed, "random": _random}
CAPS = [None, 7, 32, 256]
F_EDGES = 200


def _lengths(kind, frontiers):
    """edges: 1, the longest item, and lengths on three chunk boundaries of the schedule and one frame either side; random32: 32
    random lengths"""
    if kind == "random32":
        return [int(v) for v in np.random.default_rng(5).integers(1, 301, size=32)]
    fs = frontiers(F_EDGES)  # ends with F_EDGES itself
    picks = sorted({fs[0], fs[len(fs) // 2], fs[max(0, len(fs) - 2)]})
    out = [1, F_EDGES] + [L for f in picks for L in (f - 1, f, f + 1) if 1 <= L <= F_EDGES]
    return list(dict.fromkeys(out))


def _check(eng, case, ref, got, what):
    o_ref, ym_ref, aux_ref, ylen = ref
    chunks, o, ym, aux, _ = got
    hop = eng.cfg.hop
    joined = torch.cat(chunks, -1)
    assert joined.shape == o_ref.shape, what
    for b, L in enumerate(ylen.tolist()):
        n = min(L, o_ref.shape[-1] // hop) * hop
        assert torch.equal(joined[b, :, :n], o_ref[b, :, :n]), f"{what}: item {b} (L={L}) differs from infer(ragged=True)"
        assert (joined[b, :, n:] == 0).all(), f"{what}: item {b} (L={L}) has non-zero samples past its end"
    assert torch.equal(joined, o_ref) and torch.equal(o, o_ref), what  # and nothing rewrote a chunk once it was handed out
    assert torch.equal(ym, ym_ref) and all(torch.equal(a, r) for a, r in zip(aux, aux_ref)), what  # y_mask, z, z_p, m_p, logs_p


# ---------------------------------------------------------------- 1. end to end, bitwise against infer(ragged=True)
@pytest.mark.parametrize("kind", ["edges", "random32"])
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("cap", CAPS, ids=[f"cap{c}" for c in CAPS])
@pytest.mark.parametrize("precision", FP16)
def test_ragged_stream_bit_identical_to_ragged_infer(engines, precision, cap, schedule, kind):
    eng = engines(precision)
    frontiers = SCHEDULES[schedule](cap)
    lengths = _lengths(kind, frontiers)
    case = _batch(lengths, seed=len(lengths) + (cap or 0))
    ref = _one_shot(eng, case)
    assert ref[3].tolist() == lengths
    _check(eng, case, ref, _stream(eng, case, cap, frontiers), (precision, cap, schedule, kind))


@pytest.mark.parametrize("schedule", ["fixed_7", "random"])
@pytest.mark.parametrize("precision", FP16)
def test_ragged_stream_cap7_every_length_to_64(engines, precision, schedule):
    """every L_b in 1..64 beside a 300-frame item, cap 7: items end just before (and just after) slides at every phase of the chunk
    schedule, while the windows of their consumers are still behind"""
    eng = engines(precision)
    lengths = list(range(1, 65)) + [300]
    case = _batch(lengths, seed=65)
    ref = _one_shot(eng, case)
    assert ref[3].tolist() == lengths
    _check(eng, case, ref, _stream(eng, case, 7, SCHEDULES[schedule](7)), (precision, schedule))


@pytest.mark.parametrize("cap", [None, 32])
def test_ragged_stream_max_len(engines, cap):
    """max_len below F: items are cut at min(y_lengths[b], max_len)"""
    eng = engines("fp16")
    lengths = [1, 40, 149, 150, 151, 230, 97]
    case = _batch(lengths, seed=17)
    ref = _one_shot(eng, case, max_len=150)
    assert ref[0].shape[-1] == 150 * eng.cfg.hop
    _check(eng, case, ref, _stream(eng, case, cap, _random(cap), max_len=150), ("max_len", cap))


# ---------------------------------------------------------------- 2. B=1 agreement
@pytest.mark.parametrize("precision", FP16)
def test_ragged_stream_items_equal_b1_generator(engines, precision):
    eng = engines(precision)
    cfg, sd = model_for(True, 0)
    lengths = [int(v) for v in np.random.default_rng(9).integers(1, 260, size=12)] + [1, 256]
    case = _batch(lengths, seed=9)
    chunks, o, _, (z, _, _, _), _ = _stream(eng, case, 32, _random(32))
    g = sd["emb_g.weight"][case[0]["sid"]].unsqueeze(-1)
    hop = cfg.hop
    for b, L in enumerate(lengths):
        ref = eng.generator(z[b:b + 1, :, :L].contiguous(), g[b:b + 1]).cpu()
        assert torch.equal(o[b, :, :L * hop], ref[0]), f"item {b} (L={L}) differs from its B=1 Generator run"
        assert (o[b, :, L * hop:] == 0).all()


# ---------------------------------------------------------------- 3. launches, workspace, errors
def test_ragged_stream_launches_and_workspace_are_the_padded_streams():
    cfg, sd = model_for(True, 0)
    eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
    lengths = [300, 1, 77, 140, 8, 299]
    case = _batch(lengths, seed=3)
    B, T = case[0]["x"].shape
    eng.reserve_stream(B, T, max(lengths), 32)
    g0, ws0 = eng.workspace_grows, eng.workspace_bytes
    for cap in (32, None):
        pad = _stream(eng, case, cap, _random(32), ragged=False)
        rag = _stream(eng, case, cap, _random(32))
        assert rag[4] == pad[4], (cap, rag[4], pad[4])
        if cap is not None:
            assert eng.workspace_grows == g0 and eng.workspace_bytes == ws0
    ref = _one_shot(eng, case)
    _check(eng, case, ref, rag, "after reserve_stream")


def test_ragged_stream_over_cap_advance_raises_and_continues(engines):
    eng = engines("fp16")
    lengths = [5, 120, 64]
    case = _batch(lengths, seed=4)
    ref = _one_shot(eng, case)
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    _, F = _begin(eng, inp, nw, w)
    o, _, _, _ = eng.infer_finish_stream(B, T, F, nz, KW["noise_scale"], want_attn=False, max_chunk_frames=32, ragged=True)
    eng.stream_advance(32)
    with pytest.raises(ValueError):
        eng.stream_advance(32 + 33)
    f = 32
    while f < F:
        f = min(f + 32, F)
        eng.stream_advance(f)
    torch.cuda.synchronize()
    assert torch.equal(o.cpu(), ref[0])


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_ragged_stream_rejected_by_fp32_and_tf32(engines, precision):
    from bert_vits2_b200.models import SynthesizerTrn
    eng = engines(precision)
    case = _batch([20, 9], seed=3)
    inp, nw, nz, w = case
    B, T = inp["x"].shape
    _, F = _begin(eng, inp, nw, w)
    with pytest.raises(ValueError):
        eng.infer_finish_stream(B, T, F, nz, KW["noise_scale"], want_attn=False, ragged=True)
    # the C entry point itself: BV2_ERR_ARG, capped or not
    _, F = _begin(eng, inp, nw, w)
    nzd = nz.cuda()
    o = torch.empty(B, 1, F * eng.cfg.hop, device="cuda")
    for cap in (0, 4):
        rc = eng.lib.bv2_infer_finish_stream_ragged(eng._h, C.c_void_p(nzd.data_ptr()), nzd.shape[2], 0.6, -1, cap, C.c_void_p(o.data_ptr()),
                                                    None, None, None, None, None, None, eng._stream())
        assert rc == -1, (precision, cap, rc)
    # the engine serves the next call: a padded stream
    chunks, o2, _, _, _ = _stream(eng, case, None, _geometric(None), ragged=False)
    assert torch.isfinite(o2).all()
    cfg, _ = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=cfg.n_speakers, gin_channels=512, precision=precision, init_seed=0).to("cuda")
    args = [inp[k].cuda() for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")]
    with pytest.raises(ValueError):
        next(net.infer_stream(*args, ragged=True))


def test_module_infer_stream_ragged():
    """SynthesizerTrn.infer_stream(ragged=True): the padded stream's chunk schedule, and each utterance bit-identical to
    infer(ragged=True), final once a chunk ends at or past its end"""
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, _ = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=cfg.n_speakers, gin_channels=512, precision="fp16", init_seed=0).to("cuda")
    inp = synth.synthetic_inputs(cfg, [96, 61, 7], [0, 1, 2], seed=9)
    args = [inp[k].cuda() for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")]
    torch.manual_seed(123)
    ref = net.infer(*args, **KW, ragged=True)[0].cpu()
    ylen = net.last_y_lengths
    torch.manual_seed(123)
    pad_sizes = [c.shape[-1] for c in net.infer_stream(*args, **KW, first_chunk_frames=8, max_chunk_frames=24)]
    torch.manual_seed(123)
    hop, done, chunks = cfg.hop, 0, []
    for c in net.infer_stream(*args, **KW, first_chunk_frames=8, max_chunk_frames=24, ragged=True):
        chunks.append(c.cpu())
        done += c.shape[-1]
        for b, L in enumerate(ylen.tolist()):
            if done >= L * hop:  # utterance b is complete: final, and never rewritten by a later chunk
                assert torch.equal(torch.cat(chunks, -1)[b, :, :L * hop], ref[b, :, :L * hop])
    assert [c.shape[-1] for c in chunks] == pad_sizes
    assert torch.equal(torch.cat(chunks, -1), ref)


# ---------------------------------------------------------------- 4. kernel level: one streamed ragged k_g2_conv on resident storage
CANARY = np.uint16(0x7E5A)  # a NaN no kernel produces
# (name, Cin, Cout, K, u, dil, mode); item lengths LENS frames at LENS_SCALE M-axis rows per frame of T_IN rows
KSHAPES = [
    ("plain_k3", 256, 256, 3, 0, 1, "plain"),
    ("dilated_res_k7_d3", 128, 128, 7, 0, 3, "residual"),
    ("convT_ups0", 512, 256, 16, 8, 1, "plain"),
    ("convT_ups4", 32, 16, 2, 2, 1, "plain"),
    ("acc_k11", 64, 64, 11, 0, 1, "accumulate"),
]
T_IN, LENS, LENS_SCALE = 300, [1, 30, 64, 100, 150], 2
KWINDOWS = [(37, 201), (128, 256), (150, 300), (290, 300), (0, 140)]


def _ups_half(K, u):
    p, taps = (K - u) // 2, K // u
    offs = [(r + p) // u - m for r in range(u) for m in range(taps)]
    return max(-min(offs), max(offs))


@pytest.mark.parametrize("shape", KSHAPES, ids=[s[0] for s in KSHAPES])
def test_g2_conv_ragged_stream_kernel(shape):
    import zlib

    from kernel_harness import g2_args, g2_pads, to_h8
    from ragged_stream_harness import g2_conv_ragged_stream
    from stream_harness import g2_conv_window
    name, Cin, Cout, K, u, dil, mode = shape
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    B, T, U = len(LENS), T_IN, u or 1
    To = T * U
    pl, pr = g2_pads()
    pad = _ups_half(K, u) if u else (K - 1) // 2 * dil
    lim = [min(T, L * LENS_SCALE) for L in LENS]
    w = (rng.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    xf = rng.standard_normal((B, Cin, T)).astype(np.float32)
    for b, m in enumerate(lim):
        xf[b, :, m:] = 0.0  # what a ragged stream's producer stored after the item's end
    x = to_h8(xf)
    res = to_h8(rng.standard_normal((B, Cout, To)).astype(np.float32)) if mode == "residual" else None
    y0 = to_h8(rng.standard_normal((B, Cout, To)).astype(np.float32)) if mode == "accumulate" else np.zeros((B, Cout // 8, pl + To + pr, 8), np.float16)
    y0v = y0.view(np.uint16)
    for b, m in enumerate(lim):  # every row the launch may not read: canary
        y0v[b, :, pl + (m * U if mode == "accumulate" else -pl):, :] = CANARY
    kw = dict(B=B, T=T, Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, num_sms=132, w=w.ctypes.data, bias=bias.ctypes.data)
    if mode == "residual":
        kw.update(residual=1)
    if mode == "accumulate":
        kw.update(accumulate=1, out_scale=1.0 / 3)
    for a, e in KWINDOWS:
        x_base = max(0, a - pad)
        x_rows = min(e + pad, T) - x_base
        y_base, y_rows = a * U, (e - a) * U
        # the padded launch over the same window on whole tensors: item b's rows below its end
        yf, _, gf, ef = g2_conv_window(g2_args(**kw, x=x.ctypes.data, res=None if res is None else res.ctypes.data), a * U, e * U, y0)
        assert gf and ef == 0
        xs = np.array(x[:, :, x_base:x_base + pl + x_rows + pr], copy=True)
        if x_base > 0:
            xs[:, :, :pl] = np.nan
        if x_base + x_rows < T:
            xs[:, :, pl + x_rows:] = np.nan
        keep, rkw, res_base, res_rows = [xs], {}, 0, 0
        if res is not None:
            res_base, res_rows = max(0, a * U - 5), e * U - max(0, a * U - 5)
            rs = np.array(res[:, :, res_base:res_base + pl + res_rows + pr], copy=True)
            keep.append(rs)
            rkw = dict(res=rs.ctypes.data)
        ys0 = np.array(y0[:, :, y_base:y_base + pl + y_rows + pr], copy=True)
        ys, g, err = g2_conv_ragged_stream(g2_args(**kw, x=xs.ctypes.data, **rkw), LENS, LENS_SCALE, a * U, e * U, x_base, x_rows, y_base, y_rows,
                                           res_base, res_rows, ys0)
        assert g, (name, a, e, "guard region overwritten")
        assert err == 0, (name, a, e, "error flag")
        yv, rv, v0 = ys.view(np.uint16), yf.view(np.uint16), ys0.view(np.uint16)
        for b, m in enumerate(lim):
            mo = m * U
            # storage row i holds logical row y_base - pl + i
            rows = np.arange(ys.shape[2]) + y_base - pl
            live = (rows >= a * U) & (rows < min(e * U, mo))
            zero = (rows >= max(a * U, mo)) & (rows < e * U)
            if e == T:
                zero |= rows >= To  # the tensor's own zero halo, written by the window that reaches its end
            if a == 0:
                zero |= rows < 0
            assert np.array_equal(yv[b][:, live], rv[b][:, rows[live] + pl]), (name, a, e, b, "rows below the item's end")
            assert (yv[b][:, zero] == 0).all(), (name, a, e, b, "rows at or past the item's end inside the window are not zero")
            rest = ~(live | zero)
            assert np.array_equal(yv[b][:, rest], v0[b][:, rest]), (name, a, e, b, "wrote outside its window")
