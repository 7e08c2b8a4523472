"""Bounded streams end to end: with a cap on the chunk size, the FP16 Generator keeps only the rows later windows still read, and the
concatenated chunks stay bit-identical to infer() with the same noise.  Also the cap's rules, the workspace a reserve covers, the
fp32 / TF32 rejection and a pool serving two bounded streams.
Run on an H100: pytest -m gpu."""
import threading

import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Engine
from util import case_inputs, load_golden, model_for

pytestmark = pytest.mark.gpu

INFER_KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.625)  # bench.py's config-2 settings
CAPS = [1, 7, 32, 256]


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


def _synthetic(T, n_noise, seed):
    cfg, _ = model_for(True, 0)
    inp = synth.synthetic_inputs(cfg, [T], [0], seed=seed)
    nw, nz = synth.synthetic_noise(cfg, 1, T, n_noise, seed=seed)
    return inp, nw, nz, INFER_KW


def _config2():
    return _synthetic(256, 2048, 2)


def _long():
    return _synthetic(1024, 8192, 4)


def _tflow_b3():
    meta, _ = load_golden("tflow_b3")
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    return inp, nw, nz, kw


CASES = {"config2": _config2, "tflow_b3": _tflow_b3}


def _args(inp, nw, kw):
    return (inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw,
            kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"])


def _one_shot(eng, inp, nw, nz, kw, max_len=None):
    B, T = inp["x"].shape
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    o, _, _, _ = eng.infer_finish(B, T, F, nz, kw["noise_scale"], max_len, want_attn=False)
    torch.cuda.synchronize()
    return o.clone(), F


def _open(eng, inp, nw, nz, kw, max_len, cap):
    B, T = inp["x"].shape
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    o, _, _, _ = eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"], max_len, want_attn=False, max_chunk_frames=cap)
    return o, o.shape[-1] // eng.cfg.hop


def _stream(eng, inp, nw, nz, kw, max_len, cap, frontiers):
    """a bounded stream over the given frontiers: (chunks cloned as each became final, the final o)"""
    o, Fg = _open(eng, inp, nw, nz, kw, max_len, cap)
    hop = eng.cfg.hop
    chunks, prev = [], 0
    for f in frontiers(Fg):
        n = eng.stream_advance(f)
        assert n == min(f, Fg) * hop
        torch.cuda.current_stream().synchronize()
        chunks.append(o[:, :, prev * hop:n].clone())
        prev = min(f, Fg)
    assert prev == Fg
    return chunks, o


def _geometric(cap):
    def f(Fg):
        out, x, step = [], 0, 1
        while x < Fg:
            x = min(x + step, Fg)
            out.append(x)
            step = min(2 * step, cap)
        return out
    return f


def _fixed(cap):
    n = min(7, cap)
    return lambda Fg: list(range(n, Fg, n)) + [Fg]


def _random(cap):
    def f(Fg):
        rng = np.random.default_rng(Fg * 7919 + cap)
        out, x = [], 0
        while x < Fg:
            x = min(x + int(rng.integers(1, cap + 1)), Fg)
            out.append(x)
        return out
    return f


SCHEDULES = {"geometric": _geometric, "fixed_7": _fixed, "random": _random}


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("precision", ["fp16g", "fp16"])
def test_bounded_stream_bit_identical_to_infer(engines, precision, case, cap, schedule):
    if cap == 1 and schedule != "geometric":
        pytest.skip("with a cap of 1 every schedule advances one frame at a time")
    eng = engines(precision)
    inp, nw, nz, kw = CASES[case]()
    ref, F = _one_shot(eng, inp, nw, nz, kw)
    chunks, o = _stream(eng, inp, nw, nz, kw, None, cap, SCHEDULES[schedule](cap))
    torch.cuda.synchronize()
    got = torch.cat(chunks, -1)
    assert got.shape == ref.shape and torch.equal(got, ref), (precision, case, cap, schedule, F)
    assert torch.equal(o, ref)  # no later window or slide overwrote audio that an earlier chunk handed out


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("precision", ["fp16g", "fp16"])
def test_bounded_stream_max_len(engines, precision, cap):
    eng = engines(precision)
    inp, nw, nz, kw = _tflow_b3()
    ref, F = _one_shot(eng, inp, nw, nz, kw, 150)
    chunks, o = _stream(eng, inp, nw, nz, kw, 150, cap, _random(cap))
    torch.cuda.synchronize()
    assert torch.equal(torch.cat(chunks, -1), ref) and torch.equal(o, ref)


def test_bounded_stream_long_utterance_and_reserve():
    """~1023 and ~4000 frames: the one-shot run handles the long utterance, a cap-256 stream of it is bit-identical, and after
    reserve_stream(1, T, F_cap, 256) neither stream grows the workspace."""
    cfg, sd = model_for(True, 0)
    eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
    long_, short = _long(), _config2()
    ref_long, F_long = _one_shot(eng, *long_)
    ref_short, F_short = _one_shot(eng, *short)
    assert F_long > 3500 and F_short > 900
    del eng
    torch.cuda.synchronize()
    eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
    eng.reserve_stream(1, 1024, F_long, 256)
    g0, ws0 = eng.workspace_grows, eng.workspace_bytes
    for (inp, nw, nz, kw), ref in ((short, ref_short), (long_, ref_long)):
        chunks, o = _stream(eng, inp, nw, nz, kw, None, 256, _geometric(256))
        torch.cuda.synchronize()
        assert torch.equal(torch.cat(chunks, -1), ref)
    assert eng.workspace_grows == g0 and eng.workspace_bytes == ws0
    # the Generator storage of the bounded stream is the same for both lengths, and far below the unbounded stream's
    b = eng.stream_bytes(1, F_long, 256)
    assert b == eng.stream_bytes(1, F_short, 256) == eng.stream_bytes(1, 257, 256)
    assert b < eng.stream_bytes(1, F_long, None) // 4


def test_stream_bytes(engines):
    eng = engines("fp16")
    for cap in CAPS:
        vals = {eng.stream_bytes(2, Fg, cap) for Fg in (cap + 1, 1000, 4000, 20000)}
        assert len(vals) == 1, (cap, vals)
    for Fg in (1, 7, 300):
        full = eng.stream_bytes(1, Fg, None)
        assert eng.stream_bytes(1, Fg, 0) == full == eng.stream_bytes(1, Fg, Fg) == eng.stream_bytes(1, Fg, Fg + 100)
    assert eng.stream_bytes(1, 4000, 32) < eng.stream_bytes(1, 4000, 256) < eng.stream_bytes(1, 4000, None)
    with pytest.raises(ValueError):
        engines("fp32").stream_bytes(1, 100, 32)
    assert engines("fp32").stream_bytes(1, 100, None) == engines("fp32").stream_bytes(1, 100, 100)


def test_bounded_stream_workspace_below_unbounded():
    """The workspace a bounded stream ensures leaves out the one-shot Generator's part and the full-length tensors."""
    cfg, sd = model_for(True, 0)
    inp, nw, nz, kw = _config2()
    sizes = {}
    for cap in (None, 64):
        eng = Engine(cfg, sd, device="cuda:0", precision="fp16")
        _open(eng, inp, nw, nz, kw, None, cap)
        torch.cuda.synchronize()
        sizes[cap] = eng.workspace_bytes
        del eng
    assert sizes[64] < sizes[None] // 2, sizes


def test_over_cap_advance_raises_and_the_stream_continues(engines):
    eng = engines("fp16")
    inp, nw, nz, kw = _config2()
    ref, F = _one_shot(eng, inp, nw, nz, kw)
    o, Fg = _open(eng, inp, nw, nz, kw, None, 32)
    eng.stream_advance(32)
    with pytest.raises(ValueError):
        eng.stream_advance(32 + 33)
    with pytest.raises(ValueError):
        eng.stream_advance(Fg + 1000)
    f = 32
    while f < Fg:
        f = min(f + 32, Fg)
        eng.stream_advance(f)
    torch.cuda.synchronize()
    assert torch.equal(o, ref)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_fp32_tf32_reject_a_cap(engines, precision):
    eng = engines(precision)
    inp, nw, nz, kw = _tflow_b3()
    B, T = inp["x"].shape
    ref, F = _one_shot(eng, inp, nw, nz, kw)
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    with pytest.raises(ValueError):
        eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"], want_attn=False, max_chunk_frames=F - 1)
    for cap in (None, F):  # unbounded, or a cap no chunk can exceed: accepted
        chunks, o = _stream(eng, inp, nw, nz, kw, None, cap, _geometric(F))
        torch.cuda.synchronize()
        assert torch.equal(o, ref)
    with pytest.raises(ValueError):
        eng.reserve_stream(B, T, F, F - 1)


def _net(precision, concurrency=1):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, _ = model_for(True, 0)
    return SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                          [16, 16, 8, 2, 2], n_speakers=cfg.n_speakers, gin_channels=512, precision=precision, init_seed=0,
                          concurrency=concurrency).to("cuda"), cfg


def _net_args(cfg, lengths, seed):
    inp = synth.synthetic_inputs(cfg, lengths, list(range(len(lengths))), seed=seed)
    return [inp[k].cuda() for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")]


def test_infer_stream_cap_schedule_and_errors():
    net, cfg = _net("fp16")
    args = _net_args(cfg, [96, 61], 9)
    torch.manual_seed(123)
    ref = net.infer(*args, **INFER_KW)[0].clone()
    torch.manual_seed(123)
    chunks = [c.clone() for c in net.infer_stream(*args, **INFER_KW, first_chunk_frames=8, max_chunk_frames=24)]
    sizes = [c.shape[-1] // cfg.hop for c in chunks]
    assert sizes[:4] == [8, 16, 24, 24] and max(sizes) == 24
    assert torch.equal(torch.cat(chunks, -1), ref)
    with pytest.raises(ValueError):
        next(net.infer_stream(*args, **INFER_KW, first_chunk_frames=32, max_chunk_frames=16))
    net32, _ = _net("fp32")
    with pytest.raises(ValueError):
        next(net32.infer_stream(*args, **INFER_KW, max_chunk_frames=32))
    torch.manual_seed(123)
    ref32 = net32.infer(*args, **INFER_KW)[0].clone()
    torch.manual_seed(123)
    got = torch.cat([c.clone() for c in net32.infer_stream(*args, **INFER_KW, max_chunk_frames=100000)], -1)
    assert torch.equal(got, ref32)


def test_pool_serves_two_bounded_streams():
    net, cfg = _net("fp16", concurrency=2)
    reqs = [_net_args(cfg, [120], 11), _net_args(cfg, [90, 70], 12)]
    noise = []
    for i, a in enumerate(reqs):
        B, T = a[0].shape
        g = torch.Generator(device="cuda").manual_seed(100 + i)
        F_max = 8 * T
        noise.append((torch.randn(B, 2, T, device="cuda", generator=g), torch.randn(B, 192, F_max, device="cuda", generator=g)))
    serial = [net.infer(*a, **INFER_KW, noise_w=nw, noise_z=nz)[0].clone() for a, (nw, nz) in zip(reqs, noise)]
    out, errs = [None, None], []
    barrier = threading.Barrier(2)

    def work(i):
        try:
            nw, nz = noise[i]
            barrier.wait()
            out[i] = torch.cat([c.clone() for c in net.infer_stream(*reqs[i], **INFER_KW, noise_w=nw, noise_z=nz, first_chunk_frames=4,
                                                                      max_chunk_frames=16)], -1)
            torch.cuda.synchronize()
        except Exception as ex:  # surfaced below
            errs.append(ex)

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for i in range(2):
        assert torch.equal(out[i], serial[i]), i
