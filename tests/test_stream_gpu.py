"""Streaming synthesis end to end: the concatenated chunks are bit-identical to infer() with the same noise, every chunk is final
when it is handed out, and the stream's state rules hold.  Run on an H100: pytest -m gpu."""
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Bv2Error, Engine
from util import case_inputs, load_golden, model_for

pytestmark = pytest.mark.gpu

STREAM_PRECISIONS = ["fp32", "tf32", "fp16g", "fp16"]
INFER_KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.625)  # bench.py's config-2 settings


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


def _config2():
    cfg, _ = model_for(True, 0)
    inp = synth.synthetic_inputs(cfg, [256], [0], seed=2)
    nw, nz = synth.synthetic_noise(cfg, 1, 256, 2048, seed=2)
    return inp, nw, nz, INFER_KW


def _tflow_b3():
    meta, _ = load_golden("tflow_b3")
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    return inp, nw, nz, kw


CASES = {"config2": _config2, "tflow_b3": _tflow_b3}


def _args(inp, nw, kw):
    return (inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw,
            kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"])


def _one_shot(eng, inp, nw, nz, kw, max_len):
    B, T = inp["x"].shape
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    o, _, _, _ = eng.infer_finish(B, T, F, nz, kw["noise_scale"], max_len, want_attn=False)
    torch.cuda.synchronize()
    return o.clone(), F


def _stream(eng, inp, nw, nz, kw, max_len, frontiers):
    """streams with the given frontiers; returns (chunks cloned as each became final, the final o, launches of the Generator)"""
    B, T = inp["x"].shape
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    o, _, _, _ = eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"], max_len, want_attn=False)
    hop, Fg = eng.cfg.hop, o.shape[-1] // eng.cfg.hop
    chunks, prev = [], 0
    l0 = eng.launch_count
    for f in frontiers(Fg):
        n = eng.stream_advance(f)
        assert n == min(f, Fg) * hop
        torch.cuda.current_stream().synchronize()
        chunks.append(o[:, :, prev * hop:n].clone())
        prev = min(f, Fg)
    assert prev == Fg
    return chunks, o, eng.launch_count - l0


def _geometric(first):
    def f(Fg):
        out, x, step = [], 0, first
        while x < Fg:
            x = min(x + step, Fg)
            out.append(x)
            step *= 2
        return out
    return f


SCHEDULES = {
    "geometric_32": _geometric(32),
    "chunks_of_7": lambda Fg: list(range(7, Fg, 7)) + [Fg],
    "one_chunk": lambda Fg: [Fg],
    "tile_edges": lambda Fg: sorted({e + d for e in (16, 128, 256) for d in (-1, 0, 1) if 0 < e + d < Fg}) + [Fg + 5],
}


@pytest.mark.parametrize("max_len", [None, 150])
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("precision", STREAM_PRECISIONS)
def test_stream_bit_identical_to_infer(engines, precision, case, schedule, max_len):
    eng = engines(precision)
    inp, nw, nz, kw = CASES[case]()
    ref, F = _one_shot(eng, inp, nw, nz, kw, max_len)
    chunks, o, launches = _stream(eng, inp, nw, nz, kw, max_len, SCHEDULES[schedule])
    torch.cuda.synchronize()
    got = torch.cat(chunks, -1)
    print(f"[{precision}/{case}/{schedule}/max_len={max_len}] F={F} samples={ref.shape[-1]} chunks={len(chunks)} generator launches={launches}")
    assert got.shape == ref.shape and torch.equal(got, ref)
    assert torch.equal(o, ref)  # no later window overwrote audio that an earlier chunk handed out


def test_every_frame_schedule_config2(engines):
    eng = engines("fp16")
    inp, nw, nz, kw = _config2()
    ref, F = _one_shot(eng, inp, nw, nz, kw, None)
    chunks, o, launches = _stream(eng, inp, nw, nz, kw, None, lambda Fg: list(range(1, Fg + 1)))
    print(f"every frame: F={F} chunks={len(chunks)} generator launches={launches}")
    assert torch.equal(torch.cat(chunks, -1), ref) and torch.equal(o, ref)


@pytest.mark.parametrize("precision", STREAM_PRECISIONS)
def test_infer_stream_matches_seeded_infer(engines, precision):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, sd = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=cfg.n_speakers, gin_channels=512, precision=precision, init_seed=0).to("cuda")
    inp = synth.synthetic_inputs(cfg, [96, 61], [0, 1], seed=9)
    args = [inp[k].cuda() for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")]
    torch.manual_seed(123)
    ref = net.infer(*args, **INFER_KW)[0].clone()
    ylen = net.last_y_lengths.copy()
    torch.manual_seed(123)
    net.last_y_lengths = None
    chunks, sizes = [], []
    for c in net.infer_stream(*args, **INFER_KW, first_chunk_frames=8):
        if not sizes:
            assert (net.last_y_lengths == ylen).all()
        sizes.append(c.shape[-1] // cfg.hop)
        chunks.append(c.clone())
    assert sizes[:3] == [8, 16, 32]
    assert torch.equal(torch.cat(chunks, -1), ref)


def test_second_stream_does_not_grow_workspace(engines):
    eng = engines("fp16")
    inp, nw, nz, kw = _config2()
    _stream(eng, inp, nw, nz, kw, None, SCHEDULES["geometric_32"])
    g = eng.workspace_grows
    _stream(eng, inp, nw, nz, kw, None, SCHEDULES["geometric_32"])
    assert eng.workspace_grows == g


def test_stream_state_errors(engines):
    eng = engines("fp16")
    inp, nw, nz, kw = _tflow_b3()
    B, T = inp["x"].shape
    with pytest.raises(Bv2Error):  # nothing open yet on a fresh begin
        eng.infer_begin(*_args(inp, nw, kw))
        eng.stream_advance(1)
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"])
    eng.stream_advance(4)
    with pytest.raises(Bv2Error):  # frames must increase
        eng.stream_advance(4)
    eng.stream_advance(5)
    eng.infer_begin(*_args(inp, nw, kw))  # resets the workspace: closes the stream
    with pytest.raises(Bv2Error):
        eng.stream_advance(6)
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"])
    eng.stream_advance(F + 100)  # reaches Fg: closes the stream
    with pytest.raises(Bv2Error):
        eng.stream_advance(F + 200)
    torch.cuda.synchronize()


def test_reserve_that_regrows_closes_the_stream(engines):
    """bv2_reserve regrowing the arenas frees what an open stream reads: the stream closes instead."""
    eng = engines("fp16")
    inp, nw, nz, kw = _tflow_b3()
    B, T = inp["x"].shape
    _, F = eng.infer_begin(*_args(inp, nw, kw))
    eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"])
    eng.stream_advance(4)
    eng.reserve(B + 64, T + 512, 4 * F)
    with pytest.raises(Bv2Error):
        eng.stream_advance(8)
    torch.cuda.synchronize()


def test_infer_stream_invalidates_earlier_attn(engines):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, _ = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=cfg.n_speakers, gin_channels=512, init_seed=0).to("cuda")
    inp = synth.synthetic_inputs(cfg, [20], [0], seed=5)
    args = [inp[k].cuda() for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")]
    _, attn, _, _ = net.infer(*args, **INFER_KW)
    for _ in net.infer_stream(*args, **INFER_KW):
        pass
    with pytest.raises(RuntimeError, match="earlier infer"):
        attn.materialize()
