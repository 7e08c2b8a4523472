"""Concurrent requests on one GPU: sibling engines (bv2_create_sibling) share the packed weights and give bit-identical outputs,
requests on different siblings and CUDA streams give exactly their serial results, and SynthesizerTrn(concurrency=N) leases one
engine per request.  Run on an H100: pytest -m gpu."""
import ctypes as C
import gc
import threading

import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Bv2Error, Engine
from util import case_inputs, load_golden, model_for

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "fp16g", "fp16"]
INFER_KW = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.625)  # bench.py's config-2 settings
CTOR = (112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512, [16, 16, 8, 2, 2])
NAMES = ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")


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


def _request(lengths, languages, seed):
    """a request with its own lengths and noise, on the device"""
    cfg, _ = model_for(True, 0)
    inp = synth.synthetic_inputs(cfg, lengths, languages, seed=seed)
    nw, nz = synth.synthetic_noise(cfg, len(lengths), max(lengths), 2048, seed=seed)
    return {k: v.cuda() for k, v in inp.items()}, nw.cuda(), nz.cuda(), INFER_KW


def _args(inp, nw, kw):
    return tuple(inp[k] for k in NAMES) + (nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"])


def _run(eng, inp, nw, nz, kw, pcm16=False):
    """one request on the current stream; returns (y_lengths, o) with o final on that stream"""
    B, T = inp["x"].shape
    ylen, F = eng.infer_begin(*_args(inp, nw, kw))
    o, _, _, _ = eng.infer_finish(B, T, F, nz, kw["noise_scale"], want_attn=False, pcm16=pcm16)
    return ylen, o


def _stream_run(eng, inp, nw, nz, kw, chunk):
    B, T = inp["x"].shape
    ylen, F = eng.infer_begin(*_args(inp, nw, kw))
    o, _, _, _ = eng.infer_finish_stream(B, T, F, nz, kw["noise_scale"], want_attn=False)
    f = 0
    while f < F:
        f = min(f + chunk, F)
        eng.stream_advance(f)
    return ylen, o


# ---- sibling = source ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pcm16", [False, True])
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_sibling_equals_source(engines, precision, case, pcm16):
    src = engines(precision)
    sib = src.sibling()
    assert sib.workspace_bytes == 0
    inp, nw, nz, kw = CASES[case]()
    y0, o0 = _run(src, inp, nw, nz, kw, pcm16)
    y1, o1 = _run(sib, inp, nw, nz, kw, pcm16)
    torch.cuda.synchronize()
    assert (y0 == y1).all() and o0.shape == o1.shape and torch.equal(o0, o1)
    y2, o2 = _run(src, inp, nw, nz, kw, pcm16)  # the sibling's call left the source's results alone
    torch.cuda.synchronize()
    assert torch.equal(o2, o0)


# ---- concurrent = serial -------------------------------------------------------------------------------------------------
REQUESTS = [([64], [0], 11), ([48, 33], [1, 2], 12), ([128], [2], 13), ([40, 40, 17], [0, 1, 0], 14), ([96, 80], [0, 0], 15)]


@pytest.mark.parametrize("n_threads", [2, 4])
def test_concurrent_siblings_equal_serial(engines, n_threads):
    src = engines("fp16")
    reqs = [_request(*r) for r in REQUESTS]
    serial = []
    for r in reqs:
        y, o = _run(src, *r)
        serial.append((y, o.clone()))
    torch.cuda.synchronize()
    sibs = [src.sibling() for _ in range(n_threads)]
    got, errors = {}, []

    def worker(k):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for i in range(len(reqs)):
                    j = (i + k) % len(reqs)  # every thread runs every request, in a different order
                    got[(k, j)] = _run(sibs[k], *reqs[j])
            s.synchronize()
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(n_threads)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for (k, j), (y, o) in got.items():
        assert (y == serial[j][0]).all() and torch.equal(o, serial[j][1]), (k, j)


def test_stream_alongside_concurrent_infers(engines):
    src = engines("fp16")
    reqs = [_request(*r) for r in REQUESTS]
    serial = [_run(src, *r)[1].clone() for r in reqs]
    torch.cuda.synchronize()
    sibs = [src.sibling() for _ in range(3)]
    got, streamed, errors = {}, [], []

    def infer_worker(k):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for i in range(2 * len(reqs)):
                    j = (i + k) % len(reqs)
                    got[(k, i)] = (j, _run(sibs[k], *reqs[j])[1])
            s.synchronize()
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    def stream_worker():
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for j in (2, 4):
                    streamed.append((j, _stream_run(sibs[0], *reqs[j], chunk=5)[1]))
            s.synchronize()
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    ths = [threading.Thread(target=stream_worker)] + [threading.Thread(target=infer_worker, args=(k,)) for k in (1, 2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors  # in particular no BV2_ERR_STATE from a stream closed by another request
    for j, o in streamed:
        assert torch.equal(o, serial[j]), j
    for (j, o) in got.values():
        assert torch.equal(o, serial[j]), j


# ---- lifetime ------------------------------------------------------------------------------------------------------------
def test_sibling_outlives_source_and_family_rules(tmp_path):
    cfg, sd = model_for(True, 0)
    src = Engine(cfg, sd, device="cuda:0", precision="fp16")
    inp, nw, nz, kw = _tflow_b3()
    _, ref = _run(src, inp, nw, nz, kw)
    ref = ref.clone()
    sib = src.sibling()
    grand = sib.sibling()  # a sibling of a sibling joins the same family
    assert grand.workspace_bytes == 0
    lib = src.lib
    path = str(tmp_path / "w.bv2")
    grand.save_packed(path)  # bv2_save_packed works on any member
    del src
    gc.collect()
    _, o = _run(sib, inp, nw, nz, kw)
    _, o2 = _run(grand, inp, nw, nz, kw)
    torch.cuda.synchronize()
    assert torch.equal(o, ref) and torch.equal(o2, ref)
    w = np.zeros(4, dtype=np.float32)
    shape = (C.c_int64 * 1)(4)
    assert lib.bv2_set_weight(sib._h, b"emb_g.weight", C.c_void_p(w.ctypes.data), shape, 1, 0) == -2
    assert lib.bv2_finalize(sib._h) == -2
    assert lib.bv2_load_packed(sib._h, path.encode()) == -2
    with pytest.raises(Bv2Error):
        sib._check(lib.bv2_finalize(sib._h))
    # a packed file saved by a sibling loads into a fresh engine and gives the same output
    fresh = Engine(cfg, None, device="cuda:0", precision="fp16", packed_path=path)
    _, o3 = _run(fresh, inp, nw, nz, kw)
    torch.cuda.synchronize()
    assert torch.equal(o3, ref)
    del sib
    gc.collect()
    _, o4 = _run(grand, inp, nw, nz, kw)  # the last member still holds the weights
    torch.cuda.synchronize()
    assert torch.equal(o4, ref)


def test_sibling_of_unfinalized_engine_is_a_state_error():
    from bert_vits2_b200 import _lib
    from bert_vits2_b200.engine import PRECISIONS, _cfg_struct
    cfg, _ = model_for(True, 0)
    lib = _lib.load()
    h, s = C.c_void_p(), C.c_void_p()
    cs = _cfg_struct(cfg, PRECISIONS["fp16"])
    assert lib.bv2_create(C.byref(h), C.byref(cs), 0) == 0
    try:
        assert lib.bv2_create_sibling(C.byref(s), h) == -2 and not s.value
    finally:
        lib.bv2_destroy(h)


# ---- drop-in class -------------------------------------------------------------------------------------------------------
def _net(concurrency, precision="fp16"):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, _ = model_for(True, 0)
    return SynthesizerTrn(*CTOR, n_speakers=cfg.n_speakers, gin_channels=512, precision=precision, init_seed=0,
                          concurrency=concurrency).to("cuda")


def _net_call(net, r):
    inp, nw, nz, kw = r
    return net.infer(*[inp[k] for k in NAMES], noise_w=nw, noise_z=nz, **kw)


def _net_stream(net, r, first):
    inp, nw, nz, kw = r
    return torch.cat([c.clone() for c in net.infer_stream(*[inp[k] for k in NAMES], noise_w=nw, noise_z=nz, **kw,
                                                           first_chunk_frames=first)], -1)


def test_dropin_two_threads_one_engine():
    """concurrency=1: two threads calling infer() at once each get exactly their serial result (a request's begin..finish is
    one lease; before, the other thread's infer_begin could land in between)."""
    net = _net(1)
    reqs = [_request([120], [0], 21), _request([37, 64], [1, 2], 22)]
    serial = []
    for r in reqs:
        o = _net_call(net, r)[0].clone()
        serial.append((o, net.last_y_lengths.copy()))
    torch.cuda.synchronize()
    barrier = threading.Barrier(2)
    out, errors = {}, []

    def worker(k):
        try:
            for i in range(6):
                barrier.wait()
                o = _net_call(net, reqs[k])[0]
                out[(k, i)] = (o.clone(), net.last_y_lengths.copy())
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for (k, i), (o, y) in out.items():
        assert (y == serial[k][1]).all(), (k, i)
        assert o.shape == serial[k][0].shape and torch.equal(o, serial[k][0]), (k, i)


def test_dropin_pool_mixes_infer_and_stream():
    net = _net(3)
    reqs = [_request(*r) for r in REQUESTS[:3]]
    serial = []
    for r in reqs:
        o = _net_call(net, r)[0].clone()
        serial.append((o, net.last_y_lengths.copy()))
    torch.cuda.synchronize()
    out, errors = [], []

    def worker(k):
        try:
            for i in range(3):
                j = (i + k) % len(reqs)
                if (k + i) % 2:
                    o = _net_stream(net, reqs[j], 8)
                else:
                    o = _net_call(net, reqs[j])[0]
                out.append((k, j, o, net.last_y_lengths.copy()))
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(6)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    assert len(out) == 18
    pool = net._pool(torch.device("cuda", 0))
    assert 1 <= len(pool.engines) <= 3 and pool.engines[0] is net._engine(torch.device("cuda", 0))
    for k, j, o, y in out:
        assert (y == serial[j][1]).all(), (k, j)
        assert torch.equal(o, serial[j][0]), (k, j)


@pytest.mark.parametrize("concurrency", [1, 2])
def test_lazy_attn_after_its_engine_served_another_request(concurrency):
    net = _net(concurrency)
    r = _request([30], [0], 31)
    _, attn, _, _ = _net_call(net, r)
    _, attn2, _, _ = _net_call(net, r)  # one thread: the same (most recently released) engine serves it
    assert attn2.materialize().shape == attn2.shape
    with pytest.raises(RuntimeError, match="earlier infer"):
        attn.materialize()
