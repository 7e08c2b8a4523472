"""CPU checks of the engine pool behind SynthesizerTrn(concurrency=N), with stand-in engines: lease limits, blocking, the
self-deadlock guard, lease release by an unfinished infer_stream generator, and invalidation."""
import gc
import threading
import time
import weakref

import numpy as np
import pytest
import torch

from bert_vits2_b200.models import SynthesizerTrn
from bert_vits2_b200.pool import EnginePool

HOP = 512


class FakeEngine:
    """Stands in for engine.Engine: the calls infer() / infer_stream() make, with one frame per token."""

    def __init__(self, made):
        self.device = torch.device("cuda", 0)
        self.made = made
        made.append(self)

    def sibling(self):
        return FakeEngine(self.made)

    def infer_begin(self, x, x_lengths, *a):
        self._ylen = x_lengths.numpy().astype(np.int64)
        time.sleep(0.01)  # a window in which another thread's call could interleave
        return self._ylen.copy(), int(self._ylen.max())

    def infer_finish(self, B, T, F, noise_z, noise_scale, max_len=None, want_attn=True, pcm16=False):
        o = torch.zeros(B, 1, F * HOP)
        o[:, 0, :] = torch.from_numpy(self._ylen).float()[:, None]
        return o, None, torch.ones(B, 1, F), (None, None, None, None)

    def infer_finish_stream(self, B, T, F, noise_z, noise_scale, max_len=None, want_attn=True):
        return self.infer_finish(B, T, F, noise_z, noise_scale)

    def stream_advance(self, frames):
        return frames * HOP


class _Ev:
    def record(self, stream=None):
        pass

    def synchronize(self):
        pass


@pytest.fixture
def net(monkeypatch):
    """A SynthesizerTrn whose engines are stand-ins (no device is touched); .made lists every engine created."""
    def make(concurrency=1):
        n = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                           [16, 16, 8, 2, 2], n_speakers=4, gin_channels=512, init_seed=None, concurrency=concurrency)
        made = []
        primary = FakeEngine(made)
        monkeypatch.setattr(n, "_cuda_device", lambda what: torch.device("cuda", 0))
        monkeypatch.setattr(n, "_engine", lambda dev: primary)
        n.made = made
        return n
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "Event", _Ev)
    return make


def _args(T, n):
    x = torch.zeros(1, T, dtype=torch.int64)
    return (x, torch.tensor([n]), torch.zeros(1, dtype=torch.int64), x, x, torch.zeros(1, 1024, T), torch.zeros(1, 1024, T),
            torch.zeros(1, 1024, T))


def _kw(T):
    return dict(noise_w=torch.zeros(1, 2, T), noise_z=torch.zeros(1, 192, T))


def test_pool_never_exceeds_concurrency():
    made, active, peak = [], [0], [0]
    lock = threading.Lock()
    pool = EnginePool(FakeEngine(made), 3, lambda p: p.sibling())

    def worker():
        for _ in range(20):
            with pool.lease():
                with lock:
                    active[0] += 1
                    peak[0] = max(peak[0], active[0])
                time.sleep(0.001)
                with lock:
                    active[0] -= 1
    ths = [threading.Thread(target=worker) for _ in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert peak[0] == 3 and len(made) == 3 and len(pool.engines) == 3


def test_single_thread_reuses_the_primary():
    made = []
    pool = EnginePool(FakeEngine(made), 4, lambda p: p.sibling())
    for _ in range(5):
        with pool.lease() as e:
            assert e is made[0]
    assert len(made) == 1  # siblings are only created when every engine is leased


def test_extra_caller_blocks_until_release():
    made = []
    pool = EnginePool(FakeEngine(made), 2, lambda p: p.sibling())
    a, b = pool.acquire(), pool.acquire()
    got = []
    t = threading.Thread(target=lambda: got.append(pool.acquire()))
    t.start()
    time.sleep(0.2)
    assert not got and t.is_alive()
    pool.release(b)
    t.join(5)
    assert got == [b]
    pool.release(a)
    pool.release(b)


def test_nested_lease_raises_instead_of_deadlocking():
    made = []
    pool = EnginePool(FakeEngine(made), 1, lambda p: p.sibling())
    with pool.lease():
        with pytest.raises(RuntimeError, match="deadlock"):
            pool.acquire()
        with pytest.raises(RuntimeError, match="deadlock"):
            pool.acquire(made[0])  # a specific engine this thread holds
    with pool.lease():  # the failed attempts left nothing leased
        pass


def test_infer_inside_own_stream_raises(net):
    n = net(concurrency=1)
    gen = n.infer_stream(*_args(8, 8), **_kw(8), first_chunk_frames=2)
    next(gen)
    with pytest.raises(RuntimeError, match="deadlock"):
        n.infer(*_args(8, 8), **_kw(8))
    gen.close()
    n.infer(*_args(8, 8), **_kw(8))  # closing the stream released its lease


def test_unfinished_stream_releases_its_lease(net):
    n = net(concurrency=1)
    pool = n._pool(torch.device("cuda", 0))
    gen = n.infer_stream(*_args(8, 8), **_kw(8), first_chunk_frames=2)
    assert next(gen).shape[-1] == 2 * HOP
    assert len(pool._free) == 0
    gen.close()
    assert len(pool._free) == 1
    gen = n.infer_stream(*_args(8, 8), **_kw(8), first_chunk_frames=2)
    next(gen)
    assert len(pool._free) == 0
    del gen
    gc.collect()
    assert len(pool._free) == 1
    chunks = list(n.infer_stream(*_args(8, 8), **_kw(8), first_chunk_frames=2))  # exhausted
    assert [c.shape[-1] // HOP for c in chunks] == [2, 4, 2] and len(pool._free) == 1


def test_invalidate_drops_the_siblings(net):
    n = net(concurrency=3)
    pool = n._pool(torch.device("cuda", 0))
    held = [pool.acquire() for _ in range(3)]
    for e in held:
        pool.release(e)
    refs = [weakref.ref(e) for e in n.made[1:]]
    assert len(refs) == 2
    del held, e, pool
    n._invalidate()
    assert not n._pools
    n.made.clear()
    gc.collect()
    assert all(r() is None for r in refs)


def test_last_y_lengths_is_per_thread(net):
    n = net(concurrency=1)
    barrier = threading.Barrier(2)
    seen = {}

    def worker(k):
        for _ in range(5):
            barrier.wait()
            o = n.infer(*_args(16, 3 + k), **_kw(16))[0]
            seen.setdefault(k, []).append((int(n.last_y_lengths[0]), int(o[0, 0, 0])))
    ths = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for k in range(2):
        assert seen[k] == [(3 + k, 3 + k)] * 5
    with pytest.raises(AttributeError):
        n.last_y_lengths  # this thread has made no call
