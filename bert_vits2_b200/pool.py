"""Engine pool behind SynthesizerTrn(concurrency=N): leases one engine per request.

An engine serves one request at a time: infer_begin .. infer_finish (or a stream up to its last chunk) spans several C calls whose
state lives in the engine.  The pool hands each request a whole engine for its duration: the primary engine, or one of up to N - 1
siblings (same device weights, own workspace) created the first time every existing engine is leased.  No GPU is touched here:
engines come from the caller's `make_sibling`, so tests can substitute stand-ins.
"""
from __future__ import annotations

import contextlib
import threading


class EnginePool:
    def __init__(self, primary, concurrency: int, make_sibling):
        if int(concurrency) < 1:
            raise ValueError("concurrency must be >= 1")
        self.primary = primary
        self.concurrency = int(concurrency)
        self._make_sibling = make_sibling
        self._engines = [primary]  # every member, primary first
        self._free = [primary]     # LIFO: the most recently used engine (warm workspace) is leased first
        self._owner = {}           # id(engine) -> ident of the thread that leased it
        self._cv = threading.Condition()

    @property
    def engines(self):
        with self._cv:
            return list(self._engines)

    def acquire(self, engine=None):
        """Lease a free engine (`engine`: that member), creating a sibling if all are leased and fewer than `concurrency` exist;
        otherwise wait for a release.  A thread that already holds a lease and would have to wait raises RuntimeError instead:
        the lease it waits for may be its own."""
        me = threading.get_ident()
        with self._cv:
            if engine is not None and not any(e is engine for e in self._engines):
                raise ValueError("engine is not a member of this pool")
            while True:
                if engine is None and self._free:
                    eng = self._free.pop()
                    break
                if engine is None and len(self._engines) < self.concurrency:
                    eng = self._make_sibling(self.primary)
                    self._engines.append(eng)
                    break
                if engine is not None and any(e is engine for e in self._free):
                    self._free = [e for e in self._free if e is not engine]
                    eng = engine
                    break
                if me in self._owner.values():
                    raise RuntimeError(f"no free engine (concurrency={self.concurrency}) and this thread already holds one: waiting "
                                       "would deadlock (finish or close the open infer_stream first, or raise concurrency)")
                self._cv.wait()
            self._owner[id(eng)] = me
            return eng

    def release(self, eng):
        with self._cv:
            del self._owner[id(eng)]
            self._free.append(eng)
            self._cv.notify_all()

    @contextlib.contextmanager
    def lease(self, engine=None):
        eng = self.acquire(engine)
        try:
            yield eng
        finally:
            self.release(eng)
