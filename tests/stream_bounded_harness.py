"""ctypes binding of the bounded-stream harness (tests/cuda/stream_bounded_harness.cu): the resident-range planner of a bounded
Generator stream (host only) and the launches on tensors held as a resident row range.  Layouts as in kernel_harness.py."""
import ctypes as C
import os

import numpy as np

from bert_vits2_b200 import _lib
from kernel_harness import G2Args
from stream_harness import Graph

_h = None


def load(build=True):
    """dlopen the bounded-stream harness, rebuilding it first if it is missing or stale (BV2_STREAM_BOUNDED_HARNESS: load that library
    instead)."""
    global _h
    if _h is None:
        path = os.environ.get("BV2_STREAM_BOUNDED_HARNESS")
        if not path:
            if build:
                _lib.build_harness(bounded=True)
            path = _lib.BOUNDED_HARNESS_PATH
        h = C.CDLL(path)
        P, I = C.c_void_p, C.POINTER(C.c_int)
        h.kh_gen_tensor_need.argtypes = [P, C.c_int, C.c_int, P, C.c_int]
        h.kh_gen_resident_begin.argtypes = [P, C.c_int, C.c_int, P, C.c_int]
        h.kh_gen_stream_capacity.argtypes = [P, C.c_int, P, C.c_int]
        h.kh_gen_stream_slides.argtypes = [P, C.c_int, P, P, C.c_int, C.c_int, P, C.c_int]
        h.kh_g2_conv_resident.argtypes = [C.POINTER(G2Args)] + [C.c_int] * 8 + [P, I, I]
        h.kh_conv_post_resident.argtypes = [P, C.c_int, C.c_int, P, C.c_int, C.c_int, C.c_int, C.c_int, P, I, I]
        h.kh_g2_slide.argtypes = [C.c_int, P, P, P, P, P, P, P, I, I]
        h.kh_last_error.restype = C.c_char_p
        _h = h
    return _h


def _check(rc):
    if rc != 0:
        raise RuntimeError(load().kh_last_error().decode())


class BoundedGraph(Graph):
    """Graph (the layers, tensors and chunk windows of stream_harness) plus the bounded-stream planner"""

    def _per_tensor(self, fn, *args):
        out = np.zeros(512, np.int32)
        n = fn(C.byref(self.cs), *args, out.ctypes.data, 512)
        if n < 0:
            _check(-1)
        return out[:n].copy()

    def tensor_need(self, frontier):
        """rows of each tensor that are final once the frontier is at `frontier` frames"""
        return self._per_tensor(load().kh_gen_tensor_need, self.Fg, int(frontier))

    def resident_begin(self, done):
        """first row of each tensor that a window after frontier `done` still reads"""
        return self._per_tensor(load().kh_gen_resident_begin, self.Fg, int(done))

    def capacity(self, max_chunk_frames):
        """rows of storage per tensor of a bounded stream (does not depend on Fg)"""
        return self._per_tensor(load().kh_gen_stream_capacity, int(max_chunk_frames))

    def slides(self, cap, base, done, target):
        """slides before the chunk done -> target: [(tensor, src, dst, rows)]; `base` (int32 array) is updated in place"""
        cap = np.ascontiguousarray(cap, np.int32)
        assert base.dtype == np.int32 and base.flags.c_contiguous
        out = np.zeros((512, 4), np.int32)
        n = load().kh_gen_stream_slides(C.byref(self.cs), self.Fg, cap.ctypes.data, base.ctypes.data, int(done), int(target), out.ctypes.data, 512)
        if n < 0:
            _check(-1)
        return [tuple(map(int, r)) for r in out[:n]]



def g2_conv_resident(args, t_begin, t_end, x_base, x_rows, y_base, y_rows, res_base, res_rows, y_init):
    """k_g2_conv over [t_begin, t_end) on resident storages (args.x / args.res / y_init hold rows [base, base + rows) plus halo rows)"""
    y = np.array(y_init, copy=True)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_g2_conv_resident(C.byref(args), int(t_begin), int(t_end), int(x_base), int(x_rows), int(y_base), int(y_rows), int(res_base),
                                      int(res_rows), y.ctypes.data, C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value


def conv_post_resident(x_store, x_base, x_rows, w, B, T, t_begin, t_end, y_init):
    y = np.array(y_init, np.float32, copy=True)
    w = np.ascontiguousarray(w, np.float32)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_conv_post_resident(x_store.ctypes.data, int(x_base), int(x_rows), w.ctypes.data, B, T, int(t_begin), int(t_end), y.ctypes.data,
                                        C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value


def g2_slide(bufs, descs):
    """one k_g2_slide launch; bufs: H8 storages [B][C/8][PADL + rows + PADR][8] (float16), descs: [(src, dst, rows)] per buffer"""
    outs = [np.array(b, copy=True) for b in bufs]
    n = len(outs)
    ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    nbytes = np.array([o.nbytes for o in outs], np.int64)
    blocks = np.array([o.shape[0] * o.shape[1] for o in outs], np.int32)
    Tp = np.array([o.shape[2] for o in outs], np.int32)
    src, dst, rows = (np.array([d[k] for d in descs], np.int32) for k in range(3))
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_g2_slide(n, ptrs, nbytes.ctypes.data, blocks.ctypes.data, Tp.ctypes.data, src.ctypes.data, dst.ctypes.data, rows.ctypes.data,
                              C.byref(g), C.byref(e)))
    return outs, bool(g.value), e.value
