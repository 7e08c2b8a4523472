"""ctypes binding of the streaming harness (tests/cuda/stream_harness.cu): the Generator's wavefront planner (host only) and its
time-window kernel launches.  Layouts as in kernel_harness.py."""
import ctypes as C
import os

import numpy as np

from bert_vits2_b200 import _lib
from bert_vits2_b200.engine import _cfg_struct
from kernel_harness import G2Args, G2Plan, TcArgs, TcPlan

KINDS = ("conv_pre", "ups", "c1", "c2", "conv_post")
FIELDS = ("kind", "stage", "branch", "dil_idx", "in_", "out", "res", "reach", "u", "L_in", "L_out")

_h = None


def load(build=True):
    """dlopen the streaming harness, rebuilding it first if it is missing or stale (BV2_STREAM_HARNESS: load that library instead)."""
    global _h
    if _h is None:
        path = os.environ.get("BV2_STREAM_HARNESS")
        if not path:
            if build:
                _lib.build_harness(stream=True)
            path = _lib.STREAM_HARNESS_PATH
        h = C.CDLL(path)
        P, I = C.c_void_p, C.POINTER(C.c_int)
        h.kh_gen_graph.argtypes = [P, C.c_int, P, C.c_int, P, C.c_int, I, I]
        h.kh_gen_stream_plan.argtypes = [P, C.c_int, C.c_int, C.c_int, P, C.c_int]
        h.kh_g2_conv_window.argtypes = [C.POINTER(G2Args), C.c_int, C.c_int, P, C.POINTER(G2Plan), I, I]
        h.kh_conv_post_window.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P, I, I]
        h.kh_tc_conv1d_window.argtypes = [C.POINTER(TcArgs), C.c_int, C.c_int, P, C.c_longlong, C.POINTER(TcPlan), I, I]
        h.kh_conv1d_window.argtypes = [C.c_int] * 6 + [C.c_float, P, P, P, P, C.c_int, C.c_float, C.c_int, C.c_int, P, I, I]
        h.kh_convT_window.argtypes = [C.c_int] * 6 + [P, P, P, C.c_int, C.c_int, P, I, I]
        h.kh_conv_post_simt_window.argtypes = [P, P, C.c_int, C.c_int, C.c_int, C.c_int, P, I, I]
        h.kh_last_error.restype = C.c_char_p
        _h = h
    return _h


def _check(rc):
    if rc != 0:
        raise RuntimeError(load().kh_last_error().decode())


class Graph:
    """The Generator's layers in launch order (dicts with FIELDS) and its tensor lengths, for Fg frames."""

    def __init__(self, cfg, Fg):
        self.cs = _cfg_struct(cfg, 3)
        self.Fg = Fg
        desc = np.zeros((512, 11), np.int32)
        tl = np.zeros(512, np.int32)
        nt, hop = C.c_int(0), C.c_int(0)
        n = load().kh_gen_graph(C.byref(self.cs), Fg, desc.ctypes.data, 512, tl.ctypes.data, 512, C.byref(nt), C.byref(hop))
        if n < 0:
            _check(-1)
        self.layers = [dict(zip(FIELDS, map(int, row))) for row in desc[:n]]
        self.tensor_len = [int(v) for v in tl[:nt.value]]
        self.hop = hop.value

    def plan(self, done, target):
        """[(t_begin, t_end)] per layer for the chunk from `done` to `target` frames"""
        w = np.zeros((len(self.layers), 2), np.int32)
        n = load().kh_gen_stream_plan(C.byref(self.cs), self.Fg, int(done), int(target), w.ctypes.data, len(self.layers))
        if n < 0:
            _check(-1)
        return [tuple(map(int, r)) for r in w[:n]]


def g2_conv_window(args, t_begin, t_end, y_init):
    y = np.array(y_init, copy=True)
    p, g, e = G2Plan(), C.c_int(0), C.c_int(0)
    _check(load().kh_g2_conv_window(C.byref(args), int(t_begin), int(t_end), y.ctypes.data, C.byref(p), C.byref(g), C.byref(e)))
    return y, p, bool(g.value), e.value


def conv_post_window(x_h8, w, B, T, t_begin, t_end, y_init):
    y = np.array(y_init, np.float32, copy=True)
    w = np.ascontiguousarray(w, np.float32)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_conv_post_window(x_h8.ctypes.data, w.ctypes.data, B, T, int(t_begin), int(t_end), y.ctypes.data, C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value


def tc_conv1d_window(args, t_begin, t_end, y_init):
    y = np.array(y_init, copy=True)
    p, g, e = TcPlan(), C.c_int(0), C.c_int(0)
    _check(load().kh_tc_conv1d_window(C.byref(args), int(t_begin), int(t_end), y.ctypes.data, y.nbytes, C.byref(p), C.byref(g), C.byref(e)))
    return y, p, bool(g.value), e.value


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, np.float32)


def conv1d_window(B, T, Cin, Cout, K, dil, in_slope, w, bias, x_c4, res_c4, accumulate, out_scale, t_begin, t_end, y_init):
    """SIMT k_conv1d_c4 over a window; c4 buffers as kernel_harness.to_c4"""
    y = np.array(y_init, np.float32, copy=True)
    w, bias, x_c4, res_c4 = _f32(w), _f32(bias), _f32(x_c4), _f32(res_c4)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_conv1d_window(B, T, Cin, Cout, K, dil, in_slope, w.ctypes.data, bias.ctypes.data, x_c4.ctypes.data,
                                   None if res_c4 is None else res_c4.ctypes.data, accumulate, out_scale, int(t_begin), int(t_end),
                                   y.ctypes.data, C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value


def convT_window(B, T, Cin, Cout, K, u, w, bias, x_c4, n_begin, n_end, y_init):
    y = np.array(y_init, np.float32, copy=True)
    w, bias, x_c4 = _f32(w), _f32(bias), _f32(x_c4)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_convT_window(B, T, Cin, Cout, K, u, w.ctypes.data, bias.ctypes.data, x_c4.ctypes.data, int(n_begin), int(n_end),
                                  y.ctypes.data, C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value


def conv_post_simt_window(x_c4, w, B, T, t_begin, t_end, y_init):
    y = np.array(y_init, np.float32, copy=True)
    x_c4, w = _f32(x_c4), _f32(w)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_conv_post_simt_window(x_c4.ctypes.data, w.ctypes.data, B, T, int(t_begin), int(t_end), y.ctypes.data, C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value
