"""ctypes binding of the ragged-stream harness (tests/cuda/ragged_stream_harness.cu): one k_g2_conv launch that is a window of a ragged
stream, on tensors held as a resident row range.  Layouts as in kernel_harness.py and stream_bounded_harness.py."""
import ctypes as C

import numpy as np

from bert_vits2_b200 import _lib
from kernel_harness import G2Args

_h = None


def load():
    global _h
    if _h is None:
        h = C.CDLL(_lib.build_harness(ragged_stream=True))
        P, I = C.c_void_p, C.POINTER(C.c_int)
        h.kh_g2_conv_ragged_stream.argtypes = [C.POINTER(G2Args), P] + [C.c_int] * 9 + [P, I, I]
        h.kh_last_error.restype = C.c_char_p
        _h = h
    return _h


def g2_conv_ragged_stream(args, lens, lens_scale, t_begin, t_end, x_base, x_rows, y_base, y_rows, res_base, res_rows, y_init):
    """k_g2_conv over [t_begin, t_end) as a window of a ragged stream (item b ends at min(t_end, lens[b] * lens_scale)), on resident
    storages; returns (y after the kernel, guards intact, error flag)"""
    y = np.array(y_init, copy=True)
    lens = np.ascontiguousarray(lens, np.int32)
    g, e = C.c_int(0), C.c_int(0)
    h = load()
    if h.kh_g2_conv_ragged_stream(C.byref(args), lens.ctypes.data, int(lens_scale), int(t_begin), int(t_end), int(x_base), int(x_rows), int(y_base),
                                  int(y_rows), int(res_base), int(res_rows), y.ctypes.data, C.byref(g), C.byref(e)) != 0:
        raise RuntimeError(h.kh_last_error().decode())
    return y, bool(g.value), e.value
