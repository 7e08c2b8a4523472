"""ctypes binding of the ragged-batch harness (tests/cuda/ragged_harness.cu): one k_g2_conv launch whose batch items stop at their own
lengths.  Arguments and layouts are those of the kernel harness (tests/kernel_harness.py)."""
import ctypes as C

import numpy as np

import kernel_harness as KH
from bert_vits2_b200 import _lib

_h = None


def load():
    global _h
    if _h is None:
        h = C.CDLL(_lib.build_harness(ragged=True))
        I = C.POINTER(C.c_int)
        h.kh_g2_conv_ragged.argtypes = [C.POINTER(KH.G2Args), C.c_void_p, C.c_int, C.c_void_p, C.POINTER(KH.G2Plan), I, I]
        h.kh_last_error.restype = C.c_char_p
        _h = h
    return _h


def g2_conv_ragged(args, lens, lens_scale, y_init):
    """k_g2_conv with item b's rows ending at min(T, lens[b] * lens_scale); returns (y after the kernel, plan, guards intact, error flag)"""
    y = np.array(y_init, copy=True)
    lens = np.ascontiguousarray(lens, np.int32)
    p, g, e = KH.G2Plan(), C.c_int(0), C.c_int(0)
    h = load()
    if h.kh_g2_conv_ragged(C.byref(args), lens.ctypes.data, int(lens_scale), y.ctypes.data, C.byref(p), C.byref(g), C.byref(e)) != 0:
        raise RuntimeError(h.kh_last_error().decode())
    return y, p, bool(g.value), e.value
