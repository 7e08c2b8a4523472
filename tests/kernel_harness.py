"""ctypes binding of the kernel test harness (tests/cuda/kernel_harness.cu) and the numpy device layouts it takes:
  c4  fp32   [B][C/4][T][4]
  c8  fp16   [B][C/8][T][8]
  H8  fp16   [B][C/8][PADL + T + PADR][8]   (Generator activations with their zero halo rows)
"""
import ctypes as C
import os

import numpy as np

from bert_vits2_b200 import _lib

KIND_NAMES = {0: "one-tile", 1: "persist", 2: "pstream"}


class TcArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("B", "T", "Cin", "Cout", "K", "u", "x_C", "y_C", "nt", "kc", "f16", "num_sms")] + [
        ("in_slope", C.c_float)] + [(n, C.c_int) for n in ("in_mask", "relu", "res_mode", "res_C_total", "res_c_off", "accumulate")] + [
        ("out_scale", C.c_float)] + [(n, C.c_int) for n in ("out_mask", "bias_b_stride", "cin_off", "cout_off", "dil", "out_tf32", "skip_xform",
                                                             "in_f16", "out_f16", "gate", "res_is_y")] + [
        ("w", C.c_void_p), ("bias", C.c_void_p), ("x", C.c_void_p), ("x_bytes", C.c_longlong), ("res", C.c_void_p), ("res_elems", C.c_longlong),
        ("lens", C.c_void_p), ("bias_b", C.c_void_p), ("bias_b_elems", C.c_longlong), ("ln_gamma", C.c_void_p), ("ln_beta", C.c_void_p)]


class TcPlan(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("kind", "gen", "f16", "res_smem", "nas", "nws", "grid_x", "grid_y", "grid_z", "threads", "mtiles",
                                       "ntiles", "total", "tiles_per_cta", "nt")] + [("smem", C.c_longlong)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}

    def __str__(self):
        return (f"{KIND_NAMES[self.kind]}<GEN={self.gen},F16={self.f16}> nt={self.nt} res_smem={self.res_smem} nas={self.nas} nws={self.nws} "
                f"grid=({self.grid_x},{self.grid_y},{self.grid_z}) tiles/CTA={self.tiles_per_cta} smem={self.smem // 1024}KB")


class G2Args(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("B", "T", "Cin", "Cout", "K", "u", "dil", "residual", "accumulate")] + [("out_scale", C.c_float)] + [
        (n, C.c_int) for n in ("bias_b_stride", "st_override", "num_sms")] + [
        ("w", C.c_void_p), ("bias", C.c_void_p), ("bias_b", C.c_void_p), ("bias_b_elems", C.c_longlong), ("x", C.c_void_p), ("res", C.c_void_p)]


class G2Plan(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("resident", "NG", "MG", "nas", "nws", "grid_x", "grid_y", "grid_z", "nt", "kc")] + [("smem", C.c_longlong)]

    def __str__(self):
        return (f"g2<{'resident' if self.resident else 'streamed'}> NG={self.NG} MG={self.MG} nt={self.nt} kc={self.kc} nas={self.nas} "
                f"nws={self.nws} grid=({self.grid_x},{self.grid_y},{self.grid_z}) smem={self.smem // 1024}KB")


_lib_h = None


def load(build=True):
    """dlopen the harness, rebuilding it first if it is missing or older than its source or a product header (BV2_KERNEL_HARNESS: load that
    library instead)."""
    global _lib_h
    if _lib_h is None:
        path = os.environ.get("BV2_KERNEL_HARNESS")  # development: run the suite against another build of the harness
        if not path:
            if build:
                _lib.build_harness()
            path = _lib.HARNESS_PATH
        h = C.CDLL(path)
        P, I = C.c_void_p, C.POINTER(C.c_int)
        h.kh_tc_plan.argtypes = [C.POINTER(TcArgs), C.POINTER(TcPlan)]
        h.kh_tc_conv1d.argtypes = [C.POINTER(TcArgs), P, C.c_longlong, C.POINTER(TcPlan), I, I]
        h.kh_flow_attn.argtypes = [P, P, P, P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P, I, I, I]
        h.kh_g2_plan.argtypes = [C.POINTER(G2Args), C.POINTER(G2Plan)]
        h.kh_g2_conv.argtypes = [C.POINTER(G2Args), P, C.POINTER(G2Plan), I, I]
        h.kh_c4_to_h8.argtypes = [P, P] + [C.c_int] * 7 + [P, I, I]
        h.kh_last_error.restype = C.c_char_p
        _lib_h = h
    return _lib_h


def _check(rc):
    if rc != 0:
        raise RuntimeError(load().kh_last_error().decode())


# ---------------------------------------------------------------- layouts
def to_c4(a):
    B, Cc, T = a.shape
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(B, Cc // 4, 4, T).transpose(0, 1, 3, 2))


def from_c4(buf, B, Cc, T):
    return np.asarray(buf).view(np.float32).reshape(B, Cc // 4, T, 4).transpose(0, 1, 3, 2).reshape(B, Cc, T)


def to_c8(a):
    B, Cc, T = a.shape
    return np.ascontiguousarray(np.asarray(a, np.float32).astype(np.float16).reshape(B, Cc // 8, 8, T).transpose(0, 1, 3, 2))


def from_c8(buf, B, Cc, T):
    return np.asarray(buf).view(np.float16).reshape(B, Cc // 8, T, 8).transpose(0, 1, 3, 2).reshape(B, Cc, T).astype(np.float32)


def g2_pads():
    h = load()
    return h.kh_g2_padl(), h.kh_g2_padr()


def to_h8(a, halo=0.0):
    """[B][C][T] fp16-representable values -> H8 with halo rows set to `halo` (0 for a conv input, NaN for an output buffer)"""
    pl, pr = g2_pads()
    B, Cc, T = a.shape
    h = np.full((B, Cc // 8, pl + T + pr, 8), halo, np.float16)
    h[:, :, pl:pl + T, :] = np.asarray(a, np.float32).astype(np.float16).reshape(B, Cc // 8, 8, T).transpose(0, 1, 3, 2)
    return h


def h8_data(h):
    """H8 -> ([B][C][T] float32 data rows, halo rows [B][C/8][PADL + PADR][8])"""
    pl, pr = g2_pads()
    B, G, Tp, _ = h.shape
    T = Tp - pl - pr
    data = h[:, :, pl:pl + T, :].transpose(0, 1, 3, 2).reshape(B, G * 8, T).astype(np.float32)
    halo = np.concatenate([h[:, :, :pl, :], h[:, :, pl + T:, :]], axis=2)
    return data, halo


# ---------------------------------------------------------------- entry points
def tc_args(**kw):
    a = TcArgs()
    a.in_slope = 1.0
    a.out_scale = 1.0
    a.dil = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def tc_plan(args):
    p = TcPlan()
    _check(load().kh_tc_plan(C.byref(args), C.byref(p)))
    return p


def tc_conv1d(args, y_init):
    """runs one tc_conv1d; returns (y after the kernel, plan, guards intact, device error flag)"""
    y = np.array(y_init, copy=True)
    p, g, e = TcPlan(), C.c_int(0), C.c_int(0)
    _check(load().kh_tc_conv1d(C.byref(args), y.ctypes.data, y.nbytes, C.byref(p), C.byref(g), C.byref(e)))
    return y, p, bool(g.value), e.value


def flow_attn(qkv16, rel_k, rel_v, lens, B, T, H, heads, window, ks_override, num_sms, att_init):
    att = np.array(att_init, copy=True)
    ks, g, e = C.c_int(0), C.c_int(0), C.c_int(0)
    rel_k = np.ascontiguousarray(rel_k, np.float32)
    rel_v = np.ascontiguousarray(rel_v, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    _check(load().kh_flow_attn(qkv16.ctypes.data, rel_k.ctypes.data, rel_v.ctypes.data, lens.ctypes.data, B, T, H, heads, window,
                               ks_override, num_sms, att.ctypes.data, C.byref(ks), C.byref(g), C.byref(e)))
    return att, ks.value, bool(g.value), e.value


def g2_args(**kw):
    a = G2Args()
    a.out_scale = 1.0
    a.dil = 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def g2_plan(args):
    p = G2Plan()
    _check(load().kh_g2_plan(C.byref(args), C.byref(p)))
    return p


def g2_conv(args, y_init):
    y = np.array(y_init, copy=True)
    p, g, e = G2Plan(), C.c_int(0), C.c_int(0)
    _check(load().kh_g2_conv(C.byref(args), y.ctypes.data, C.byref(p), C.byref(g), C.byref(e)))
    return y, p, bool(g.value), e.value


def c4_to_h8(x_c4, lens, B, Cc, T, t_begin, t_end, y_base, y_init):
    """k_c4_to_h8 over rows [t_begin, t_end) into an H8 holding the logical rows from y_base (y_init: [B][C/8][PADL + rows + PADR][8] f16);
    returns (y after the kernel, guards intact, device error flag)"""
    pl, pr = g2_pads()
    y = np.array(y_init, np.float16, copy=True)
    x_c4 = np.ascontiguousarray(x_c4, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    g, e = C.c_int(0), C.c_int(0)
    _check(load().kh_c4_to_h8(x_c4.ctypes.data, lens.ctypes.data, B, Cc, T, int(t_begin), int(t_end), int(y_base), y.shape[2] - pl - pr,
                              y.ctypes.data, C.byref(g), C.byref(e)))
    return y, bool(g.value), e.value
