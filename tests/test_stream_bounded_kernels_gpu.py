"""Kernels of a bounded stream: k_g2_conv and k_conv_post_tanh_h8 on tensors held as a resident row range (storage smaller than the
tensor, at a non-zero base) are bitwise equal to the same window on the whole tensors and leave every other stored row untouched, and
k_g2_slide moves exactly the requested rows.
Run on an H100: pytest -m gpu."""
import zlib

import numpy as np
import pytest

from kernel_harness import g2_args, g2_pads, to_h8
from stream_bounded_harness import conv_post_resident, g2_conv_resident, g2_slide
from stream_harness import conv_post_window, g2_conv_window

pytestmark = pytest.mark.gpu

# (name, Cin, Cout, K, u, dil, mode)
SHAPES = [
    ("plain_k3", 256, 256, 3, 0, 1, "plain"),
    ("dilated_res_k7_d3", 128, 128, 7, 0, 3, "residual"),
    ("convT_ups0", 512, 256, 16, 8, 1, "plain"),
    ("convT_ups4", 32, 16, 2, 2, 1, "plain"),
    ("acc_k11", 64, 64, 11, 0, 1, "accumulate"),
]
T_IN = 300
WINDOWS = [(37, 201), (128, 256), (150, 300), (290, 300)]  # input-rate rows [a, b): inside, tile-aligned, to the end


def _ups_half(K, u):
    p, taps = (K - u) // 2, K // u
    offs = [(r + p) // u - m for r in range(u) for m in range(taps)]
    return max(-min(offs), max(offs))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


def _store(full, base, rows, canary=np.nan):
    """storage of logical rows [base, base + rows) of an H8 `full` (halo rows included): physical rows [-PADL, rows + PADR); rows the
    storage holds but that are not resident (below base, or past base + rows and before the tensor's end) hold a canary"""
    pl, pr = g2_pads()
    T = full.shape[2] - pl - pr
    s = np.array(full[:, :, base:base + pl + rows + pr], copy=True)
    if base > 0:
        s[:, :, :pl] = canary
    if base + rows < T:
        s[:, :, pl + rows:] = canary
    return s


@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_g2_conv_resident_bitwise(shape):
    name, Cin, Cout, K, u, dil, mode = shape
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    B, T = 2, T_IN
    U = u or 1
    To = T * U
    pl, pr = g2_pads()
    pad = _ups_half(K, u) if u else (K - 1) // 2 * dil
    w = (rng.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    x = to_h8(rng.standard_normal((B, Cin, T)).astype(np.float32))
    res = to_h8(rng.standard_normal((B, Cout, To)).astype(np.float32)) if mode == "residual" else None
    if mode == "accumulate":
        y0 = to_h8(rng.standard_normal((B, Cout, To)).astype(np.float32), halo=7.0)
    else:
        y0 = to_h8(np.full((B, Cout, To), np.nan, np.float32), halo=7.0)
    kw = dict(B=B, T=T, Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, num_sms=132, w=w.ctypes.data, bias=bias.ctypes.data)
    if mode == "residual":
        kw.update(residual=1)
    if mode == "accumulate":
        kw.update(accumulate=1, out_scale=1.0 / 3)
    for a, b in WINDOWS:
        x_base = a - pad
        x_rows = min(b + pad, T) - x_base
        y_base, y_rows = a * U, b * U - a * U
        assert x_base > 0 and x_rows < T and y_rows < To
        # the whole-tensor launch over the same window
        full_args = g2_args(**kw, x=x.ctypes.data, res=None if res is None else res.ctypes.data)
        yf, _, gf, ef = g2_conv_window(full_args, a * U, b * U, y0)
        assert gf and ef == 0
        xs = _store(x, x_base, x_rows)
        keep = [xs]
        res_base = res_rows = 0
        rkw = {}
        if res is not None:
            res_base, res_rows = a * U - 5, b * U - a * U + 5
            rs = _store(res, res_base, res_rows)
            keep.append(rs)
            rkw = dict(res=rs.ctypes.data)
        args = g2_args(**kw, x=xs.ctypes.data, **rkw)
        ys0 = np.array(y0[:, :, y_base:y_base + pl + y_rows + pr], copy=True)
        ys, g, e = g2_conv_resident(args, a * U, b * U, x_base, x_rows, y_base, y_rows, res_base, res_rows, ys0)
        assert g and e == 0, (name, a, b)
        # storage row i holds logical row y_base - pl + i, i.e. full row y_base + i
        inside = np.zeros(ys.shape[2], bool)
        inside[pl:pl + y_rows] = True
        if b == T:
            inside[pl + y_rows:] = True  # the zero halo after the tensor's end, written by the window that reaches it
        ref = yf[:, :, y_base:y_base + pl + y_rows + pr]
        assert np.array_equal(_bits(ys[:, :, inside]), _bits(ref[:, :, inside])), (name, a, b)
        assert np.array_equal(_bits(ys[:, :, ~inside]), _bits(ys0[:, :, ~inside])), (name, a, b, "wrote outside its window")
        assert np.isfinite(ys[:, :, pl:pl + y_rows].astype(np.float32)).all()


@pytest.mark.parametrize("T", [1500, 2048])
def test_conv_post_resident_bitwise(T):
    rng = np.random.default_rng(T)
    B = 2
    x = to_h8(rng.standard_normal((B, 16, T)).astype(np.float32))
    w = (rng.standard_normal((16, 7)) / np.sqrt(16 * 7)).astype(np.float32)
    y0 = np.full((B, T), np.nan, np.float32)
    for a, b in [(600, 1100), (511, 1025), (T - 700, T), (T - 3, T)]:
        yf, g, e = conv_post_window(x, w, B, T, a, b, y0)
        assert g and e == 0
        x_base, x_rows = a - 3, min(b + 3, T) - (a - 3)
        xs = _store(x, x_base, x_rows)
        yw, g, e = conv_post_resident(xs, x_base, x_rows, w, B, T, a, b, y0)
        assert g and e == 0
        assert np.array_equal(yw[:, a:b].view(np.uint32), yf[:, a:b].view(np.uint32)), (T, a, b)
        out = np.ones(T, bool)
        out[a:b] = False
        assert np.isnan(yw[:, out]).all(), (T, a, b, "wrote outside its window")


def test_g2_slide_moves_exactly_the_rows():
    rng = np.random.default_rng(7)
    pl, pr = g2_pads()
    # (B, C, rows of storage, src, dst, rows moved)
    cases = [(1, 512, 40, 25, 0, 12), (2, 256, 300, 170, 0, 130), (3, 16, 1000, 999, 0, 1), (1, 64, 64, 32, 0, 32), (2, 8, 50, 20, 3, 17)]
    bufs, descs = [], []
    for B, Cc, R, src, dst, n in cases:
        bufs.append(rng.standard_normal((B, Cc // 8, pl + R + pr, 8)).astype(np.float16))
        descs.append((src, dst, n))
    outs, g, e = g2_slide(bufs, descs)
    assert g and e == 0
    for buf, out, (src, dst, n) in zip(bufs, outs, descs):
        want = np.array(buf, copy=True)
        want[:, :, pl + dst:pl + dst + n] = buf[:, :, pl + src:pl + src + n]
        assert np.array_equal(_bits(out), _bits(want)), (src, dst, n)
