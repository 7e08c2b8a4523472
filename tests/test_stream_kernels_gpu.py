"""Time-window launches of the Generator kernels (k_g2_conv and tc_conv1d in every dispatch variant, the SIMT convs, the ConvTransposes,
conv_post): a windowed launch is bitwise equal to the full launch inside its window and leaves every row outside it untouched, halo
rows included.
Run on an H100: pytest -m gpu."""
import zlib

import numpy as np
import pytest

from kernel_harness import g2_args, g2_pads, to_h8
from stream_harness import conv1d_window, conv_post_simt_window, conv_post_window, convT_window, g2_conv_window, tc_conv1d_window

pytestmark = pytest.mark.gpu

# (name, Cin, Cout, K, u, dil, mode, st_override, T, (NG, MG) of the whole launch or None): the Generator's conv shapes of the default
# configuration; the forced super-tiles are those of a long utterance's stage 4 (NG 4 x MG 2, MG 5) and a stage-3 pipeline of 4 groups
SHAPES = [
    ("conv_pre", 192, 512, 7, 0, 1, "bias_b", 0, 300, None),
    ("ups0", 512, 256, 16, 8, 1, "plain", 0, 300, None),
    ("ups4", 32, 16, 2, 2, 1, "plain", 0, 300, None),
    ("s0_c1_k11_d5", 256, 256, 11, 0, 5, "plain", 0, 300, None),
    ("s0_c2_res", 256, 256, 3, 0, 1, "residual", 0, 300, None),
    ("s0_c2_acc", 256, 256, 7, 0, 1, "accumulate", 0, 300, None),
    ("s3_c1_k7_d3_st4", 32, 32, 7, 0, 3, "plain", 4, 600, (4, 1)),
    ("s2_c2_res_st1", 64, 64, 11, 0, 1, "residual", 1, 300, None),
    ("s4_resident_acc", 16, 16, 11, 0, 1, "accumulate", 0, 300, None),
    ("s4_resident_c1_d5", 16, 16, 3, 0, 5, "plain", 0, 300, None),
    ("s4_c2_res_ng4_mg2", 16, 16, 3, 0, 1, "residual", 8, 1500, (4, 2)),
    ("s4_c2_acc_mg5", 16, 16, 11, 0, 1, "accumulate", 5, 1500, (1, 5)),
]


def _windows(T):
    return [(0, T), (0, 1), (37, 201), (128, 256), (127, 129), (T - 5, T), (1, T - 1)]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_g2_window_bitwise(shape):
    name, Cin, Cout, K, u, dil, mode, st, T, expect = shape  # T: M rows of the launch (input rows of a ConvTranspose)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    B = 2
    To = T * (u or 1)
    pl, pr = g2_pads()
    w = (rng.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    x = to_h8(rng.standard_normal((B, Cin, T)).astype(np.float32))
    kw = dict(B=B, T=T, Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, st_override=st, num_sms=132,
              w=w.ctypes.data, bias=bias.ctypes.data, x=x.ctypes.data)
    keep = [w, bias, x]
    if mode == "bias_b":
        bb = (0.1 * rng.standard_normal((B, Cout))).astype(np.float32)
        keep.append(bb)
        kw.update(bias_b=bb.ctypes.data, bias_b_elems=bb.size, bias_b_stride=Cout)
    if mode == "residual":
        res = to_h8(rng.standard_normal((B, Cout, To)).astype(np.float32))
        keep.append(res)
        kw.update(res=res.ctypes.data, residual=1)
    if mode == "accumulate":
        kw.update(accumulate=1, out_scale=1.0 / 3)
    args = g2_args(**kw)
    # initial output: old values where a running sum accumulates, a NaN canary elsewhere; halo rows hold a distinct canary
    y0 = to_h8(rng.standard_normal((B, Cout, To)).astype(np.float32), halo=7.0) if mode == "accumulate" else to_h8(np.full((B, Cout, To), np.nan, np.float32), halo=7.0)
    yf, pf, gf, ef = g2_conv_window(args, 0, -1, y0)
    assert gf and ef == 0
    assert expect is None or (pf.NG, pf.MG) == expect, (name, str(pf))
    for a, b in _windows(T):
        yw, plan, g, e = g2_conv_window(args, a * (u or 1), b * (u or 1), y0)
        assert g and e == 0, (a, b)
        lo, hi = pl + a * (u or 1), pl + b * (u or 1)
        inside = np.zeros(yw.shape[2], bool)
        inside[lo:hi] = True
        if a == 0:
            inside[:pl] = True
        if b == T:
            inside[pl + To:] = True
        assert np.array_equal(_bits(yw[:, :, inside]), _bits(yf[:, :, inside])), (name, a, b, str(plan))
        assert np.array_equal(_bits(yw[:, :, ~inside]), _bits(y0[:, :, ~inside])), (name, a, b, "wrote outside its window")
        assert np.isfinite(yw[:, :, lo:hi].astype(np.float32)).all()


@pytest.mark.parametrize("T", [1, 511, 512, 513, 1500])
def test_conv_post_window_bitwise(T):
    rng = np.random.default_rng(T)
    B = 2
    x = to_h8(rng.standard_normal((B, 16, T)).astype(np.float32))
    w = (rng.standard_normal((16, 7)) / np.sqrt(16 * 7)).astype(np.float32)
    y0 = np.full((B, T), np.nan, np.float32)
    yf, g, e = conv_post_window(x, w, B, T, 0, T, y0)
    assert g and e == 0 and np.isfinite(yf).all()
    for a, b in {(0, T), (0, 1), (T // 3, T // 2 + 1), (max(0, T - 5), T), (min(T - 1, 511), T)}:
        if b <= a:
            continue
        yw, g, e = conv_post_window(x, w, B, T, a, b, y0)
        assert g and e == 0
        assert np.array_equal(yw[:, a:b].view(np.uint32), yf[:, a:b].view(np.uint32)), (T, a, b)
        out = np.ones(T, bool)
        out[a:b] = False
        assert np.isnan(yw[:, out]).all(), (T, a, b, "wrote outside its window")


# ---- TF32 Generator convs through tc_conv1d: every dispatch variant (forced through num_sms), windows keep the full-length plan
TC_FAMILIES = ["tf32.conv_pre", "tf32.ups0", "tf32.ups2", "tf32.ups4", "tf32.rb256.c1_k11d5", "tf32.rb256.c2_k11_acc", "tf32.rb32.c2_k7",
               "tf32.rb16.c1_k3d1", "tf32.rb64.c2_k11_acc"]


def _tc_case(name, B, T, num_sms, rng):
    import kernel_cases as KC
    from kernel_harness import to_c4
    f = KC.FAMILIES[name]
    u, Cin, Cout, K = f.get("u", 0), f["Cin"], f["Cout"], f["K"]
    a = KC.family_args(name, B, T, [T] * B, num_sms)
    To = T * (u or 1)
    keep = {}
    keep["x"] = to_c4(rng.standard_normal((B, Cin, T)).astype(np.float32))
    keep["w"] = (rng.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K)).astype(np.float32)
    keep["bias"] = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    keep["lens"] = np.full(B, T, np.int32)
    a.x, a.x_bytes, a.w, a.bias, a.lens = keep["x"].ctypes.data, keep["x"].nbytes, keep["w"].ctypes.data, keep["bias"].ctypes.data, keep["lens"].ctypes.data
    if f.get("bias_b"):
        keep["bb"] = (0.1 * rng.standard_normal((B, a.bias_b_stride))).astype(np.float32)
        a.bias_b, a.bias_b_elems = keep["bb"].ctypes.data, keep["bb"].size
    if f.get("res_mode"):
        keep["res"] = to_c4(rng.standard_normal((B, Cout, To)).astype(np.float32))
        a.res, a.res_elems = keep["res"].ctypes.data, keep["res"].size
    y0 = to_c4(rng.standard_normal((B, Cout, To)).astype(np.float32) if f.get("accumulate") else np.full((B, Cout, To), np.nan, np.float32))
    return a, y0, keep, u or 1, To


@pytest.mark.parametrize("num_sms", [132, 100000, 3], ids=["h100", "one_tile", "persistent"])
@pytest.mark.parametrize("name", TC_FAMILIES)
def test_tc_conv1d_window_bitwise(name, num_sms):
    rng = np.random.default_rng(zlib.crc32(f"{name}/{num_sms}".encode()))
    B, T = 2, 300
    a, y0, keep, u, To = _tc_case(name, B, T, num_sms, rng)
    yf, pf, gf, ef = tc_conv1d_window(a, 0, -1, y0)
    assert gf and ef == 0
    for lo, hi in _windows(T):
        yw, pw, g, e = tc_conv1d_window(a, lo * u, hi * u, y0)
        assert g and e == 0 and pw.kind == pf.kind and pw.nt == pf.nt, (name, lo, hi, str(pw), str(pf))
        inside = np.zeros(To, bool)
        inside[lo * u:hi * u] = True
        assert np.array_equal(yw[:, :, inside].view(np.uint32), yf[:, :, inside].view(np.uint32)), (name, lo, hi, str(pw))
        assert np.array_equal(yw[:, :, ~inside].view(np.uint32), y0[:, :, ~inside].view(np.uint32)), (name, lo, hi, "wrote outside its window")


# ---- fp32 SIMT Generator kernels
@pytest.mark.parametrize("shape", [(2, 300, 192, 512, 7, 1, 1.0, 0, 0), (2, 300, 256, 256, 11, 5, 0.1, 0, 0), (2, 300, 64, 64, 7, 1, 0.1, 1, 1),
                                   (1, 40, 16, 16, 3, 3, 0.1, 1, 0), (1, 40, 32, 32, 11, 1, 0.1, 1, 1)],
                         ids=["conv_pre", "c1_k11d5", "c2_res_acc", "small_tile_res", "small_tile_acc"])
def test_simt_conv1d_window_bitwise(shape):
    from kernel_harness import to_c4
    B, T, Cin, Cout, K, dil, slope, res, acc = shape
    rng = np.random.default_rng(zlib.crc32(str(shape).encode()))
    w = (rng.standard_normal((Cout, Cin, K)) / np.sqrt(Cin * K)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    x = to_c4(rng.standard_normal((B, Cin, T)).astype(np.float32))
    r = to_c4(rng.standard_normal((B, Cout, T)).astype(np.float32)) if res else None
    y0 = to_c4(rng.standard_normal((B, Cout, T)).astype(np.float32) if acc else np.full((B, Cout, T), np.nan, np.float32))
    yf, g, e = conv1d_window(B, T, Cin, Cout, K, dil, slope, w, bias, x, r, acc, 1.0 / 3 if acc else 1.0, 0, -1, y0)
    assert g and e == 0
    for lo, hi in [(0, T), (0, 1), (T // 3, T // 2 + 1), (T - 5, T), (1, T - 1)]:
        yw, g, e = conv1d_window(B, T, Cin, Cout, K, dil, slope, w, bias, x, r, acc, 1.0 / 3 if acc else 1.0, lo, hi, y0)
        assert g and e == 0
        inside = np.zeros(T, bool)
        inside[lo:hi] = True
        assert np.array_equal(yw[:, :, inside].view(np.uint32), yf[:, :, inside].view(np.uint32)), (shape, lo, hi)
        assert np.array_equal(yw[:, :, ~inside].view(np.uint32), y0[:, :, ~inside].view(np.uint32)), (shape, lo, hi, "outside")


@pytest.mark.parametrize("shape", [(512, 256, 16, 8), (128, 64, 8, 2), (32, 16, 2, 2)], ids=["ups0", "ups2", "ups4"])
def test_simt_convT_window_bitwise(shape):
    from kernel_harness import to_c4
    Cin, Cout, K, u = shape
    B, T = 2, 100
    rng = np.random.default_rng(zlib.crc32(str(shape).encode()))
    w = (rng.standard_normal((Cin, Cout, K)) / np.sqrt(Cin * K)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    x = to_c4(rng.standard_normal((B, Cin, T)).astype(np.float32))
    To = T * u
    y0 = to_c4(np.full((B, Cout, To), np.nan, np.float32))
    yf, g, e = convT_window(B, T, Cin, Cout, K, u, w, bias, x, 0, -1, y0)
    assert g and e == 0
    for lo, hi in [(0, T), (0, 1), (37, 61), (T - 5, T)]:
        yw, g, e = convT_window(B, T, Cin, Cout, K, u, w, bias, x, lo * u, hi * u, y0)
        inside = np.zeros(To, bool)
        inside[lo * u:hi * u] = True
        assert g and e == 0
        assert np.array_equal(yw[:, :, inside].view(np.uint32), yf[:, :, inside].view(np.uint32)), (shape, lo, hi)
        assert np.isnan(yw[:, :, ~inside]).all(), (shape, lo, hi, "outside")


@pytest.mark.parametrize("T", [1, 255, 256, 257, 1500])
def test_simt_conv_post_window_bitwise(T):
    from kernel_harness import to_c4
    rng = np.random.default_rng(T)
    B = 2
    x = to_c4(rng.standard_normal((B, 16, T)).astype(np.float32))
    w = (rng.standard_normal((16, 7)) / np.sqrt(16 * 7)).astype(np.float32)
    y0 = np.full((B, T), np.nan, np.float32)
    yf, g, e = conv_post_simt_window(x, w, B, T, 0, T, y0)
    assert g and e == 0 and np.isfinite(yf).all()
    for a, b in {(0, T), (0, 1), (T // 3, T // 2 + 1), (max(0, T - 5), T)}:
        if b <= a:
            continue
        yw, g, e = conv_post_simt_window(x, w, B, T, a, b, y0)
        assert g and e == 0
        assert np.array_equal(yw[:, a:b].view(np.uint32), yf[:, a:b].view(np.uint32)), (T, a, b)
        out = np.ones(T, bool)
        out[a:b] = False
        assert np.isnan(yw[:, out]).all()
