"""Kernel-level parity of the Generator kernels other than k_g2_conv on an H100, each against a float64 reference built from the module
semantics: the FP16 tail k_conv_post_tanh_h8, the fp32 tail k_conv_post_tanh, the Generator input conversion k_c4_to_h8, and the fp32
Generator's k_conv1d_c4 (both tiles) and k_convT_c4.  Run: pytest -m gpu tests/test_gen_kernels_gpu.py -v -s

Every case also checks: the output buffer starts as a NaN canary and every element the launch covers is written and finite, the guard
regions around the output are intact, the device error flag is clear, and a second run is bitwise identical.

Tolerances: fp32 accumulation |got - ref| <= 1e-5 mag + 1e-6 (mag = sum of |terms|, as tests/kernel_ref.py derives); the tanh tails
add 1e-6 for tanhf (tanh is 1-Lipschitz); k_c4_to_h8 is exact."""
import zlib

import numpy as np
import pytest

import kernel_cases as KC
import kernel_harness as KH
import kernel_ref as R
from stream_harness import conv1d_window, conv_post_simt_window, conv_post_window, convT_window
from util import report

pytestmark = pytest.mark.gpu

POST_T = [1, 3, 4, 511, 512, 513, 1500, 4099]  # the edges of the 512-output block (256 for the fp32 tail) and of the 7-tap halo


def _rng(cid):
    return np.random.default_rng(zlib.crc32(cid.encode()))


def _conv_post_ref(act, w):
    """tanh(conv_post(act)) in float64: act [B][16][T] already activated (leaky relu 0.01), w [16][7], zero padding 3"""
    acc, mag = R.conv1d(act, np.asarray(w, np.float64)[None])
    return np.tanh(acc[:, 0]), mag[:, 0]


def _check_run(name, r1, r2):
    (y1, g1, e1), (y2, g2, e2) = r1, r2
    assert e1 == 0 and e2 == 0, f"{name}: device error flag raised"
    assert g1 and g2, f"{name}: guard region around the output overwritten"
    assert y1.tobytes() == y2.tobytes(), f"{name}: second run not bitwise identical"
    assert np.isfinite(y1).all(), f"{name}: output elements left unwritten (NaN canary) or non-finite"


# ------------------------------------------------------------------------------------------------------------ conv_post + tanh
@pytest.mark.parametrize("T", POST_T)
def test_conv_post_tanh_h8(T):
    """FP16 tail on stored activations a = f16(lrelu_0.1(x)): the module computes tanh(conv_post(leaky_relu(x, 0.01))) with
    x = a >= 0 ? a : 10 a.  |a| up to 4 and both signs: tanh saturates in some outputs and is linear in others."""
    cid = f"conv_post_h8-T{T}"
    g = _rng(cid)
    B = 2
    a = R.f16(g.uniform(-4.0, 4.0, (B, 16, T)).astype(np.float32))
    w = (0.15 * g.standard_normal((16, 7))).astype(np.float32)
    x = KH.to_h8(a)
    y0 = np.full((B, T), np.nan, np.float32)
    r1 = conv_post_window(x, w, B, T, 0, T, y0)
    _check_run(cid, r1, conv_post_window(x, w, B, T, 0, T, y0))
    xm = R.unlrelu10(a).astype(np.float64)
    ref, mag = _conv_post_ref(np.where(xm >= 0, xm, 0.01 * xm), w)
    if T >= 511:
        assert (np.abs(ref) > 0.99).any() and (np.abs(ref) < 0.5).any(), "inputs must reach both the saturated and the linear range"
    report(cid, f"k_conv_post_tanh_h8<16,7> grid=({-(-T // 512)},{B})", np.abs(r1[0].astype(np.float64) - ref), 1e-5 * mag + 2e-6, mag,
           np.ones(ref.shape, bool), "(b, t)")


@pytest.mark.parametrize("T", POST_T)
def test_conv_post_tanh_fp32(T):
    """fp32 tail: tanh(conv_post(leaky_relu(x, 0.01))) on fp32 activations"""
    cid = f"conv_post_fp32-T{T}"
    g = _rng(cid)
    B = 2
    x = g.uniform(-4.0, 4.0, (B, 16, T)).astype(np.float32)
    w = (0.15 * g.standard_normal((16, 7))).astype(np.float32)
    xc = KH.to_c4(x)
    y0 = np.full((B, T), np.nan, np.float32)
    r1 = conv_post_simt_window(xc, w, B, T, 0, T, y0)
    _check_run(cid, r1, conv_post_simt_window(xc, w, B, T, 0, T, y0))
    x64 = x.astype(np.float64)
    ref, mag = _conv_post_ref(np.where(x64 >= 0, x64, 0.01 * x64), w)
    report(cid, f"k_conv_post_tanh<16,7> grid=({-(-T // 256)},{B})", np.abs(r1[0].astype(np.float64) - ref), 1e-5 * mag + 2e-6, mag,
           np.ones(ref.shape, bool), "(b, t)")


# ------------------------------------------------------------------------------------------------------------ k_c4_to_h8
# (id, C, T, lens, t_begin, t_end, y_base, storage rows): whole tensors with ragged lengths (1 and T included) around the 128-row block,
# and windows of a bounded stream's input written into storage that starts at logical row y_base > 0
C4H8_CASES = [
    ("whole-T1", 16, 1, [1, 1, 1], 0, 1, 0, 1),
    ("whole-T127", 192, 127, [127, 1, 64], 0, 127, 0, 127),
    ("whole-T128", 16, 128, [1, 128, 127], 0, 128, 0, 128),
    ("whole-T129", 192, 129, [129, 128, 1], 0, 129, 0, 129),
    ("whole-T300", 32, 300, [300, 1, 129], 0, 300, 0, 300),
    ("window-mid-base100", 192, 300, [300, 1, 250], 130, 260, 100, 200),
    ("window-end-base150", 16, 300, [300, 200, 1], 200, 300, 150, 150),
    ("window-start", 32, 400, [400, 129, 1], 0, 129, 0, 200),
]


@pytest.mark.parametrize("cid,Cc,T,lens,a,b,base,rows", C4H8_CASES, ids=[c[0] for c in C4H8_CASES])
def test_c4_to_h8(cid, Cc, T, lens, a, b, base, rows):
    """exact: logical row t of the output is f16_rn(x[t]) for t < lens[b] and +0 past it (rows past the length are not read: they hold
    huge values here), saturating at +-65504; halo rows are zero where the window reaches an end of the tensor; every other storage row
    keeps its canary bit for bit"""
    g = _rng(cid)
    B = len(lens)
    pl, pr = KH.g2_pads()
    x = (3 * g.standard_normal((B, Cc, T))).astype(np.float32)
    x.reshape(-1)[::97] = 1e5   # saturates to 65504
    x.reshape(-1)[5::89] = np.float32(1 + 2.0 ** -11)  # a tie: rounds to even (1.0)
    valid = np.arange(T)[None, :] < np.asarray(lens)[:, None]
    x = np.where(valid[:, None, :], x, np.float32(3e38))
    canary = np.frombuffer(np.uint16(0x7E5A).tobytes(), np.float16)[0]  # a NaN payload the kernel never writes
    y0 = np.full((B, Cc // 8, pl + rows + pr, 8), canary, np.float16)
    r1 = KH.c4_to_h8(KH.to_c4(x), lens, B, Cc, T, a, b, base, y0)
    r2 = KH.c4_to_h8(KH.to_c4(x), lens, B, Cc, T, a, b, base, y0)
    assert r1[2] == 0 and r2[2] == 0 and r1[1] and r2[1], f"{cid}: device error flag or guard region"
    assert r1[0].tobytes() == r2[0].tobytes(), f"{cid}: second run not bitwise identical"
    want = y0.copy()
    ref = R.f16(np.where(valid[:, None, :], x, 0.0)).astype(np.float16)  # [B][C][T]
    want[:, :, pl + a - base:pl + b - base, :] = ref[:, :, a:b].reshape(B, Cc // 8, 8, b - a).transpose(0, 1, 3, 2)
    if a == 0:
        want[:, :, :pl, :] = 0
    if b == T:
        want[:, :, pl + T - base:pl + T - base + pr, :] = 0
    got = r1[0].view(np.uint16)
    bad = got != want.view(np.uint16)
    print(f"\n  {cid}: k_c4_to_h8 rows [{a}, {b}) base {base} | {int(bad.sum())} element(s) differ")
    if bad.any():
        bi = tuple(int(i) for i in np.argwhere(bad)[0])
        pytest.fail(f"{cid}: {int(bad.sum())} element(s) differ; first at (b, group, physical row, lane)={bi}: got {got[bi]:#06x}, "
                    f"want {want.view(np.uint16)[bi]:#06x}")


# ------------------------------------------------------------------------------------------------------------ fp32 Generator convs
@pytest.mark.parametrize("cid,Cc,K,dil,T,B,res,acc", KC.CONV1D_CASES, ids=[c[0] for c in KC.CONV1D_CASES])
def test_conv1d_c4(cid, Cc, K, dil, T, B, res, acc):
    """resblock conv: (conv(lrelu_0.1(x)) + bias [+ residual] [+ old output]) * out_scale, whole output"""
    g = _rng(cid)
    scale = 1.0 / 3 if acc else 1.0
    x = g.standard_normal((B, Cc, T)).astype(np.float32)
    w = (g.standard_normal((Cc, Cc, K)) / np.sqrt(Cc * K)).astype(np.float32)
    bias = (0.5 * g.standard_normal(Cc)).astype(np.float32)
    r = g.standard_normal((B, Cc, T)).astype(np.float32) if res else None
    y_old = g.standard_normal((B, Cc, T)).astype(np.float32) if acc else np.full((B, Cc, T), np.nan, np.float32)
    y0 = KH.to_c4(y_old)
    run = lambda: conv1d_window(B, T, Cc, Cc, K, dil, 0.1, w, bias, KH.to_c4(x), KH.to_c4(r) if res else None, acc, scale, 0, -1, y0)
    r1 = run()
    _check_run(cid, r1, run())
    ref = R.tc_conv(x, w, bias, op=None, dil=dil, in_slope=0.1, res=r, res_mode=1 if res else 0, y_old=y_old if acc else None,
                    out_scale=scale)
    tile = "128x64" if KC.conv1d_big_tile(T, Cc, B) else "16x16 split-4"
    got = KH.from_c4(r1[0], B, Cc, T).astype(np.float64)
    report(cid, f"k_conv1d_c4<K={K}> tile {tile}", np.abs(got - ref["ref"]), ref["tol"], ref["mag"], np.ones(got.shape, bool), "(b, c, t)")


@pytest.mark.parametrize("cid,K,u,Co,T", KC.CONVT_CASES, ids=[c[0] for c in KC.CONVT_CASES])
def test_convT_c4(cid, K, u, Co, T):
    """upsampling: ConvTranspose1d(lrelu_0.1(x), stride u, padding (K - u) / 2) + bias, whole output"""
    g = _rng(cid)
    Ci, B = 2 * Co, 2
    x = g.standard_normal((B, Ci, T)).astype(np.float32)
    w = (g.standard_normal((Ci, Co, K)) / np.sqrt(Ci * K / u)).astype(np.float32)
    bias = (0.5 * g.standard_normal(Co)).astype(np.float32)
    y0 = KH.to_c4(np.full((B, Co, T * u), np.nan, np.float32))
    run = lambda: convT_window(B, T, Ci, Co, K, u, w, bias, KH.to_c4(x), 0, -1, y0)
    r1 = run()
    _check_run(cid, r1, run())
    acc, mag = R.conv_transpose1d(R.lrelu32(x, 0.1), w, u)
    b64 = bias.astype(np.float64)[None, :, None]
    ref, mag = acc + b64, mag + np.abs(b64)
    got = KH.from_c4(r1[0], B, Co, T * u).astype(np.float64)
    report(cid, f"k_convT_c4 grid=({-(-T * u // 128)},{-(-Co // 64)},{B})", np.abs(got - ref), 1e-5 * mag + 1e-6, mag, np.ones(got.shape, bool),
           "(b, c, n)")
