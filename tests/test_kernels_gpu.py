"""Kernel-level parity of the tensor-core kernels on an H100: tc_conv1d (one-tile / persistent / streamed kernels, TF32 and FP16 operands,
plain and generic epilogues), the fused flow attention k_flow_attn and the Generator conv k_g2_conv, each against the float64 reference
of tests/kernel_ref.py with the kernel's own operand rounding, element by element.  Run: pytest -m gpu tests/test_kernels_gpu.py -v -s

Every case also checks: valid outputs finite, channels / rows the kernel must not write bitwise unchanged, guard regions around the
output intact, the device error flag clear, and a second run bitwise identical.

Tolerances (derivations in kernel_ref.py): fp32 outputs |got - ref| <= 1e-5 mag + 1e-6 (mag = sum of |terms|); outputs rounded to fp16
or TF32 add 2^-11 |ref|; LayerNorm tails bound the pre-normalisation values scaled by rstd |gamma|; attention |err| <= 4e-3 (max|v| +
max|Ev|).  A dropped tap / channel group / row moves an element by ~mag / n with n <= 2816 terms: far above 1e-5 mag."""
import zlib

import numpy as np
import pytest

import kernel_cases as KC
import kernel_harness as KH
import kernel_ref as R
from util import report

pytestmark = pytest.mark.gpu


def _rng(cid):
    return np.random.default_rng(zlib.crc32(cid.encode()))


# ------------------------------------------------------------------------------------------------------------ tc_conv1d
@pytest.mark.parametrize("cid,fam,B,T,lens,sms,expect", KC.conv_cases(), ids=[c[0] for c in KC.conv_cases()])
def test_tc_conv1d(cid, fam, B, T, lens, sms, expect):
    f = KC.FAMILIES[fam]
    g = _rng(cid)
    op = f["op"]
    a = KC.family_args(fam, B, T, lens, sms)
    u, Cin, Cout, K = a.u, a.Cin, a.Cout, a.K
    To = T * max(1, u)
    Cw = Cout // 2 if a.gate else Cout  # output channels the kernel writes
    lens_a = np.asarray(lens, np.int32)
    # ---- inputs
    x = g.standard_normal((B, a.x_C, T)).astype(np.float32)
    if a.in_f16:
        x = R.f16(np.maximum(x, 0.1 * x))
    elif a.skip_xform:
        x = R.tf32(x)
    w = (g.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K / max(1, u))).astype(np.float32)
    bias = (0.5 * g.standard_normal(Cout)).astype(np.float32)
    bias_b = (0.5 * g.standard_normal((B, a.bias_b_stride))).astype(np.float32) if f.get("bias_b") else None
    gamma = (1 + 0.2 * g.standard_normal(Cout)).astype(np.float32) if f.get("ln") else None
    beta = (0.2 * g.standard_normal(Cout)).astype(np.float32) if f.get("ln") else None
    y16 = bool(a.out_f16 or a.gate)
    y_init = g.standard_normal((B, a.y_C, To)).astype(np.float32)  # finite sentinel: channels outside the window stay bitwise
    win = slice(a.cout_off, a.cout_off + Cw)
    if not (a.res_is_y or a.accumulate):
        y_init[:, win] = np.nan
    if y16:
        y_init = R.f16(y_init)
    res = None
    if a.res_mode and not a.res_is_y:
        res = g.standard_normal((B, a.res_C_total, To)).astype(np.float32)
    # ---- reference
    xin = x[:, a.cin_off:a.cin_off + Cin]
    res_win = y_init[:, a.res_c_off:a.res_c_off + Cout] if a.res_is_y else (res[:, a.res_c_off:a.res_c_off + Cout] if res is not None else None)
    ref = R.tc_conv(xin, w, bias, op=op, u=u, dil=a.dil, in_slope=a.in_slope, in_mask=a.in_mask, lens=lens_a, in_f16=a.in_f16,
                    skip_xform=a.skip_xform, bias_b=None if bias_b is None else bias_b[:, :Cout], res=res_win, res_mode=a.res_mode,
                    y_old=y_init[:, win] if a.accumulate else None, relu=a.relu, out_scale=a.out_scale, out_mask=a.out_mask,
                    out_tf32=a.out_tf32, out_f16=a.out_f16, gate=a.gate, ln=(gamma, beta) if f.get("ln") else None)
    # ---- device buffers
    keep = []
    xb = KH.to_c8(x) if a.in_f16 else KH.to_c4(x)
    yb = KH.to_c8(y_init) if y16 else KH.to_c4(y_init)
    for name, arr in (("w", w), ("bias", bias), ("lens", lens_a), ("bias_b", bias_b), ("ln_gamma", gamma), ("ln_beta", beta)):
        if arr is not None:
            arr = np.ascontiguousarray(arr)
            keep.append(arr)
            setattr(a, name, arr.ctypes.data)
        else:
            setattr(a, name, None)
    a.x, a.x_bytes = xb.ctypes.data, xb.nbytes
    if res is not None:
        rb = KH.to_c4(res)
        keep.append(rb)
        a.res, a.res_elems = rb.ctypes.data, rb.size
    if bias_b is not None:
        a.bias_b_elems = bias_b.size
    out1, plan, guard1, err1 = KH.tc_conv1d(a, yb)
    out2, _, guard2, err2 = KH.tc_conv1d(a, yb)
    assert err1 == 0 and err2 == 0, f"{cid}: device error flag raised (barrier timeout); plan {plan}"
    assert guard1 and guard2, f"{cid}: guard region around the output overwritten; plan {plan}"
    if expect:
        got = dict(kind=KH.KIND_NAMES[plan.kind], res_smem=plan.res_smem)
        assert all(got[k] == v for k, v in expect.items()), (cid, expect, str(plan))
    assert out1.tobytes() == out2.tobytes(), f"{cid}: second run not bitwise identical; plan {plan}"
    y = KH.from_c8(out1, B, a.y_C, To) if y16 else KH.from_c4(out1, B, a.y_C, To)
    outside = np.ones(a.y_C, bool)
    outside[win] = False
    yi = KH.from_c8(yb, B, a.y_C, To) if y16 else KH.from_c4(yb, B, a.y_C, To)
    assert np.array_equal(y[:, outside], yi[:, outside]), \
        f"{cid}: channels outside the output window changed; plan {plan}"
    got = y[:, win].astype(np.float64)
    assert np.isfinite(got).all(), f"{cid}: non-finite outputs at (b, c, t)={tuple(int(i) for i in np.argwhere(~np.isfinite(got))[0])}; plan {plan}"
    report(cid, plan, np.abs(got - ref["ref"]), ref["tol"], ref["mag"], np.ones(got.shape, bool), "(b, c, t)")


# ------------------------------------------------------------------------------------------------------------ fused flow attention
H, HEADS, DK, WIN = 192, 2, 96, 4


def _attn_inputs(g, B, T, lens, planted):
    q = (0.3 * g.standard_normal((B, HEADS, T, DK))).astype(np.float32)
    k = g.standard_normal((B, HEADS, T, DK)).astype(np.float32)
    v = g.standard_normal((B, HEADS, T, DK)).astype(np.float32)
    ek = (0.5 * g.standard_normal((2 * WIN + 1, DK))).astype(np.float32)
    ev = (0.5 * g.standard_normal((2 * WIN + 1, DK))).astype(np.float32)
    if planted:
        # q_i = 40 e_c(i): one key (or one band offset) scores ~40 above every other key of row i, so the output is ~ that key's v
        # (+ Ev of its offset): a mis-addressed key, band entry or merge row shows up as an error of order max|v|
        i = np.arange(T)
        q[:] = 0
        k *= 0.05
        ek *= 0.04
        if planted == "keys":  # dominant keys on both sides of the 32-column and 128 / 256-key tile boundaries
            pos = [31, 32, 127, 128, 255, 256]
            c = i % len(pos)
            q[:, :, i, c] = 40.0
            for ci, p in enumerate(pos):
                if p < T:
                    k[:, :, p, ci] = 1.0
        else:  # dominant band offsets -w (channel 0) and +w (channel 1) on every row, so rows at every tile / column boundary
            q[:, :, i, i % 2] = 40.0
            ek[0, 0] = 1.0
            ek[2 * WIN, 1] = 1.0
    return R.f16(q), R.f16(k), R.f16(v), ek, ev


@pytest.mark.parametrize("cid,B,T,lens,ks,planted", KC.attn_cases(), ids=[c[0] for c in KC.attn_cases()])
def test_flow_attention(cid, B, T, lens, ks, planted):
    g = _rng(cid)
    q, k, v, ek, ev = _attn_inputs(g, B, T, lens, planted)
    chan = lambda a: a.transpose(0, 1, 3, 2).reshape(B, H, T)  # [B][heads][T][dk] -> [B][H][T]
    qkv16 = KH.to_c8(np.concatenate([chan(q), chan(k), chan(v)], axis=1))
    att0 = KH.to_c8(np.full((B, H, T), np.nan, np.float32))
    out1, ks_used, guard1, err1 = KH.flow_attn(qkv16, ek, ev, lens, B, T, H, HEADS, WIN, ks, KC.H100_SMS, att0)
    out2, _, guard2, err2 = KH.flow_attn(qkv16, ek, ev, lens, B, T, H, HEADS, WIN, ks, KC.H100_SMS, att0)
    plan = f"k_flow_attn ks={ks_used} grid=({-(-T // 128) * ks_used},{HEADS},{B})"
    assert err1 == 0 and err2 == 0, f"{cid}: device error flag raised; {plan}"
    assert guard1 and guard2, f"{cid}: guard region around the output overwritten; {plan}"
    assert out1.tobytes() == out2.tobytes(), f"{cid}: second run not bitwise identical; {plan}"
    got = KH.from_c8(out1, B, H, T).reshape(B, HEADS, DK, T).transpose(0, 1, 3, 2).astype(np.float64)
    assert np.isfinite(got).all(), f"{cid}: non-finite outputs; {plan}"
    ref = R.flow_attn(q, k, v, ek, ev, lens, WIN)
    # P rounded to fp16 (2^-11 relative per weight: <= 2^-11 max|v| after normalisation) + the fp16 output (2^-11 |out|, |out| <= max|v| +
    # max|Ev|) + fp32 scores / ex2.approx (<< 2^-11): ~1e-3 (max|v| + max|Ev|); 4e-3 leaves 4x margin.  Rows >= len: exact zeros.
    valid = (np.arange(T)[None, :] < np.asarray(lens)[:, None])[:, None, :, None]
    tol = np.where(valid, 4e-3 * (np.abs(v).max() + np.abs(ev).max()), 0.0) * np.ones_like(ref)
    report(cid, plan, np.abs(got - ref), tol, np.full(ref.shape, np.abs(v).max() + np.abs(ev).max()), np.ones(ref.shape, bool),
            "(b, head, t, d)")


# ------------------------------------------------------------------------------------------------------------ Generator conv (H8)
@pytest.mark.parametrize("cid,Cin,Cout,K,dil,u,T,B,res,acc,scale,st,bb,sms,expect", KC.g2_cases(), ids=[c[0] for c in KC.g2_cases()])
def test_g2_conv(cid, Cin, Cout, K, dil, u, T, B, res, acc, scale, st, bb, sms, expect):
    g = _rng(cid)
    To = T * max(1, u)
    act = lambda s: R.f16(R.lrelu32(g.standard_normal(s).astype(np.float32), 0.1))  # stored Generator activations
    a = act((B, Cin, T))
    w = (g.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K / max(1, u))).astype(np.float32)
    bias = g.standard_normal(Cout).astype(np.float32)
    stride = Cout + 40
    bias_b = (0.5 * g.standard_normal((B, stride))).astype(np.float32) if bb else None
    r = act((B, Cout, To)) if res else None
    y_old = act((B, Cout, To)) if acc else None
    xh = KH.to_h8(a, 0.0)
    rh = KH.to_h8(r, 0.0) if res else None
    yh = KH.to_h8(y_old if acc else np.full((B, Cout, To), np.nan, np.float32), np.nan)  # halos NaN: the kernel must zero them
    arrs = [np.ascontiguousarray(v) for v in (w, bias)]
    args = KH.g2_args(B=B, T=T, Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, residual=res, accumulate=acc, out_scale=scale, st_override=st,
                      num_sms=sms, w=arrs[0].ctypes.data, bias=arrs[1].ctypes.data, x=xh.ctypes.data,
                      res=rh.ctypes.data if res else None, bias_b=bias_b.ctypes.data if bb else None,
                      bias_b_elems=bias_b.size if bb else 0, bias_b_stride=stride if bb else 0)
    out1, plan, guard1, err1 = KH.g2_conv(args, yh)
    out2, _, guard2, err2 = KH.g2_conv(args, yh)
    assert err1 == 0 and err2 == 0, f"{cid}: device error flag raised; plan {plan}"
    assert guard1 and guard2, f"{cid}: guard region around the output overwritten; plan {plan}"
    if expect:
        assert KC.g2_key(plan) == expect, (cid, KC.g2_key_name(expect), str(plan))
    assert out1.tobytes() == out2.tobytes(), f"{cid}: second run not bitwise identical; plan {plan}"
    data, halo = KH.h8_data(out1)
    assert (halo == 0).all(), f"{cid}: halo rows of the output not zero after the conv; plan {plan}"
    assert np.isfinite(data).all(), f"{cid}: non-finite outputs; plan {plan}"
    ref = R.g2_conv(a, w, bias, u=u, dil=dil, bias_b=None if bias_b is None else bias_b[:, :Cout], res=r, y_old=y_old, out_scale=scale)
    report(cid, plan, np.abs(data.astype(np.float64) - ref["ref"]), ref["tol"], ref["mag"], np.ones(data.shape, bool), "(b, c, t)")
