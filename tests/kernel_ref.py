"""Float64 references of the tensor-core kernels, written from their documented semantics (TcEpi / G2Epi in csrc/tc_conv.cuh and
csrc/tc_gen.cuh, AttnParams in csrc/tc_attn.cuh) and the reference model, not from the kernel code.

Operands are rounded exactly as the kernels round them, so the only difference left is fp32 accumulation order:
  * TF32: round to nearest, ties away from zero, on the bit pattern ((u + 0x1000) & 0xffffe000, finite values only);
  * FP16: round to nearest even, saturating at +-65504;
  * weights as the packers round them, activations after the leaky-relu (fp32 multiply) and the input mask.
Every conv reference returns `ref` and `mag`, the float64 sum of |term| over every term of each output element (|a*w| products, bias,
residual, old output): the tests bound |got - ref| per element by a multiple of `mag`.

Layouts here are plain [B][C][T] (channels, then time); tests/kernel_harness.py converts to and from the device layouts.
"""
import numpy as np

F16_MAX = 65504.0


def tf32(a):
    """fp32 -> TF32 (round to nearest, ties away from zero), as the packers and the operand prologue round."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    u = a.view(np.uint32)
    finite = (u & np.uint32(0x7F800000)) != np.uint32(0x7F800000)
    r = np.where(finite, (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000), u).astype(np.uint32)
    return r.view(np.float32)


def f16(a):
    """fp32 -> fp16 (round to nearest even, saturating) -> fp32."""
    a = np.asarray(a, dtype=np.float32)
    return np.clip(a, -F16_MAX, F16_MAX).astype(np.float16).astype(np.float32)


def round_op(a, kind):
    return {"tf32": tf32, "f16": f16, None: lambda v: np.asarray(v, np.float32)}[kind](a)


def lrelu32(x, slope):
    """leaky relu in fp32 arithmetic (x * slope rounded to fp32, as the kernels compute it)."""
    x = np.asarray(x, np.float32)
    return np.where(x > 0, x, x * np.float32(slope)).astype(np.float32)


def unlrelu10(a):
    """inverse of lrelu(., 0.1) on a stored Generator activation (a >= 0 ? a : 10 a), fp32."""
    a = np.asarray(a, np.float32)
    return np.where(a >= 0, a, a * np.float32(10.0)).astype(np.float32)


def conv1d(x, w, dil=1):
    """Same-padded dilated Conv1d without bias: x [B][Cin][T], w [Cout][Cin][K] (K odd), pad (K-1)/2*dil.
    Returns (out, mag) in float64, mag = sum |w||x| over the terms of each output."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    B, Cin, T = x.shape
    K = w.shape[2]
    pad = (K - 1) // 2 * dil
    xp = np.zeros((B, Cin, T + 2 * pad))
    xp[:, :, pad:pad + T] = x
    out = np.zeros((B, w.shape[0], T))
    mag = np.zeros_like(out)
    for j in range(K):
        xs = xp[:, :, j * dil:j * dil + T]
        out += np.matmul(w[None, :, :, j], xs)
        mag += np.matmul(np.abs(w[None, :, :, j]), np.abs(xs))
    return out, mag


def conv_transpose1d(x, wT, u):
    """ConvTranspose1d(stride u, padding (K-u)/2) without bias: x [B][Cin][T], wT [Cin][Cout][K] -> [B][Cout][T*u], plus mag.
    out[n] = sum over (i, j) with n = i*u - p + j of x[i] wT[j]."""
    x = np.asarray(x, np.float64)
    wT = np.asarray(wT, np.float64)
    B, Cin, T = x.shape
    Cout, K = wT.shape[1], wT.shape[2]
    p = (K - u) // 2
    L = T * u
    out = np.zeros((B, Cout, L + K + u))
    mag = np.zeros_like(out)
    for j in range(K):
        # inputs i land on n = i*u + (j - p); shift by p so every index is >= 0
        c = np.matmul(wT[None, :, :, j].transpose(0, 2, 1), x)
        m = np.matmul(np.abs(wT[None, :, :, j]).transpose(0, 2, 1), np.abs(x))
        out[:, :, j:j + T * u:u] += c
        mag[:, :, j:j + T * u:u] += m
    return out[:, :, p:p + L], mag[:, :, p:p + L]


def _mask_rows(B, T, lens):
    """[B][1][T] bool: t < lens[b]"""
    return (np.arange(T)[None, :] < np.asarray(lens)[:, None])[:, None, :]


def tc_conv(x, w, bias, *, op="tf32", u=0, dil=1, in_slope=1.0, in_mask=False, lens=None, in_f16=False, skip_xform=False,
            bias_b=None, res=None, res_mode=0, y_old=None, relu=False, out_scale=1.0, out_mask=False, out_tf32=False, out_f16=False,
            gate=False, ln=None):
    """tc_conv1d (TcEpi semantics).  x: the Cin input channels [B][Cin][T] (fp32 values; already the 16-bit / TF32 operand when in_f16 /
    skip_xform), w: [Cout][Cin][K] or, with u > 0, the ConvTranspose weight [Cin][Cout][K].  res / y_old: [B][Cout][T_out] slices.
    Returns dict(ref, mag, tol) over the Cout output channels ([B][Cout/2][T] with the gate), tol = the per-element bound."""
    x = np.asarray(x, np.float32)
    B, Cin, T = x.shape
    if in_f16 or skip_xform:
        xa = x
    else:
        xa = x * _mask_rows(B, T, lens) if in_mask else x
        xa = round_op(lrelu32(xa, in_slope), op)
    wr = round_op(w, op)
    if u:
        acc, mag = conv_transpose1d(xa, wr, u)
    else:
        acc, mag = conv1d(xa, wr, dil)
    To = acc.shape[2]
    b64 = np.asarray(bias, np.float64)[None, :, None]
    v = acc + b64
    mag = mag + np.abs(b64)
    if bias_b is not None:
        bb = np.asarray(bias_b, np.float64)[:, :, None]
        v = v + bb
        mag = mag + np.abs(bb)
    if res_mode:
        r = np.asarray(res, np.float64)
        v = v + r if res_mode == 1 else r - v
        mag = mag + np.abs(r)
    if y_old is not None:
        v = v + np.asarray(y_old, np.float64)
        mag = mag + np.abs(np.asarray(y_old, np.float64))
    if relu:
        v = np.maximum(v, 0.0)
    # accumulation bound of the pre-scale value v: fp32 accumulation of products that are exact in fp32 (11-bit x 11-bit significands),
    # error <= (additions in the longest chain) * 2^-24 * mag; 1e-5 * mag covers ~170 chained additions at worst-case alignment, and a
    # dropped tap / channel group / row moves an element by ~mag / n (n <= 2816 terms) -- far above it.  1e-6 absolute for tiny mags.
    # Measured on an H100 80GB HBM3 (400 W) over the 307 fp32-output cases of tests/test_kernels_gpu.py: worst err / mag 2.7e-6.
    e = 1e-5 * mag + 1e-6
    keep = _mask_rows(B, To, lens) if out_mask else np.ones((B, 1, To), bool)
    s = float(out_scale)
    if ln is not None:
        g, beta = (np.asarray(a, np.float64) for a in ln)
        mu = v.mean(axis=1, keepdims=True)
        var = ((v - mu) ** 2).mean(axis=1, keepdims=True)
        rstd = 1.0 / np.sqrt(var + 1e-5)
        xhat = (v - mu) * rstd
        ref = xhat * g[None, :, None] + beta[None, :, None]
        # LayerNorm of perturbed inputs: x_c - mean moves by <= e_c + mean(e), the standard deviation by <= 2 max(e), so the output
        # moves by <= rstd |gamma_c| (e_c + mean(e) + 2 |xhat_c| max(e)); plus the tail's own fp32 arithmetic (sums over Cout channels,
        # rsqrtf): 2e-5 relative to |y| + |beta|
        tol = rstd * np.abs(g)[None, :, None] * (e + e.mean(axis=1, keepdims=True) + 2 * np.abs(xhat) * e.max(axis=1, keepdims=True))
        tol = tol + 2e-5 * (np.abs(ref) + np.abs(beta)[None, :, None]) + 1e-6
        ref = np.where(keep, ref, 0.0)
        tol = np.where(keep, tol, 0.0)
        return dict(ref=ref, mag=mag, tol=tol, pre=v)
    if gate:
        a, bsig = v[:, 0::2], v[:, 1::2]
        ref = np.tanh(a) / (1.0 + np.exp(-bsig)) * s
        ref = np.where(keep, ref, 0.0)
        # tanh is 1-Lipschitz, the sigmoid 1/4-Lipschitz, |tanh|, |sigmoid| <= 1; tanhf / expf add a few ulp (1e-6 absolute);
        # the 16-bit store adds 2^-11 |y|
        tol = abs(s) * (e[:, 0::2] + 0.25 * e[:, 1::2]) + 2.0 ** -11 * np.abs(ref) + 1e-6
        tol = np.where(keep, tol, 0.0)
        return dict(ref=ref, mag=mag[:, 0::2] + mag[:, 1::2], tol=tol)
    ref = np.where(keep, v * s, 0.0)
    tol = abs(s) * e
    if out_tf32 or out_f16:
        tol = tol + 2.0 ** -11 * np.abs(ref)  # RN to an 11-bit significand (ties away for TF32, even for fp16): <= 2^-11 relative
    tol = np.where(keep, tol, 0.0)  # masked rows are exact zeros
    return dict(ref=ref, mag=mag, tol=tol)


def g2_conv(a, w, bias, *, u=0, dil=1, bias_b=None, res=None, y_old=None, out_scale=1.0):
    """k_g2_conv (G2Epi semantics) on stored Generator activations a = f16(lrelu_0.1(x)) [B][Cin][T] (the MMA operand itself):
    y = f16(lrelu_0.1(out_scale * (conv(a) + bias [+ bias_b] [+ unlrelu(res)] [+ unlrelu(y_old)]))).  Weights rounded to fp16."""
    wr = f16(w)
    acc, mag = conv_transpose1d(a, wr, u) if u else conv1d(a, wr, dil)
    b64 = np.asarray(bias, np.float64)[None, :, None]
    v = acc + b64
    mag = mag + np.abs(b64)
    if bias_b is not None:
        bb = np.asarray(bias_b, np.float64)[:, :, None]
        v, mag = v + bb, mag + np.abs(bb)
    for extra in (res, y_old):
        if extra is not None:
            r = unlrelu10(extra).astype(np.float64)
            v, mag = v + r, mag + np.abs(r)
    v = v * out_scale
    ref = np.where(v >= 0, v, 0.1 * v)
    # lrelu is 1-Lipschitz: the accumulation bound of tc_conv, scaled, plus the 16-bit store (2^-11 relative)
    tol = abs(out_scale) * (1e-5 * mag + 1e-6) + 2.0 ** -11 * np.abs(ref)
    return dict(ref=ref, mag=mag, tol=tol)


def flow_attn(q, k, v, rel_k, rel_v, lens, window, round_p=True, round_out=True):
    """k_flow_attn: windowed relative-position attention per (batch, head).  q (pre-scaled by 1/sqrt(dk)), k, v: [B][heads][T][dk],
    rel_k / rel_v: [2w+1][dk].  Keys j >= len are excluded; query rows i >= len are zero (the kernel's contract -- the reference
    model's masked softmax gives a uniform distribution there).  round_p: the unnormalised probabilities exp(s - max) are rounded to fp16
    before the P.V product (the kernel feeds them to the tensor cores as fp16); the relative-value weights and the row sum are not.
    Returns [B][heads][T][dk] in float64 (rounded to fp16 when round_out)."""
    q, k, v = (np.asarray(a, np.float64) for a in (q, k, v))
    ek, ev = np.asarray(rel_k, np.float64), np.asarray(rel_v, np.float64)
    B, nh, T, dk = q.shape
    out = np.zeros_like(q)
    nrel = 2 * window + 1
    for b in range(B):
        L = int(min(lens[b], T))
        if L == 0:
            continue
        qb, kb, vb = q[b, :, :L], k[b, :, :L], v[b, :, :L]
        s = np.matmul(qb, kb.transpose(0, 2, 1))  # [h][i][j]
        rel = np.matmul(qb, ek.T)                  # [h][i][r]: q_i . Ek[r], key j = i + r - w
        i = np.arange(L)
        for r in range(nrel):
            j = i + r - window
            ok = (j >= 0) & (j < L)
            s[:, i[ok], j[ok]] += rel[:, i[ok], r]
        e = np.exp(s - s.max(axis=2, keepdims=True))
        l = e.sum(axis=2, keepdims=True)
        ep = f16(e).astype(np.float64) if round_p else e
        o = np.matmul(ep, vb)
        for r in range(nrel):
            j = i + r - window
            ok = (j >= 0) & (j < L)
            o[:, i[ok], :] += e[:, i[ok], j[ok]][:, :, None] * ev[r][None, None, :]
        o = o / l
        out[b, :, :L] = f16(o).astype(np.float64) if round_out else o
    return out
