"""Case matrix of the kernel tests: every tensor-core conv call shape the engine makes with the default model config (with the engine's
N tile / K chunk), at the edges where tiling goes wrong, plus num_sms values that force each dispatch branch of tc_conv1d.
Shared by tests/test_kernels_cpu.py (dispatch coverage through the host planner) and tests/test_kernels_gpu.py (H100 runs)."""
import numpy as np

import kernel_harness as KH

H, FC, HALF = 192, 768, 96
EDGE_T = [1, 127, 128, 129, 300, 1000]
BIG_SMS, SMALL_SMS, H100_SMS = 100000, 3, 132


def _ragged(T):
    """B = 3 lengths from {T, 1, 127, 128, 129} that fit in T"""
    pool = [t for t in (129, 1, 128, 127) if t < T]
    return [T] + (pool + [T, T])[:2]


# family: shapes + epilogue flags of one engine call.  op: operand type; x16 / y16: the tensor is 16-bit c8.
# small: the kernel tc_conv1d picks at num_sms = 3 (nctas >= 2 * num_sms) -- persist where eligible, else pstream where it fits
FAMILIES = {
    # ---- FP16 flow (generator_precision 3): transformer layers + couplings
    "f16.pre": dict(op="f16", Cin=HALF, Cout=H, K=1, nt=96, kc=32, x_C=2 * HALF, cin_off=HALF, y_C=H, out_mask=1, small="pstream"),
    "f16.qkv": dict(op="f16", Cin=H, Cout=3 * H, K=1, nt=96, kc=64, out_f16=1, y16=1, small="one-tile"),  # K chunk 64: rings do not fit pstream
    # conv_o + residual + LayerNorm: at 192 channels the staged residual tile (96 KB) does not fit next to the accumulator image and the
    # rings, so the residual is always pre-loaded into the accumulator (res_smem = 0 at any SM count)
    "f16.conv_o_ln": dict(op="f16", Cin=H, Cout=H, K=1, nt=H, kc=64, in_f16=1, x16=1, res_mode=1, res_is_y=1, ln=1, small="one-tile",
                          big_res_smem=0),
    "f16.ffn1": dict(op="f16", Cin=H, Cout=FC, K=3, nt=128, kc=64, relu=1, in_mask=1, out_mask=1, out_f16=1, y16=1, small="one-tile"),
    "f16.ffn2": dict(op="f16", Cin=FC, Cout=H, K=3, nt=32, kc=64, in_f16=1, x16=1, out_mask=1, small="one-tile"),
    "f16.post": dict(op="f16", Cin=H, Cout=HALF, K=1, nt=48, kc=32, y_C=2 * HALF, cout_off=HALF, res_mode=2, res_is_y=1, out_mask=1,
                     small="one-tile"),
    "f16.post_wn": dict(op="f16", Cin=H, Cout=HALF, K=1, nt=48, kc=32, y_C=2 * HALF, cout_off=0, res_mode=2, res_is_y=1, out_mask=1,
                        in_mask=1, small="one-tile"),
    "f16.wn_in": dict(op="f16", Cin=H, Cout=2 * H, K=5, nt=128, kc=32, gate=1, bias_b=1, y16=1, y_C=H, small="pstream"),
    "f16.wn_res": dict(op="f16", Cin=H, Cout=H, K=1, nt=96, kc=32, in_f16=1, x16=1, res_mode=1, res_is_y=1, out_mask=1, small="one-tile"),
    "f16.wn_skip": dict(op="f16", Cin=H, Cout=H, K=1, nt=96, kc=32, in_f16=1, x16=1, accumulate=1, small="one-tile"),
    # ---- TF32 flow (generator_precision 1)
    "tf32.pre": dict(op="tf32", Cin=HALF, Cout=H, K=1, nt=96, kc=32, x_C=2 * HALF, cin_off=0, y_C=H, out_mask=1, small="pstream"),
    "tf32.qkv": dict(op="tf32", Cin=H, Cout=3 * H, K=1, nt=96, kc=64, out_tf32=1, small="pstream"),
    "tf32.conv_o": dict(op="tf32", Cin=H, Cout=H, K=1, nt=48, kc=64, skip_xform=1, res_mode=1, small="one-tile"),
    "tf32.post": dict(op="tf32", Cin=H, Cout=HALF, K=1, nt=48, kc=32, y_C=2 * HALF, cout_off=HALF, res_mode=2, res_is_y=1, out_mask=1,
                      small="one-tile"),
    # ---- TF32 Generator (generator_precision 1): conv_pre, upsampling (polyphase ConvTranspose1d)
    "tf32.conv_pre": dict(op="tf32", Cin=H, Cout=512, K=7, nt=128, kc=32, bias_b=1, in_mask=1, small="pstream"),
    "tf32.ups0": dict(op="tf32", Cin=512, Cout=256, K=16, u=8, nt=128, kc=32, in_slope=0.1, small="pstream"),
    "tf32.ups2": dict(op="tf32", Cin=128, Cout=64, K=8, u=2, nt=128, kc=32, in_slope=0.1, small="pstream"),
    "tf32.ups3": dict(op="tf32", Cin=64, Cout=32, K=2, u=2, nt=128, kc=32, in_slope=0.1, small="pstream"),
    "tf32.ups4": dict(op="tf32", Cin=32, Cout=16, K=2, u=2, nt=128, kc=32, in_slope=0.1, small="persist"),
    # ---- FP16 operand kernels of narrow layers (no default-config engine call: they complete the kernel x operand x epilogue matrix)
    "f16.narrow": dict(op="f16", Cin=32, Cout=32, K=7, nt=0, kc=32, in_slope=0.1, res_mode=1, small="persist"),
    "f16.narrow_gen": dict(op="f16", Cin=32, Cout=32, K=3, nt=0, kc=32, relu=1, bias_b=1, small="persist"),
    # LayerNorm tail with the residual tile staged in shared memory by TMA (fits at <= 96 channels), out_mask on ragged rows
    "f16.ln96": dict(op="f16", Cin=H, Cout=HALF, K=1, nt=HALF, kc=32, in_f16=1, x16=1, res_mode=1, res_is_y=1, ln=1, out_mask=1,
                     small="one-tile", big_res_smem=1),
}
# TF32 Generator resblocks: convs1 (K, dilation d, lrelu 0.1 input) and convs2 (K, dilation 1, + residual; the last one of a chain
# accumulates into the MRF running sum, scaled by 1/3 for the last kernel size)
for _C in (256, 128, 64, 32, 16):
    _small = "persist" if _C <= 32 else "pstream"
    for _K, _d in ((3, 1), (7, 3), (11, 5)):
        FAMILIES[f"tf32.rb{_C}.c1_k{_K}d{_d}"] = dict(op="tf32", Cin=_C, Cout=_C, K=_K, dil=_d, nt=0, kc=32, in_slope=0.1, small=_small)
    FAMILIES[f"tf32.rb{_C}.c2_k7"] = dict(op="tf32", Cin=_C, Cout=_C, K=7, nt=0, kc=32, in_slope=0.1, res_mode=1, small=_small)
    FAMILIES[f"tf32.rb{_C}.c2_k11_acc"] = dict(op="tf32", Cin=_C, Cout=_C, K=11, nt=0, kc=32, in_slope=0.1, res_mode=1, accumulate=1,
                                               out_scale=1.0 / 3, small=_small)


def _is_resblock(name):
    return ".rb" in name


def conv_cases():
    """(id, family name, B, T, lens, num_sms, expected plan or None)"""
    out = []
    for name, f in FAMILIES.items():
        ts = [1, 129, 1000] if _is_resblock(name) or name.startswith("tf32.ups0") else EDGE_T
        for T in ts:
            out.append((f"{name}-T{T}-B1", name, 1, T, [T], H100_SMS, None))
        for T in ([300] if _is_resblock(name) else [300, 1000]):
            out.append((f"{name}-T{T}-B3", name, 3, T, _ragged(T), H100_SMS, None))
        # forced dispatch: a huge SM count -> one tile per CTA (LayerNorm: residual staged in shared memory); 3 SMs -> persistent kernels
        T = 1000 if f.get("small") == "persist" else 300
        out.append((f"{name}-T{T}-B3-sms{BIG_SMS}", name, 3, T, _ragged(T), BIG_SMS, dict(kind="one-tile", res_smem=f.get("big_res_smem", 0))))
        exp = dict(kind=f["small"])
        if f.get("ln"):
            exp["res_smem"] = 0
        out.append((f"{name}-T{T}-B3-sms{SMALL_SMS}", name, 3, T, _ragged(T), SMALL_SMS, exp))
    return out


def family_args(name, B, T, lens, num_sms):
    """TcArgs of a case without data pointers (host planning)"""
    f = FAMILIES[name]
    u = f.get("u", 0)
    Cin, Cout = f["Cin"], f["Cout"]
    return KH.tc_args(B=B, T=T, Cin=Cin, Cout=Cout, K=f["K"], u=u, x_C=f.get("x_C", Cin), y_C=f.get("y_C", Cout // 2 if f.get("gate") else Cout),
                      nt=f["nt"], kc=f["kc"], f16=int(f["op"] == "f16"), num_sms=num_sms, in_slope=f.get("in_slope", 1.0),
                      in_mask=f.get("in_mask", 0), relu=f.get("relu", 0), res_mode=f.get("res_mode", 0),
                      res_C_total=f.get("y_C", Cout) if f.get("res_mode") else 0, res_c_off=f.get("cout_off", 0) if f.get("res_mode") else 0,
                      accumulate=f.get("accumulate", 0), out_scale=f.get("out_scale", 1.0), out_mask=f.get("out_mask", 0),
                      bias_b_stride=(Cout * max(1, u)) + 40 if f.get("bias_b") else 0, cin_off=f.get("cin_off", 0), cout_off=f.get("cout_off", 0),
                      dil=f.get("dil", 1), out_tf32=f.get("out_tf32", 0), skip_xform=f.get("skip_xform", 0), in_f16=f.get("in_f16", 0),
                      out_f16=f.get("out_f16", 0), gate=f.get("gate", 0), res_is_y=f.get("res_is_y", 0),
                      lens=1 if lens is not None else None, bias_b=1 if f.get("bias_b") else None,
                      ln_gamma=1 if f.get("ln") else None, ln_beta=1 if f.get("ln") else None,
                      res=1 if f.get("res_mode") and not f.get("res_is_y") else None)


# ---- fused flow attention: (id, B, T, lens, ks_override, planted)
def attn_cases():
    out = []
    for T in (1, 100, 128, 129, 256, 300, 512, 1000):
        for ks in (0, 1, 2, 4):
            out.append((f"T{T}-ks{ks or 'auto'}", 1, T, [T], ks, None))
    # ragged batch: the short row's query tiles past its length are all zero, and ranks of its tile's cluster get no key tile
    for ks in (0, 2, 4):
        out.append((f"ragged-B2-T512-L512,100-ks{ks or 'auto'}", 2, 512, [512, 100], ks, None))
    out.append(("ragged-B3-T300-L1,129,300-ksauto", 3, 300, [1, 129, 300], 0, None))
    for ks in (1, 2, 4):
        out.append((f"planted-keys-T512-ks{ks}", 1, 512, [512], ks, "keys"))
        out.append((f"planted-band-T512-ks{ks}", 1, 512, [512], ks, "band"))
        out.append((f"planted-keys-B2-T300-L300,257-ks{ks}", 2, 300, [300, 257], ks, "keys"))
    return out


# ---- Generator conv (k_g2_conv): (id, Cin, Cout, K, dil, u, T, B, res, acc, scale, st_override, bias_b)
def g2_cases():
    base = [  # the shape matrix: every tail, edge tiles, both weight modes
        (16, 16, 3, 1, 0, 300, 1, 0, 0, 1.0, 0), (16, 16, 11, 5, 0, 1000, 2, 1, 0, 1.0, 0), (16, 16, 7, 3, 0, 5000, 1, 1, 1, 1 / 3, 0),
        (32, 32, 11, 5, 0, 3000, 1, 1, 0, 1.0, 0), (32, 32, 3, 1, 0, 129, 3, 1, 1, 1.0, 0), (64, 64, 7, 3, 0, 2000, 1, 1, 0, 1.0, 0),
        (64, 64, 11, 1, 0, 700, 2, 0, 0, 1.0, 3), (128, 128, 3, 1, 0, 1000, 1, 1, 0, 1.0, 4), (128, 128, 11, 5, 0, 600, 1, 1, 1, 1 / 3, 2),
        (256, 256, 7, 3, 0, 500, 1, 1, 0, 1.0, 2), (192, 512, 7, 1, 0, 300, 2, 0, 0, 1.0, 0),
        (512, 256, 16, 1, 8, 200, 1, 0, 0, 1.0, 0), (128, 64, 8, 1, 2, 700, 2, 0, 0, 1.0, 0), (32, 16, 8, 1, 2, 3000, 1, 0, 0, 1.0, 0),
    ]
    out = [(f"probe-{i}", *c, 0) for i, c in enumerate(base)]
    # every super-tile override of a streamed and a resident layer, T at the 128-row tile edges
    # (streamed layers hold at most 128 / nt m-tiles of accumulators: MG <= 2 at C = 64)
    for st in (1, 2):
        out.append((f"st{st}-streamed-C64-T1000", 64, 64, 11, 1, 0, 1000, 1, 1, 0, 1.0, st, 0))
    for st in (1, 2, 3, 4, 8):
        out.append((f"st{st}-resident-C32-T3000", 32, 32, 11, 5, 0, 3000, 1, 1, 1, 1 / 3, st, 0))
    for T in (1, 127, 128, 129, 255, 257):
        out.append((f"edge-C64-K11d5-T{T}", 64, 64, 11, 5, 0, T, 2, 1, 1, 1 / 3, 0, 0))
        out.append((f"edge-C16-K3-T{T}", 16, 16, 3, 1, 0, T, 1, 1, 0, 1.0, 0, 0))
    for T in (1, 129, 1000):  # conv_pre with the per-batch (speaker) bias
        out.append((f"conv_pre-bias_b-T{T}", 192, 512, 7, 1, 0, T, 2, 0, 0, 1.0, 0, 1))
    out.append(("ups-K2u2-C64-T129", 64, 32, 2, 1, 2, 129, 1, 0, 0, 1.0, 0, 0))
    return out
