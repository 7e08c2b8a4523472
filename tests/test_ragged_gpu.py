"""Ragged batches on the FP16 Generator (precision fp16 / fp16g): each utterance of a batch runs the Generator at its own length, and
its samples are bit-identical to a B=1 run of it at that length, with zeros past it.  Checked at the Generator entry point
(bv2_generator_ragged against B=1 bv2_generator), at the kernel (one ragged k_g2_conv against B=1 launches, with a canary in the rows
no CTA may write), end to end against the CPU oracle run of each utterance alone, and for the error paths.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.engine import Engine
from util import model_for, rms

pytestmark = pytest.mark.gpu

FP16 = ["fp16", "fp16g"]
TOL_WAV = 1e-3  # waveform RMS against the oracle: the FP16 Generator's bar (test_gpu_parity.py)


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(precision):
        if precision not in cache:
            cfg, sd = model_for(True, 0)
            cache[precision] = Engine(cfg, sd, device="cuda:0", precision=precision)
        return cache[precision]

    yield get
    cache.clear()


# ---------------------------------------------------------------- 1. Generator level, bitwise
EDGES = [1, 2, 13, 127, 128, 129, 255, 256, 257]


def _lengths(case):
    kind, F = case
    if kind == "edges":
        return [L for L in EDGES if L < F] + [F]
    r = np.random.default_rng(F)
    return [int(v) for v in r.integers(1, F + 1, size=32)]


GEN_CASES = [("edges", 300), ("edges", 520), ("random32", 400), ("random32", 90)]


def _scales(cfg):
    """M-axis rows per frame of every k_g2_conv layer of kernel_cases.g2_layers (a ConvTranspose's M axis is its input)"""
    import kernel_cases as KC
    rates = list(cfg.upsample_rates)
    out = []
    for f in KC.g2_layers(cfg):
        n = f["name"]
        stage = -1 if n == "conv_pre" else int(n[3:]) - 1 if n.startswith("ups") else int(n[1:n.index("_")])
        out.append((f, int(np.prod(rates[:stage + 1]))))
    return out


def _plans(cfg, B, F, lengths):
    """distinct k_g2_conv plans of the ragged batch and of the B=1 runs it is compared with"""
    import kernel_cases as KC
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    batch, alone = set(), set()
    for f, s in _scales(cfg):
        batch.add(KC.g2_key_name(KC.g2_key(KC.g2_layer_plan(f, F * s, B, sms))))
        for L in sorted(set(lengths)):
            alone.add(KC.g2_key_name(KC.g2_key(KC.g2_layer_plan(f, L * s, 1, sms))))
    return batch, alone


def _zg(cfg, B, F, seed):
    z, g = synth.synthetic_generator_inputs(cfg, B, F, seed=seed)
    return z, g


@pytest.mark.parametrize("case", GEN_CASES, ids=[f"{k}-F{F}" for k, F in GEN_CASES])
@pytest.mark.parametrize("precision", FP16)
def test_generator_ragged_bitwise_vs_alone(engines, precision, case):
    eng = engines(precision)
    cfg, hop = eng.cfg, eng.cfg.hop
    lengths = _lengths(case)
    B, F = len(lengths), case[1]
    batch, alone = _plans(cfg, B, F, lengths)
    print(f"[{precision} B={B} F={F}] ragged-batch plans: {sorted(batch)}\n  B=1 plans: {sorted(alone)}")
    assert any(p.endswith("-res") for p in batch | alone) and any(p.endswith("-str") for p in batch | alone)
    z, g = _zg(cfg, B, F, seed=F)
    o = eng.generator(z, g, lengths=lengths).cpu()
    for b, L in enumerate(lengths):
        ref = eng.generator(z[b:b + 1, :, :L].contiguous(), g[b:b + 1]).cpu()
        assert torch.equal(o[b, :, :L * hop], ref[0]), f"item {b} (L={L}) differs from its B=1 run"
        assert (o[b, :, L * hop:] == 0).all(), f"item {b} (L={L}) has non-zero samples past its length"


@pytest.mark.parametrize("precision", FP16)
def test_generator_ragged_full_lengths_equal_padded(engines, precision):
    eng = engines(precision)
    B, F = 5, 333
    z, g = _zg(eng.cfg, B, F, seed=7)
    padded = eng.generator(z, g).cpu()
    assert torch.equal(eng.generator(z, g, lengths=[F] * B).cpu(), padded)


def test_generator_ragged_lengths_are_clamped(engines):
    eng = engines("fp16")
    F = 200
    z, g = _zg(eng.cfg, 4, F, seed=8)
    got = eng.generator(z, g, lengths=[0, -7, F + 1000, 3]).cpu()
    assert torch.equal(got, eng.generator(z, g, lengths=[1, 1, F, 3]).cpu())


# ---------------------------------------------------------------- 2. kernel level: one ragged k_g2_conv
CANARY = np.uint16(0x7E5A)  # a NaN no kernel produces
KCASES = {  # name: (Cin, Cout, K, u, dil, residual, accumulate, out_scale, T (M-axis rows), lens (frames), lens_scale)
    "ups_u2": (128, 64, 8, 2, 1, 0, 0, 1.0, 160, [1, 100, 160], 1),
    "res_streamed": (256, 256, 3, 0, 1, 1, 0, 1.0, 300, [1, 64, 150], 2),
    "acc_scale": (64, 64, 5, 0, 1, 1, 1, 1.0 / 3, 300, [2, 129, 300], 1),
    "dil5": (32, 32, 3, 0, 5, 0, 0, 1.0, 400, [1, 3, 100], 4),
}


@pytest.mark.parametrize("name", list(KCASES))
def test_g2_conv_ragged_kernel(name):
    import kernel_harness as KH
    import ragged_harness as RH
    Cin, Cout, K, u, dil, res, acc, scale, T, lens, s = KCASES[name]
    B, uu = len(lens), max(u, 1)
    pl, pr = KH.g2_pads()
    To = T * uu
    lim = [min(T, L * s) for L in lens]
    r = np.random.default_rng(len(name))
    w = (r.standard_normal((Cin, Cout, K) if u else (Cout, Cin, K)) / np.sqrt(Cin * K)).astype(np.float32)
    bias = (0.1 * r.standard_normal(Cout)).astype(np.float32)
    # input: item b's rows, then the zero rows its producer leaves, then stale workspace (random) that no kept output may read
    x = r.standard_normal((B, Cin, T)).astype(np.float32)
    for b, m in enumerate(lim):
        x[b, :, m:m + pr] = 0.0
    xh = KH.to_h8(x)
    resh = KH.to_h8(r.standard_normal((B, Cout, To)).astype(np.float32)) if res else None
    old = r.standard_normal((B, Cout, To)).astype(np.float32)
    y0 = KH.to_h8(old) if acc else np.full((B, Cout // 8, pl + To + pr, 8), 0, np.float16)
    y0v = y0.view(np.uint16)
    for b, m in enumerate(lim):
        y0v[b, :, pl + (m * uu if acc else 0):, :] = CANARY  # everything the kernel may not read or must write
    kw = dict(Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, residual=res, accumulate=acc, out_scale=scale, num_sms=132,
              w=w.ctypes.data, bias=bias.ctypes.data)
    y, plan, guard, err = RH.g2_conv_ragged(KH.g2_args(B=B, T=T, x=xh.ctypes.data, res=None if resh is None else resh.ctypes.data, **kw),
                                            lens, s, y0)
    print(f"{name}: {plan} lims {lim}")
    assert guard and err == 0
    yv = y.view(np.uint16)
    for b, m in enumerate(lim):
        mo = m * uu
        xb = np.ascontiguousarray(xh[b:b + 1, :, :pl + m + pr]).copy()
        xb[:, :, pl + m:] = 0
        rb = None if resh is None else np.ascontiguousarray(resh[b:b + 1, :, :pl + mo + pr])
        yb0 = np.ascontiguousarray(y0[b:b + 1, :, :pl + mo + pr]).copy()
        yb0.view(np.uint16)[:, :, pl + mo:, :] = CANARY
        ref, _, g1, e1 = KH.g2_conv(KH.g2_args(B=1, T=m, x=xb.ctypes.data, res=None if rb is None else rb.ctypes.data, **kw), yb0)
        assert g1 and e1 == 0
        assert np.array_equal(yv[b, :, :pl + mo], ref.view(np.uint16)[0, :, :pl + mo]), f"{name} item {b}: rows < {mo} (or the lead halo)"
        assert (yv[b, :, pl + mo:pl + mo + pr] == 0).all(), f"{name} item {b}: rows [{mo}, {mo + pr}) not zero"
        assert (yv[b, :, pl + mo + pr:] == CANARY).all(), f"{name} item {b}: rows past {mo + pr} were written"


# ---------------------------------------------------------------- 3. end to end against the CPU oracle
E2E_LENGTHS = [64, 12, 40, 57, 25, 33, 6, 48]


@pytest.fixture(scope="module")
def e2e_case():
    """B=8 batch with spread lengths, and the oracle's run of each utterance alone (same noise slices); the batch's durations are
    teacher-forced to the oracle's so that every utterance has the frames it has alone"""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    B, T = len(E2E_LENGTHS), max(E2E_LENGTHS)
    inp = synth.synthetic_inputs(cfg, E2E_LENGTHS, [i % 3 for i in range(B)], seed=61)
    nw, nz = synth.synthetic_noise(cfg, B, T, 1024, seed=61)
    kw = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)
    alone, w_ceil = [], torch.zeros(B, T)
    for b, t in enumerate(E2E_LENGTHS):
        one = {k: (v[b:b + 1, ..., :t] if v.dim() >= 2 else v[b:b + 1]) for k, v in inp.items()}
        one["x_lengths"] = torch.tensor([t])
        st = O.infer(sd, cfg, **one, noise_w=nw[b:b + 1, :, :t], noise_z=nz[b:b + 1], return_stages=True, **kw)
        alone.append(st)
        w_ceil[b, :t] = torch.as_tensor(st["w_ceil"]).reshape(-1)[:t]
    return inp, nw, nz, kw, alone, w_ceil


def _begin(eng, inp, nw, kw, w_ceil):
    return eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                           inp["en_bert"], nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"], w_ceil_override=w_ceil)


@pytest.mark.parametrize("precision", FP16)
def test_infer_ragged_vs_oracle_alone(engines, precision, e2e_case):
    inp, nw, nz, kw, alone, w_ceil = e2e_case
    eng = engines(precision)
    hop = eng.cfg.hop
    B, T = inp["x"].shape
    ylen, F = _begin(eng, inp, nw, kw, w_ceil)
    assert ylen.tolist() == [int(st["y_lengths"][0]) for st in alone]
    eng.reserve(B, T, F)
    l0 = eng.launch_count
    o_pad, _, ym_pad, aux_pad = eng.infer_finish(B, T, F, nz, kw["noise_scale"], want_attn=False)
    torch.cuda.synchronize()
    n_pad = eng.launch_count - l0
    o_pad, ym_pad, aux_pad = o_pad.cpu(), ym_pad.cpu(), [a.cpu() for a in aux_pad]
    grows = eng.workspace_grows
    _begin(eng, inp, nw, kw, w_ceil)
    l0 = eng.launch_count
    o, _, ym, aux = eng.infer_finish(B, T, F, nz, kw["noise_scale"], want_attn=False, ragged=True)
    torch.cuda.synchronize()
    assert eng.launch_count - l0 == n_pad
    assert eng.workspace_grows == grows
    o, ym, aux = o.cpu(), ym.cpu(), [a.cpu() for a in aux]
    assert torch.equal(ym, ym_pad) and all(torch.equal(a, p) for a, p in zip(aux, aux_pad))  # y_mask, z, z_p, m_p, logs_p
    for b, st in enumerate(alone):
        n = int(ylen[b]) * hop
        ref = torch.as_tensor(st["o"]).reshape(-1)
        assert ref.numel() == n
        e, e_pad = rms(o[b, 0, :n], ref), rms(o_pad[b, 0, :n], ref)
        print(f"[{precision}] item {b}: frames {int(ylen[b])}, waveform RMS vs oracle alone: ragged {e:.2e}, padded {e_pad:.2e}")
        assert e < TOL_WAV
        assert (o[b, 0, n:] == 0).all()
    # 16-bit PCM: the ragged float waveform converted per utterance
    _begin(eng, inp, nw, kw, w_ceil)
    o16, _, _, _ = eng.infer_finish(B, T, F, nz, kw["noise_scale"], want_attn=False, pcm16=True, ragged=True)
    want = eng.wave_to_pcm16(o.to(eng.device), torch.as_tensor(ylen * hop))
    assert torch.equal(o16.cpu(), want.cpu())


# ---------------------------------------------------------------- 4. errors
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_ragged_rejected_by_fp32_and_tf32(precision):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, sd = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=cfg.n_speakers, gin_channels=512, precision=precision, init_seed=0).to("cuda")
    inp = synth.synthetic_inputs(cfg, [20, 9], [0, 1], seed=3)
    args = [inp[k].cuda() for k in ("x", "x_lengths", "sid", "tone", "language", "bert", "ja_bert", "en_bert")]
    with pytest.raises(ValueError):
        net.infer(*args, ragged=True)
    assert torch.isfinite(net.infer(*args)[0]).all()  # the module still serves
    # the engine itself: BV2_ERR_ARG (ValueError) from both ragged entry points, then the next call is served
    eng = net._engine(torch.device("cuda:0"))
    B, T = inp["x"].shape
    nw, nz = synth.synthetic_noise(cfg, B, T, 512, seed=3)
    _, F = eng.infer_begin(*args, nw, 0.8, 1.0, 0.0)
    with pytest.raises(ValueError):
        eng.infer_finish(B, T, F, nz, 0.667, want_attn=False, ragged=True)
    z, g = _zg(cfg, 2, 50, seed=4)
    with pytest.raises(ValueError):
        eng.generator(z, g, lengths=[10, 50])
    _, F = eng.infer_begin(*args, nw, 0.8, 1.0, 0.0)
    o, _, _, _ = eng.infer_finish(B, T, F, nz, 0.667, want_attn=False)
    assert torch.isfinite(o).all()
    assert torch.isfinite(eng.generator(z, g)).all()
