"""GPU parity: the CUDA engine (through the C ABI / drop-in class) against the CPU oracle and against the
committed reference-generated goldens.  Run on an H100: pytest -m gpu."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bert_vits2_b200 import synth
from bert_vits2_b200.spec import ModelConfig
from util import GOLDEN_CASES, case_inputs, load_golden, model_for, rms

pytestmark = pytest.mark.gpu

# Stated tolerances (fp32 path: different summation order only; tf32 / fp16 paths: 11-bit-significand operands, fp32 accumulate)
TOL_FP32 = 2e-4        # max-abs per stage, pre-Generator stages (values are O(1))
TOL_WAV_FP32 = 2e-5    # waveform RMS, fp32 Generator
TOL_WAV_TF32 = 1e-3    # waveform RMS, tf32 / fp16-operand wgmma Generator (north_star bar)
PRECISIONS = ["fp32", "tf32", "fp16g", "fp16"]


@pytest.fixture(scope="module")
def engines():
    from bert_vits2_b200.engine import Engine
    cache = {}

    def get(tflow: bool, precision: str):
        key = (tflow, precision)
        if key not in cache:
            cfg, sd = model_for(tflow, 0)
            cache[key] = Engine(cfg, sd, device="cuda:0", precision=precision)
        return cache[key]

    yield get
    cache.clear()


def _oracle_stages(meta):
    from oracle import vits2_oracle as O
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)
    return cfg, sd, inp, nw, nz, kw, st


@pytest.mark.parametrize("precision", PRECISIONS)  # every engine runs this stage on FP32 FMA (it feeds ceil(durations))
@pytest.mark.parametrize("name", ["tflow_b1", "tflow_b3"])
def test_text_encoder_stage(engines, name, precision):
    meta, gold = load_golden(name)
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    eng = engines(True, precision)
    x, m, logs = eng.text_encoder(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"],
                                  inp["ja_bert"], inp["en_bert"])
    for got, key in ((x, "x"), (m, "m_p_tok"), (logs, "logs_p_tok")):
        err = float((got.cpu() - gold[key]).abs().max())
        print(f"[{name}/{precision}] {key} max-abs err {err:.2e}")
        assert err < TOL_FP32, (key, err)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", ["tflow_b1", "tflow_b3"])
def test_duration_stage(engines, name, precision):
    meta, gold = load_golden(name)
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    eng = engines(True, precision)
    a, b = eng.duration(gold["x"], inp["x_lengths"], inp["sid"], nw, kw["noise_scale_w"])
    assert float((a.cpu() - gold["logw_sdp"]).abs().max()) < TOL_FP32
    assert float((b.cpu() - gold["logw_dp"]).abs().max()) < TOL_FP32


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_flow_stage(engines, name):
    meta, gold = load_golden(name)
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    eng = engines(meta["use_transformer_flow"], "fp32")
    z = eng.flow_reverse(gold["z_p"], gold["y_lengths"], inp["sid"])
    err = float((z.cpu() - gold["z"]).abs().max())
    assert err < TOL_FP32, err


@pytest.mark.parametrize("precision", PRECISIONS)
def test_generator_stage(engines, precision):
    meta, gold = load_golden("tflow_b3")
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    eng = engines(True, precision)
    g = torch.nn.functional.embedding(inp["sid"], sd["emb_g.weight"])
    zin = gold["z"] * gold["y_mask"]
    o = eng.generator(zin, g).cpu()
    assert o.shape == gold["o"].shape
    e = rms(o, gold["o"])
    assert e < (TOL_WAV_FP32 if precision == "fp32" else TOL_WAV_TF32), e


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_full_infer_vs_reference_golden(engines, name, precision):
    """Whole SynthesizerTrn.infer through the C ABI against outputs of the unmodified reference."""
    meta, gold = load_golden(name)
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    eng = engines(meta["use_transformer_flow"], precision)
    B, T = inp["x"].shape
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"])
    w_ceil = eng.debug_read("w_ceil", (B, 1, T))
    flips = int((w_ceil != gold["w_ceil"]).sum())
    if flips:  # SURVEY.md §7 H1: ceil() is discontinuous; teacher-force and report
        print(f"[{name}] {flips} duration flips; teacher-forcing reference w_ceil")
        ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"],
                                  inp["ja_bert"], inp["en_bert"], nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"],
                                  w_ceil_override=gold["w_ceil"][:, 0])
    assert flips <= 1
    assert ylen.tolist() == gold["y_lengths"].tolist()
    o, attn, y_mask, (z, z_p, m_p, logs_p) = eng.infer_finish(B, T, F, nz, kw["noise_scale"])
    assert torch.equal(y_mask.cpu(), gold["y_mask"])
    assert torch.equal(attn.cpu().sum(2), gold["w_ceil"])
    for got, key in ((m_p, "m_p"), (logs_p, "logs_p"), (z_p, "z_p")):
        assert float((got.cpu() - gold[key]).abs().max()) < TOL_FP32, key
    ztol = TOL_FP32 if precision == "fp32" else 5e-3
    assert float((z.cpu() - gold["z"]).abs().max()) < ztol
    e = rms(o.cpu(), gold["o"])
    print(f"[{name}/{precision}] waveform RMS err {e:.3e}")
    assert e < (5e-5 if precision == "fp32" else TOL_WAV_TF32), e


def test_dropin_class_like_get_net_g():
    """Construct / load / infer exactly as reference infer.get_net_g + infer.infer do (infer.py:95-104, 302-318)."""
    from bert_vits2_b200.models import SynthesizerTrn
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    hps_model = dict(inter_channels=192, hidden_channels=192, filter_channels=768, n_heads=2, n_layers=6, kernel_size=3,
                     p_dropout=0.1, resblock="1", resblock_kernel_sizes=[3, 7, 11],
                     resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], upsample_rates=[8, 8, 2, 2, 2],
                     upsample_initial_channel=512, upsample_kernel_sizes=[16, 16, 8, 2, 2], n_layers_q=3, use_spectral_norm=False,
                     gin_channels=512, use_spk_conditioned_encoder=True, use_noise_scaled_mas=True, slm={"x": 1})
    net = SynthesizerTrn(112, 1025, 32, n_speakers=850, init_seed=None, precision="fp32", **hps_model).to("cuda:0")
    net.eval()
    missing = net.load_state_dict(sd, strict=False)
    assert not missing.missing_keys and not missing.unexpected_keys
    inp = synth.synthetic_inputs(cfg, [19], [0], seed=11)
    dev = {k: v.to("cuda:0") for k, v in inp.items()}
    torch.manual_seed(123)
    o, attn, y_mask, (z, z_p, m_p, logs_p) = net.infer(dev["x"], dev["x_lengths"], dev["sid"], dev["tone"], dev["language"],
                                                       dev["bert"], dev["ja_bert"], dev["en_bert"], sdp_ratio=0.5,
                                                       noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)
    audio = o[0, 0].data.cpu().float().numpy()  # as infer.py:315-318
    assert audio.ndim == 1 and np.isfinite(audio).all()
    F = int(y_mask.sum())
    assert audio.shape[0] == F * 512 and attn.shape == (1, 1, F, 19)
    # same device RNG stream => reproduce the noise and check against the oracle
    torch.manual_seed(123)
    nw = torch.randn(1, 2, 19, device="cuda:0").cpu()
    nz = torch.randn(1, 192, F, device="cuda:0").cpu()
    ref, _, _, _ = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9,
                           length_scale=1.0)
    assert ref.shape == o.shape and rms(o.cpu(), ref) < 5e-5


def test_max_len_and_cpu_module_raises():
    from bert_vits2_b200.models import SynthesizerTrn
    from bert_vits2_b200.engine import Bv2Error
    cfg, sd = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=850, gin_channels=512, init_seed=None, precision="fp32")
    net.load_state_dict(sd, strict=False)
    inp = synth.synthetic_inputs(cfg, [12], [2], seed=3)
    with pytest.raises(Bv2Error):
        net.infer(**inp)
    net = net.to("cuda:0")
    dev = {k: v.to("cuda:0") for k, v in inp.items()}
    torch.manual_seed(5)
    o_full, _, y_mask, _ = net.infer(**dev, sdp_ratio=0.2)
    torch.manual_seed(5)
    o_cut, _, _, _ = net.infer(**dev, sdp_ratio=0.2, max_len=10)
    assert o_cut.shape[-1] == 10 * 512
    # the Generator's receptive field (~14 frames/side) means only the early samples agree exactly
    assert torch.allclose(o_cut[..., : 2 * 512], o_full[..., : 2 * 512], atol=2e-2)
    with pytest.raises(ValueError):
        net.infer(dev["x"], dev["x_lengths"], dev["sid"], dev["tone"], dev["language"], dev["bert"][:, :, :5], dev["ja_bert"],
                  dev["en_bert"])


def test_single_token_and_determinism(engines):
    cfg, sd = model_for(True, 0)
    eng = engines(True, "fp32")
    inp = synth.synthetic_inputs(cfg, [1, 3], [0, 1], seed=4)
    nw, nz = synth.synthetic_noise(cfg, 2, 3, 256, seed=9)
    outs = []
    for _ in range(2):
        ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                                  inp["en_bert"], nw, 0.9, 1.0, 0.5)
        o, *_ = eng.infer_finish(2, 3, F, nz, 0.6)
        outs.append(o.cpu())
    assert torch.equal(outs[0], outs[1]) and torch.isfinite(outs[0]).all()
    from oracle import vits2_oracle as O
    ref, _, _, _ = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)
    assert ref.shape == outs[0].shape and rms(outs[0], ref) < 5e-5


def test_peer_slab_output_pointer_world1(engines):
    """SURVEY.md section 8e exchange step, single-process part: the engine stores the waveform batch through a raw output
    pointer into a libbv2-owned slab (the address a peer rank would have mapped with CUDA IPC), the meta record follows by
    bv2_peer_write, and the root-side views equal an ordinary infer() bit for bit.  Both the fused (out_ptr) and the
    API-level (copy of a finished tensor) variants, two slots."""
    from bert_vits2_b200.sharding import PeerWaveSlab
    cfg, sd = model_for(True, 0)
    eng = engines(True, "tf32")
    inp = synth.synthetic_inputs(cfg, [7, 12], [0, 2], seed=31)
    nw, nz = synth.synthetic_noise(cfg, 2, 12, 512, seed=32)
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, 0.9, 1.0, 0.5)
    o_ref, *_ = eng.infer_finish(2, 12, F, nz, 0.6)
    L = F * cfg.hop
    slab = PeerWaveSlab("cuda:0", 2, 2 * L, slots=2)
    try:
        assert slab.fits(2, L) and not slab.fits(3, L) and not slab.fits(2, 5 * L)
        ylen2, F2 = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                                    inp["en_bert"], nw, 0.9, 1.0, 0.5)
        assert F2 == F
        o_none, *_ = eng.infer_finish(2, 12, F, nz, 0.6, out_ptr=slab.wave_ptr(0))
        assert o_none is None
        slab.publish(0, 2, L, ylen2 * cfg.hop)
        slab.publish(1, 2, L, ylen * cfg.hop, wave=o_ref)
        for slot in (0, 1):
            waves, counts = slab.collect(slot)
            assert len(waves) == 1 and tuple(waves[0].shape) == (2, 1, L)
            assert torch.equal(waves[0], o_ref)
            assert counts[0].tolist() == [int(v) * cfg.hop for v in ylen]
        with pytest.raises(ValueError):
            slab.publish(0, 3, L, [1, 2, 3])
    finally:
        slab.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_config2_full_size_against_oracle(engines, precision):
    """BASELINE.json config 2: B=1, 256-phoneme ZH utterance, full path; waveform RMS vs the CPU oracle < 1e-3."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    eng = engines(True, precision)
    inp = synth.synthetic_inputs(cfg, [256], [0], seed=2)
    nw, nz = synth.synthetic_noise(cfg, 1, 256, 4096, seed=2)
    st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0,
                 return_stages=True)
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, 0.9, 1.0, 0.5)
    w_ceil = eng.debug_read("w_ceil", (1, 1, 256))
    flips = int((w_ceil != st["w_ceil"]).sum())
    print(f"config2: frames ref {int(st['y_lengths'][0])} got {int(ylen[0])}, duration flips {flips}")
    if flips:
        ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"],
                                  inp["ja_bert"], inp["en_bert"], nw, 0.9, 1.0, 0.5, w_ceil_override=st["w_ceil"][:, 0])
    assert flips <= 2 and int(ylen[0]) == int(st["y_lengths"][0])
    o, *_ = eng.infer_finish(1, 256, F, nz, 0.6)
    e = rms(o.cpu(), st["o"])
    print(f"config2/{precision}: waveform RMS err {e:.3e} (signal RMS {float(st['o'].pow(2).mean().sqrt()):.3f})")
    assert e < (5e-5 if precision == "fp32" else TOL_WAV_TF32)


def test_infer_batch_api_matches_single_calls():
    """SURVEY.md section 8f item 2: batched caller-side API; each utterance equals its own B=1 result except in the tail
    the padded-batch semantics of the reference touch (receptive field of flow + Generator)."""
    from bert_vits2_b200.infer_api import infer_batch
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, sd = model_for(True, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=850, gin_channels=512, init_seed=None, precision="fp32")
    net.load_state_dict(sd, strict=False)
    net = net.to("cuda:0").eval()
    items = []
    for k, t in enumerate([9, 14, 11, 14]):
        inp = synth.synthetic_inputs(cfg, [t], [k % 3], seed=20 + k)
        items.append((inp["bert"][0], inp["ja_bert"][0], inp["en_bert"][0], inp["x"][0], inp["tone"][0], inp["language"][0]))
    outs = infer_batch(net, items, sid=0, batch_size=2, sdp_ratio=0.0, noise_scale=0.0, noise_scale_w=0.0)  # deterministic: no noise
    assert len(outs) == 4 and all(o.ndim == 1 and o.size % 512 == 0 and np.isfinite(o).all() for o in outs)
    for k, it in enumerate(items):
        d = {n: v.unsqueeze(0).to("cuda:0") for n, v in zip(("bert", "ja_bert", "en_bert", "x", "tone", "language"), it)}
        o1, _, ym, _ = net.infer(d["x"], torch.tensor([it[3].shape[0]], device="cuda:0"), torch.zeros(1, dtype=torch.int64, device="cuda:0"),
                                 d["tone"], d["language"], d["bert"], d["ja_bert"], d["en_bert"], sdp_ratio=0.0, noise_scale=0.0, noise_scale_w=0.0)
        ref = o1[0, 0].cpu().numpy()
        assert ref.shape == outs[k].shape
        body = slice(0, max(0, ref.size - 20 * 512))
        assert np.abs(ref[body] - outs[k][body]).max() < 1e-4 if ref.size > 20 * 512 else True


def test_long_utterance_T512_and_batch8(engines):
    """BASELINE.json config 4 upper bound (512 phonemes, ~3k frames) and a B=8 ragged batch: full path vs the CPU oracle."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    eng = engines(True, "tf32")
    for lengths, langs, seed in (([512], [0], 31), ([64, 57, 33, 64, 12, 40, 64, 25], [0, 1, 2, 0, 1, 2, 0, 1], 32)):
        B, T = len(lengths), max(lengths)
        inp = synth.synthetic_inputs(cfg, lengths, langs, seed=seed)
        nw, nz = synth.synthetic_noise(cfg, B, T, 8192, seed=seed)
        st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0,
                     return_stages=True)
        ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                                  inp["en_bert"], nw, 0.9, 1.0, 0.5)
        w_ceil = eng.debug_read("w_ceil", (B, 1, T))
        flips = int((w_ceil != st["w_ceil"]).sum())
        if flips:
            ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                                      inp["en_bert"], nw, 0.9, 1.0, 0.5, w_ceil_override=st["w_ceil"][:, 0])
        assert flips <= 2 and ylen.tolist() == st["y_lengths"].tolist()
        o, attn, y_mask, (z, z_p, m_p, logs_p) = eng.infer_finish(B, T, F, nz, 0.6)
        e = rms(o.cpu(), st["o"])
        print(f"B={B} T={T} F={F}: duration flips {flips}, waveform RMS err {e:.3e}, z max err {float((z.cpu() - st['z']).abs().max()):.2e}")
        assert torch.isfinite(o).all() and e < TOL_WAV_TF32


# ================================================================================================
# round 2: parity gaps named by VERDICT r1 (spline tails, named configs at size, caller-side API vs the oracle, fp16
# checkpoints, WN flow at size, 16-bit PCM epilogue, lazy attn, input validation, tensor-core flow stage)
# ================================================================================================
TOL_Z_TC = 5e-3  # flow output max-abs, tensor-core engines (11-bit-significand operands through 16 transformer layers)


def _infer_checked(eng, inp, nw, nz, kw, st, max_flips=2):
    """Engine infer with the duration-flip protocol: report flips, teacher-force the oracle's w_ceil if any."""
    B, T = inp["x"].shape
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                              inp["en_bert"], nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"])
    w_ceil = eng.debug_read("w_ceil", (B, 1, T))
    flips = int((w_ceil != st["w_ceil"]).sum())
    if flips:
        ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"],
                                  inp["en_bert"], nw, kw["noise_scale_w"], kw["length_scale"], kw["sdp_ratio"],
                                  w_ceil_override=st["w_ceil"][:, 0])
    assert flips <= max_flips and ylen.tolist() == st["y_lengths"].tolist(), (flips, ylen.tolist())
    return ylen, F, flips


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_spline_tails_through_bv2_duration(engines, precision):
    """noise_w scaled so that the SDP latent crosses the +-5 tail bound: identity branch (reference transforms.py:61-74), the
    outermost bins and the boundary itself (inside = (x >= -5) & (x <= 5)).  The oracle is pinned against the live reference
    on exactly this regime (oracle/validate_against_reference.py case 4)."""
    from oracle import vits2_oracle as O
    import torch.nn.functional as Fn
    cfg, sd = model_for(True, 0)
    eng = engines(True, precision)
    inp = synth.synthetic_inputs(cfg, [40, 23], [0, 1], seed=51)
    nw, _ = synth.synthetic_noise(cfg, 2, 40, 64, seed=52)
    nw = nw.clone()
    nw[0, :, :8] = torch.tensor([[-9.0, -5.0, -4.999, 0.0, 4.999, 5.0, 6.0, 9.0]] * 2)  # scaled by 1.0 below: exact tail-bound values
    g = Fn.embedding(inp["sid"], sd["emb_g.weight"]).unsqueeze(-1)
    h, _, _, x_mask = O.text_encoder(sd, cfg, inp["x"], inp["x_lengths"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], g)
    for nsw in (1.0, 8.0):
        ref = O.sdp_reverse(sd, cfg, h, x_mask, g, nw, nsw)
        a, _ = eng.duration(h, inp["x_lengths"], inp["sid"], nw, nsw)
        outside = int(((nw * nsw).abs() > 5).sum())
        err = float((a.cpu() - ref).abs().max())
        print(f"[{precision}] noise_scale_w={nsw}: {outside} latent values beyond the tail bound, logw_sdp max-abs err {err:.2e} (|ref| max {float(ref.abs().max()):.1f})")
        assert outside > 0 and err < TOL_FP32 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("precision", ["tf32", "fp16"])
@pytest.mark.parametrize("name", ["tflow_b1", "tflow_b3", "random_F600_B2_ragged"])
def test_flow_stage_tensor_core_engines(engines, name, precision):
    if name.startswith("random"):
        # 600 frames (5 query / key tiles) at B = 2 with lengths 600 and 100: the fused attention splits the keys over a cluster
        # (ks = 4 on 132 SMs), walks several key tiles and crosses 128-key tile boundaries inside the relative-position band
        from oracle import vits2_oracle as O
        cfg, sd = model_for(True, 0)
        g = torch.Generator().manual_seed(600)
        z_p = torch.randn(2, cfg.inter_channels, 600, generator=g) * 0.8
        lens, sid = torch.tensor([600, 100]), torch.tensor([3, 11])
        y_mask = (torch.arange(600)[None, :] < lens[:, None]).float()[:, None, :]
        z_p = z_p * y_mask
        z_ref = O.flow_reverse(sd, cfg, z_p, y_mask, F.embedding(sid, sd["emb_g.weight"]).unsqueeze(-1))
        z = engines(True, precision).flow_reverse(z_p, lens, sid).cpu()
        err = max(float((z[b, :, :L] - z_ref[b, :, :L]).abs().max()) for b, L in enumerate(lens.tolist()))
    else:
        meta, gold = load_golden(name)
        cfg, sd, inp, nw, nz, kw = case_inputs(meta)
        eng = engines(True, precision)
        z = eng.flow_reverse(gold["z_p"], gold["y_lengths"], inp["sid"])
        err = float((z.cpu() - gold["z"]).abs().max())
    print(f"[{name}/{precision}] flow z max-abs err {err:.2e}")
    assert err < TOL_Z_TC, err


def test_config3_full_size_vs_oracle(engines):
    """BASELINE.json config 3 at size: B=32 mixed ZH/JA/EN 128-phoneme utterances (length_scale 0.625 as in bench.py)."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    eng = engines(True, "fp16")
    inp = synth.synthetic_inputs(cfg, [128] * 32, [i % 3 for i in range(32)], seed=3)
    nw, nz = synth.synthetic_noise(cfg, 32, 128, 2048, seed=3)
    kw = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.625)
    st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)
    ylen, F, flips = _infer_checked(eng, inp, nw, nz, kw, st, max_flips=6)
    o, attn, y_mask, (z, *_) = eng.infer_finish(32, 128, F, nz, kw["noise_scale"])
    e = rms(o.cpu(), st["o"])
    print(f"config3 B=32 T=128 F={F}: flips {flips}, waveform RMS err {e:.3e}, z max err {float((z.cpu() - st['z']).abs().max()):.2e}")
    assert torch.equal(attn.cpu().sum(2), st["w_ceil"]) and e < TOL_WAV_TF32


def test_config4_shaped_ragged_batch_vs_oracle(engines):
    """BASELINE.json config 4 shape (one rank's share, subsampled for the CPU oracle): ragged T in [64, 512] in one padded batch."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    eng = engines(True, "fp16")
    lengths = [64, 173, 512, 256, 384, 450]
    inp = synth.synthetic_inputs(cfg, lengths, [i % 3 for i in range(len(lengths))], seed=41)
    nw, nz = synth.synthetic_noise(cfg, len(lengths), 512, 4096, seed=41)
    kw = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.5)
    st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)
    ylen, F, flips = _infer_checked(eng, inp, nw, nz, kw, st, max_flips=4)
    o, attn, y_mask, (z, *_) = eng.infer_finish(len(lengths), 512, F, nz, kw["noise_scale"])
    e = rms(o.cpu(), st["o"])
    print(f"config4-shaped B={len(lengths)} T<=512 F={F}: flips {flips}, waveform RMS err {e:.3e}")
    assert torch.equal(y_mask.cpu(), st["y_mask"]) and e < TOL_WAV_TF32


@pytest.mark.parametrize("precision", ["fp32", "tf32", "fp16"])
def test_config5_generator_1024_frames(engines, precision):
    """BASELINE.json config 5: Generator-only, z[1,192,1024] -> wav[1,1,524288] through bv2_generator."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    eng = engines(True, precision)
    z, g = synth.synthetic_generator_inputs(cfg, 1, 1024)
    ref = O.generator(sd, cfg, z, g)
    o = eng.generator(z, g).cpu()
    e = rms(o, ref)
    print(f"config5/{precision}: waveform RMS err {e:.3e} (signal RMS {float(ref.pow(2).mean().sqrt()):.3f})")
    assert o.shape == ref.shape == (1, 1, 1024 * 512) and e < (TOL_WAV_FP32 if precision == "fp32" else TOL_WAV_TF32)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_wn_flow_T256_vs_oracle(engines, precision):
    """use_transformer_flow=False (ResidualCouplingBlock / WN, reference models.py:403-445, modules.py:185-210) at config-2 size."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(False, 0)
    eng = engines(False, precision)
    inp = synth.synthetic_inputs(cfg, [256], [0], seed=2)
    nw, nz = synth.synthetic_noise(cfg, 1, 256, 8192, seed=2)
    kw = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=0.3)
    st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)
    ylen, F, flips = _infer_checked(eng, inp, nw, nz, kw, st)
    o, attn, y_mask, (z, *_) = eng.infer_finish(1, 256, F, nz, kw["noise_scale"])
    e, ez = rms(o.cpu(), st["o"]), float((z.cpu() - st["z"]).abs().max())
    print(f"WN flow T=256 F={F} [{precision}]: flips {flips}, z max err {ez:.2e}, waveform RMS err {e:.3e}")
    assert ez < (TOL_FP32 if precision == "fp32" else TOL_Z_TC) and e < (5e-5 if precision == "fp32" else TOL_WAV_TF32)


def _dropin(precision="fp32", tflow=True):
    from bert_vits2_b200.models import SynthesizerTrn
    cfg, sd = model_for(tflow, 0)
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=850, gin_channels=512, init_seed=None, precision=precision, use_transformer_flow=tflow)
    net.load_state_dict(sd, strict=False)
    return cfg, sd, net.to("cuda:0").eval()


def test_infer_batch_vs_oracle():
    """SURVEY.md section 8f.2: the batched caller-side API against the ORACLE on the same padded buckets and the same RNG draws
    (torch.randn on the device in the reference's order: [B,2,T] first, then [B,192,F], per bucket)."""
    from bert_vits2_b200.infer_api import infer_batch
    from bert_vits2_b200.sharding import deal_buckets
    from oracle import vits2_oracle as O
    cfg, sd, net = _dropin("fp32")
    lens = [9, 14, 11, 14, 30]
    items, inps = [], []
    for k, t in enumerate(lens):
        inp = synth.synthetic_inputs(cfg, [t], [k % 3], seed=20 + k)
        inps.append(inp)
        items.append((inp["bert"][0], inp["ja_bert"][0], inp["en_bert"][0], inp["x"][0], inp["tone"][0], inp["language"][0]))
    kw = dict(sdp_ratio=0.3, noise_scale=0.6, noise_scale_w=0.8, length_scale=1.0)
    torch.manual_seed(77)
    outs = infer_batch(net, items, sid=0, batch_size=2, **kw)
    # replay: same buckets, same device RNG stream
    torch.manual_seed(77)
    plan = deal_buckets(lens, world_size=1, batch_size=2)[0]
    for bucket in plan:
        ls = [lens[i] for i in bucket]
        B, T = len(ls), max(ls)
        pad = {k: torch.zeros(B, T, dtype=torch.int64) for k in ("x", "tone", "language")}
        feats = {k: torch.zeros(B, 1024, T) for k in ("bert", "ja_bert", "en_bert")}
        for b, i in enumerate(bucket):
            t = lens[i]
            for k in pad:
                pad[k][b, :t] = inps[i][k][0]
            for k in feats:
                feats[k][b, :, :t] = inps[i][k][0]
        nw = torch.randn(B, 2, T, device="cuda:0").cpu()
        g = torch.nn.functional.embedding(torch.zeros(B, dtype=torch.int64), sd["emb_g.weight"]).unsqueeze(-1)
        # frames are needed to draw noise_z with the reference's shape: run the oracle's front end first
        h, m_p, logs_p, x_mask = O.text_encoder(sd, cfg, pad["x"], torch.tensor(ls), pad["tone"], pad["language"], feats["bert"], feats["ja_bert"], feats["en_bert"], g)
        logw = O.sdp_reverse(sd, cfg, h, x_mask, g, nw, kw["noise_scale_w"]) * kw["sdp_ratio"] + O.duration_predictor(sd, cfg, h, x_mask, g) * (1 - kw["sdp_ratio"])
        F = int(torch.ceil(torch.exp(logw) * x_mask * kw["length_scale"]).sum((1, 2)).clamp_min(1).max())
        nz = torch.randn(B, 192, F, device="cuda:0").cpu()
        ref, _, ym, _ = O.infer(sd, cfg, pad["x"], torch.tensor(ls), torch.zeros(B, dtype=torch.int64), pad["tone"], pad["language"], feats["bert"],
                                feats["ja_bert"], feats["en_bert"], noise_w=nw, noise_z=nz, **kw)
        for b, i in enumerate(bucket):
            n = int(ym[b].sum()) * 512
            assert outs[i].shape == (n,), (outs[i].shape, n)
            e = float(np.sqrt(np.mean((outs[i].astype(np.float64) - ref[b, 0, :n].double().numpy()) ** 2)))
            assert e < 5e-5, (i, e)


def test_max_len_vs_oracle():
    """train_ms.evaluate-style call (max_len cuts the decoder input, reference models.py:1073) against the oracle."""
    from oracle import vits2_oracle as O
    cfg, sd, net = _dropin("fp32")
    inp = synth.synthetic_inputs(cfg, [12], [2], seed=3)
    dev = {k: v.to("cuda:0") for k, v in inp.items()}
    nw, nz = synth.synthetic_noise(cfg, 1, 12, 512, seed=5)
    kw = dict(sdp_ratio=0.2, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)
    o_cut, _, y_mask, _ = net.infer(**dev, **kw, max_len=10, noise_w=nw.cuda(), noise_z=nz.cuda())
    ref, _, ym, _ = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, max_len=10, **kw)
    assert int(ym.sum()) > 10 and o_cut.shape == ref.shape == (1, 1, 10 * 512)
    assert rms(o_cut.cpu(), ref) < 5e-5


def test_fp16_checkpoint_load():
    """compress_model.py:49-52 style fp16 checkpoints: bv2_set_weight dtype 1 converts on load; equals the oracle run on the
    same half-rounded weights."""
    from bert_vits2_b200.engine import Engine
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    sd16 = {k: v.half() for k, v in sd.items()}
    eng = Engine(cfg, sd16, device="cuda:0", precision="fp32")
    sdr = {k: v.float() for k, v in sd16.items()}
    inp = synth.synthetic_inputs(cfg, [21], [0], seed=61)
    nw, nz = synth.synthetic_noise(cfg, 1, 21, 1024, seed=62)
    kw = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)
    st = O.infer(sdr, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)
    ylen, F, flips = _infer_checked(eng, inp, nw, nz, kw, st)
    o, *_ = eng.infer_finish(1, 21, F, nz, kw["noise_scale"])
    assert rms(o.cpu(), st["o"]) < 5e-5


def test_pcm16_epilogue_bit_exact(engines):
    """SURVEY.md section 8f.4: 16-bit PCM exactly as the reference's callers convert every infer() result (gradio
    convert_to_16_bit_wav, webui.py:86).  (1) the device conversion of the ORACLE's float waveform is bit-identical to the
    restated reference conversion; (2) infer_finish(pcm16=True) is bit-identical to converting the float output of the same call."""
    from oracle import vits2_oracle as O
    cfg, sd = model_for(True, 0)
    eng = engines(True, "fp16")
    inp = synth.synthetic_inputs(cfg, [17, 9], [0, 1], seed=71)
    nw, nz = synth.synthetic_noise(cfg, 2, 17, 1024, seed=72)
    kw = dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0)
    ref, _, ym, _ = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, **kw)
    nvalid = (ym.sum((1, 2)).long() * 512)
    got = eng.wave_to_pcm16(ref, nvalid).cpu().numpy()
    for b in range(2):
        n = int(nvalid[b])
        want = O.convert_to_16_bit_wav(ref[b, 0, :n].numpy())
        assert np.array_equal(got[b, 0, :n], want) and not got[b, 0, n:].any()
    ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw, 0.9, 1.0, 0.5)
    o_f, *_ = eng.infer_finish(2, 17, F, nz, 0.6)
    eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw, 0.9, 1.0, 0.5)
    o_i, *_ = eng.infer_finish(2, 17, F, nz, 0.6, pcm16=True)
    assert o_i.dtype == torch.int16 and o_i.shape == o_f.shape
    for b in range(2):
        n = int(ylen[b]) * 512
        assert np.array_equal(o_i[b, 0, :n].cpu().numpy(), O.convert_to_16_bit_wav(o_f[b, 0, :n].cpu().numpy()))


def test_lazy_attn_and_no_hidden_allocation():
    """attn is materialised on demand (reference callers never read it) and equals the eager path; a steady workload does not
    touch the allocator after reserve()."""
    cfg, sd, net = _dropin("fp32")
    inp = synth.synthetic_inputs(cfg, [13, 8], [0, 2], seed=81)
    dev = {k: v.to("cuda:0") for k, v in inp.items()}
    eng = net._engine(torch.device("cuda:0"))
    eng.reserve(2, 13, 512)
    g0 = eng.workspace_grows
    nw, nz = synth.synthetic_noise(cfg, 2, 13, 512, seed=82)
    for _ in range(3):
        o, attn, y_mask, _ = net.infer(**dev, sdp_ratio=0.5, noise_w=nw.cuda(), noise_z=nz.cuda())
    assert eng.workspace_grows == g0
    assert type(attn).__name__ == "LazyAttn" and attn.shape == (2, 1, int(y_mask.shape[-1]), 13)
    dense = attn.materialize()
    ylen, F = eng.infer_begin(dev["x"], dev["x_lengths"], dev["sid"], dev["tone"], dev["language"], dev["bert"], dev["ja_bert"], dev["en_bert"],
                              nw, 0.8, 1.0, 0.5)
    _, eager, *_ = eng.infer_finish(2, 13, F, nz, 0.667, want_attn=True)
    assert torch.equal(dense, eager) and torch.equal(attn.sum(3).squeeze(1), y_mask.squeeze(1))


def test_out_of_range_ids_raise_index_error(engines):
    """The reference raises IndexError from nn.Embedding; the engine validates on the device (no out-of-bounds read, context alive)."""
    cfg, sd = model_for(True, 0)
    eng = engines(True, "fp32")
    inp = synth.synthetic_inputs(cfg, [10], [0], seed=91)
    nw, nz = synth.synthetic_noise(cfg, 1, 10, 256, seed=92)
    args = lambda d: (d["x"], d["x_lengths"], d["sid"], d["tone"], d["language"], d["bert"], d["ja_bert"], d["en_bert"], nw, 0.9, 1.0, 0.5)  # noqa: E731
    for key, val in (("sid", cfg.n_speakers), ("x", cfg.n_vocab + 5), ("tone", -1), ("language", 7)):
        bad = {k: v.clone() for k, v in inp.items()}
        bad[key].view(-1)[0] = val
        with pytest.raises(IndexError):
            eng.infer_begin(*args(bad))
    bad = {k: v.clone() for k, v in inp.items()}
    bad["x_lengths"][0] = 11
    with pytest.raises(IndexError):
        eng.infer_begin(*args(bad))
    ylen, F = eng.infer_begin(*args(inp))  # still healthy
    o, *_ = eng.infer_finish(1, 10, F, nz, 0.6)
    assert torch.isfinite(o).all()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_packed_weight_file_roundtrip(tmp_path, precision):
    """SURVEY.md section 8f.4: pre-folded, pre-packed engine weight file.  An engine loaded from the file (one cudaMemcpy) produces
    bit-identical output to the engine that wrote it; a file written for another precision is rejected."""
    import time
    from bert_vits2_b200.engine import Bv2Error, Engine
    cfg, sd = model_for(True, 0)
    t0 = time.perf_counter()
    eng = Engine(cfg, sd, device="cuda:0", precision=precision)
    t_build = time.perf_counter() - t0
    path = str(tmp_path / f"bv2_{precision}.pack")
    eng.save_packed(path)
    t0 = time.perf_counter()
    eng2 = Engine(cfg, None, device="cuda:0", precision=precision, packed_path=path)
    t_load = time.perf_counter() - t0
    inp = synth.synthetic_inputs(cfg, [19, 7], [0, 1], seed=101)
    nw, nz = synth.synthetic_noise(cfg, 2, 19, 1024, seed=102)
    outs = []
    for e in (eng, eng2):
        ylen, F = e.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw, 0.9, 1.0, 0.5)
        o, *_ = e.infer_finish(2, 19, F, nz, 0.6)
        outs.append((ylen.tolist(), o.cpu()))
    print(f"[{precision}] engine from state_dict {t_build:.2f} s, from packed file {t_load:.2f} s ({os.path.getsize(path) / 1e6:.0f} MB)")
    assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])
    other = "fp32" if precision != "fp32" else "tf32"
    with pytest.raises((Bv2Error, ValueError)):
        Engine(cfg, None, device="cuda:0", precision=other, packed_path=path)


def test_two_engines_two_devices_one_process():
    """ADVICE r1: the > 48 KB dynamic shared memory opt-in is a per-device function attribute -- one process driving one engine per
    GPU must work on every device (set per engine in finalize, not once per process)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs in one process")
    from bert_vits2_b200.engine import Engine
    cfg, sd = model_for(True, 0)
    inp = synth.synthetic_inputs(cfg, [33], [0], seed=111)
    nw, nz = synth.synthetic_noise(cfg, 1, 33, 1024, seed=112)
    outs = []
    for d in ("cuda:0", "cuda:1"):
        eng = Engine(cfg, sd, device=d, precision="fp16")
        with torch.cuda.device(d):
            ylen, F = eng.infer_begin(inp["x"], inp["x_lengths"], inp["sid"], inp["tone"], inp["language"], inp["bert"], inp["ja_bert"], inp["en_bert"], nw, 0.9, 1.0, 0.5)
            o, *_ = eng.infer_finish(1, 33, F, nz, 0.6)
            torch.cuda.synchronize(d)
        outs.append(o.cpu())
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
