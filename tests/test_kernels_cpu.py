"""CPU checks of the kernel-test machinery: the float64 references in tests/kernel_ref.py against PyTorch and the oracle (rounding off),
the operand rounding helpers, and the dispatch coverage of the GPU case matrix through the host planner (no GPU needed)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_cases as KC
import kernel_harness as KH
import kernel_ref as R


def _rng(seed):
    return np.random.default_rng(seed)


@pytest.mark.parametrize("K,dil", [(1, 1), (3, 1), (5, 1), (7, 3), (11, 5), (3, 5)])
def test_conv1d_ref_matches_torch(K, dil):
    g = _rng(K * 10 + dil)
    x = g.standard_normal((2, 12, 37))
    w = g.standard_normal((8, 12, K))
    ref, mag = R.conv1d(x, w, dil)
    want = F.conv1d(torch.from_numpy(x), torch.from_numpy(w), padding=(K - 1) // 2 * dil, dilation=dil).numpy()
    np.testing.assert_allclose(ref, want, rtol=1e-12, atol=1e-12)
    want_mag = F.conv1d(torch.from_numpy(np.abs(x)), torch.from_numpy(np.abs(w)), padding=(K - 1) // 2 * dil, dilation=dil).numpy()
    np.testing.assert_allclose(mag, want_mag, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("K,u", [(16, 8), (8, 2), (2, 2), (4, 2), (6, 2)])
@pytest.mark.parametrize("T", [1, 5, 33])
def test_conv_transpose1d_ref_matches_torch(K, u, T):
    g = _rng(K * 100 + u * 10 + T)
    x = g.standard_normal((2, 6, T))
    w = g.standard_normal((6, 4, K))
    ref, mag = R.conv_transpose1d(x, w, u)
    want = F.conv_transpose1d(torch.from_numpy(x), torch.from_numpy(w), stride=u, padding=(K - u) // 2).numpy()
    assert ref.shape == want.shape == (2, 4, T * u)
    np.testing.assert_allclose(ref, want, rtol=1e-12, atol=1e-12)
    want_mag = F.conv_transpose1d(torch.from_numpy(np.abs(x)), torch.from_numpy(np.abs(w)), stride=u, padding=(K - u) // 2).numpy()
    np.testing.assert_allclose(mag, want_mag, rtol=1e-12, atol=1e-12)


def test_tc_conv_ref_without_rounding_is_the_module_semantics():
    """op=None: tc_conv is exactly conv + bias (+ per-batch bias) (+/- residual) (+ old output), lrelu input, scale and masks."""
    g = _rng(3)
    B, Cin, Cout, T, K = 2, 8, 8, 20, 3
    x, w, b = g.standard_normal((B, Cin, T)), g.standard_normal((Cout, Cin, K)), g.standard_normal(Cout)
    res, yo, bb = g.standard_normal((B, Cout, T)), g.standard_normal((B, Cout, T)), g.standard_normal((B, Cout))
    lens = [20, 7]
    out = R.tc_conv(x, w, b, op=None, in_slope=0.1, in_mask=True, lens=lens, bias_b=bb, res=res, res_mode=1, y_old=yo, out_scale=0.5,
                    out_mask=True)["ref"]
    m = torch.from_numpy((np.arange(T)[None, :] < np.array(lens)[:, None])[:, None, :].astype(np.float64))
    xt = F.leaky_relu(torch.from_numpy(x.astype(np.float32).astype(np.float64)) * m, 0.1)
    want = (F.conv1d(xt, torch.from_numpy(w.astype(np.float32).astype(np.float64)), torch.from_numpy(b), padding=1)
            + torch.from_numpy(bb)[:, :, None] + torch.from_numpy(res) + torch.from_numpy(yo)) * 0.5 * m
    np.testing.assert_allclose(out, want.numpy(), rtol=1e-6, atol=1e-6)  # fp32 lrelu / operand storage only
    out2 = R.tc_conv(x, w, b, op=None, res=res, res_mode=2)["ref"]
    want2 = torch.from_numpy(res) - F.conv1d(torch.from_numpy(x.astype(np.float32).astype(np.float64)),
                                             torch.from_numpy(w.astype(np.float32).astype(np.float64)), torch.from_numpy(b), padding=1)
    np.testing.assert_allclose(out2, want2.numpy(), rtol=1e-12, atol=1e-12)


def test_attention_ref_matches_oracle_mha_rel():
    """flow_attn without fp16 rounding == the oracle's windowed relative attention core on rows < len."""
    from oracle import vits2_oracle as O
    g = _rng(11)
    B, nh, dk, T, w = 2, 2, 8, 23, 4
    C = nh * dk
    lens = [23, 9]
    sd = {}
    for n in ("q", "k", "v"):
        sd[f"a.conv_{n}.weight"] = torch.from_numpy(g.standard_normal((C, C, 1)))
        sd[f"a.conv_{n}.bias"] = torch.zeros(C, dtype=torch.float64)
    sd["a.conv_o.weight"] = torch.eye(C, dtype=torch.float64)[:, :, None]
    sd["a.conv_o.bias"] = torch.zeros(C, dtype=torch.float64)
    sd["a.emb_rel_k"] = torch.from_numpy(g.standard_normal((1, 2 * w + 1, dk)))
    sd["a.emb_rel_v"] = torch.from_numpy(g.standard_normal((1, 2 * w + 1, dk)))
    x = torch.from_numpy(g.standard_normal((B, C, T)))
    xm = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None]).double()[:, None, :]
    attn_mask = xm.unsqueeze(2) * xm.unsqueeze(-1)
    want = O.mha_rel(sd, "a", x, attn_mask, nh, w).numpy()  # [B][C][T]
    proj = {n: torch.einsum("oc,bct->bot", sd[f"a.conv_{n}.weight"][:, :, 0], x).numpy().reshape(B, nh, dk, T).transpose(0, 1, 3, 2)
            for n in ("q", "k", "v")}
    got = R.flow_attn(proj["q"] / math.sqrt(dk), proj["k"], proj["v"], sd["a.emb_rel_k"][0].numpy(), sd["a.emb_rel_v"][0].numpy(), lens, w,
                      round_p=False, round_out=False)
    got = got.transpose(0, 1, 3, 2).reshape(B, C, T)
    for b, L in enumerate(lens):
        np.testing.assert_allclose(got[b, :, :L], want[b, :, :L], rtol=1e-10, atol=1e-12)
        assert not got[b, :, L:].any()  # the kernel's contract: rows >= len are zero


def test_operand_rounding_helpers():
    # TF32: ties away from zero on the 13 dropped bits; non-finite values pass through
    one = np.float32(1.0)
    ulp = np.float32(2.0 ** -10)
    tie = one + ulp / 2
    assert R.tf32(np.array([tie]))[0] == one + ulp
    assert R.tf32(np.array([-tie]))[0] == -(one + ulp)
    assert R.tf32(np.array([np.nextafter(tie, np.float32(0))], np.float32))[0] == one
    assert np.isinf(R.tf32(np.array([np.inf], np.float32))[0]) and np.isnan(R.tf32(np.array([np.nan], np.float32))[0])
    x = _rng(5).standard_normal(10000).astype(np.float32) * 100
    r = R.tf32(x)
    assert np.all((r.view(np.uint32) & 0x1FFF) == 0) and np.all(np.abs(r - x) <= np.abs(x) * 2.0 ** -11)
    # FP16: round to nearest even, saturating instead of overflowing to inf
    assert R.f16(np.array([1e6, -1e6], np.float32)).tolist() == [65504.0, -65504.0]
    np.testing.assert_array_equal(R.f16(x), torch.from_numpy(x).half().float().numpy())


def test_dispatch_coverage_of_the_case_matrix():
    """Every tc_conv1d variant the engine can select is reached by at least one GPU case, and the forced-dispatch cases plan what they
    state.  A change to the dispatch that drops a variant (or moves a case off the branch it is meant to test) fails here."""
    KH.load()
    reached, persist_tiles = set(), 0
    for cid, fam, B, T, lens, sms, expect in KC.conv_cases():
        p = KH.tc_plan(KC.family_args(fam, B, T, lens, sms))
        kind = KH.KIND_NAMES[p.kind]
        reached.add((kind, p.f16, p.gen))
        reached.add(("res_smem", p.res_smem))
        if kind == "persist":
            persist_tiles = max(persist_tiles, p.tiles_per_cta)
        if expect:
            got = dict(kind=kind, res_smem=p.res_smem)
            assert all(got[k] == v for k, v in expect.items()), (cid, expect, str(p))
    for kind in ("one-tile", "persist", "pstream"):
        for f16 in (0, 1):
            for gen in (0, 1):
                assert (kind, f16, gen) in reached, (kind, f16, gen)
    assert ("res_smem", 0) in reached and ("res_smem", 1) in reached
    # the persistent kernel walks many tiles per CTA: wraps its 3-deep activation ring and double-buffered accumulator phases
    assert persist_tiles >= 6, persist_tiles


def test_n_tile_widths_of_the_case_matrix():
    """N tiles that split the MMA warpgroup's work into 64 / 32 / 16-column wgmma slices in every combination the engine uses."""
    KH.load()
    widths = {KH.tc_plan(KC.family_args(fam, B, T, lens, sms)).nt for _, fam, B, T, lens, sms, _ in KC.conv_cases()}
    assert {16, 32, 48, 64, 96, 128, 192} <= widths, sorted(widths)


def test_g2_plan_cases_reach_both_weight_modes_and_super_tiles():
    KH.load()
    modes, mgs = set(), set()
    for cid, Cin, Cout, K, dil, u, T, B, res, acc, scale, st, bb, sms, expect in KC.g2_cases():
        p = KH.g2_plan(KH.g2_args(B=B, T=T, Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, residual=res, accumulate=acc, out_scale=scale,
                                  st_override=st, num_sms=sms, res=1 if res else None, bias_b=1 if bb else None,
                                  bias_b_stride=Cout + 40 if bb else 0))
        if expect:
            assert KC.g2_key(p) == expect, (cid, KC.g2_key_name(expect), str(p))
        modes.add(p.resident)
        mgs.add((p.resident, p.NG, p.MG))
    assert modes == {0, 1}
    assert {m for r, n, m in mgs if not r} == {1, 2}, sorted(mgs)  # streamed: one or two m-tiles per weight pass
    assert any(n > 1 for r, n, m in mgs if r) and any(m > 1 for r, n, m in mgs if r), sorted(mgs)  # resident: pipelined m-groups
