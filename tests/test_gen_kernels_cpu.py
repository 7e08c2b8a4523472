"""CPU checks of the Generator kernel cases (no GPU needed): every k_g2_conv plan the engine can select at the default configuration is
planned by a case of tests/test_kernels_gpu.py, the generated cases plan the key and the super-tile shape their ids name, and the fp32
Generator case lists reach both tiles of k_conv1d_c4 for every kernel size."""
import kernel_cases as KC
import kernel_harness as KH
from bert_vits2_b200.spec import ModelConfig


def _case_plan(c):
    cid, Cin, Cout, K, dil, u, T, B, res, acc, scale, st, bb, sms, expect = c
    f = dict(Cin=Cin, Cout=Cout, K=K, u=u, dil=dil, res=res, acc=acc, scale=scale, bb=bb)
    return KC.g2_layer_plan(f, T, B, sms, st)


def test_g2_layers_are_the_engine_launches():
    """the Generator's k_g2_conv launches at the default config: conv_pre, 5 upsampling layers and 5 stages x 3 branches x 3 dilations x
    (convs1, convs2) -- 96 in all (conv_post has a kernel of its own)"""
    cfg = ModelConfig()
    L = KC.g2_layers(cfg)
    assert len(L) == 96, len(L)
    eps = [KC.g2_epilogue(f) for f in L]
    assert eps.count("pre") == 1 and eps.count("ups") == len(cfg.upsample_rates)
    assert eps.count("c2acc") == eps.count("c2acc3") == len(cfg.upsample_rates)  # the last convs2 of branches 1 and 2 of every stage
    assert {(f["Cin"], f["Cout"], f["K"], f["u"]) for f in L if f["u"]} == {(512, 256, 16, 8), (256, 128, 16, 8), (128, 64, 8, 2),
                                                                            (64, 32, 2, 2), (32, 16, 2, 2)}


def test_g2_cases_plan_every_reachable_key():
    """Every plan key the engine can select (every layer, B in 1..32, every window length, 132 and 114 SMs) is planned by a GPU case.
    Also prints the issuer instantiations k_g2_conv compiles that no default-config plan reaches."""
    reach = KC.g2_reachable()
    planned = {KC.g2_key(_case_plan(c)) for c in KC.g2_cases()}
    missing = sorted(set(reach) - planned)
    lines = [f"  {KC.g2_key_name(k)}: e.g. layer {reach[k][0]['name']} (Cin {reach[k][0]['Cin']}, Cout {reach[k][0]['Cout']}, K {reach[k][0]['K']}, "
             f"u {reach[k][0]['u']}, dil {reach[k][0]['dil']}) at T={reach[k][1]} B={reach[k][2]} num_sms={reach[k][3]}" for k in missing]
    assert not missing, f"{len(missing)} engine plan(s) without a kernel case:\n" + "\n".join(lines)
    issuers = {(k[0], k[1], k[2]) for k in reach}
    unreachable = [i for i in KC.G2_ISSUERS if i not in issuers]
    print(f"\n{len(reach)} reachable plan keys: {', '.join(KC.g2_key_name(k) for k in sorted(reach))}")
    print(f"issuer instantiations (NK, NT, MG) compiled but unreachable at the default config: {unreachable}")


def test_g2_generated_cases_plan_what_they_claim():
    """each generated case plans its key; tail cases fill every group, partial cases leave the last CTA's super-tile partial (with
    NG > 1: at least one whole group past T, whose activation copy is 0 bytes); T is never a multiple of 128"""
    gen = [c for c in KC.g2_cases() if c[-1] is not None]
    assert gen
    for c in gen:
        cid, T, expect = c[0], c[6], c[-1]
        p = _case_plan(c)
        assert KC.g2_key(p) == expect and cid.startswith(f"plan-{KC.g2_key_name(expect)}-"), (cid, str(p))
        assert T % 128, cid
        m, st = -(-T // 128), p.NG * p.MG
        rem = m - (p.grid_x - 1) * st
        if cid.endswith("-tail"):
            assert rem == st, (cid, str(p))
        else:
            assert cid.endswith("-partial") and p.grid_x >= 2, (cid, str(p))
            if p.NG > 1:
                pad = (c[3] - 1) // 2 * c[4]
                first_empty = (p.grid_x - 1) * st * 128 + -(-rem // p.MG) * p.MG * 128  # first row of the first group past T
                assert first_empty - pad >= T + KH.g2_pads()[1], (cid, str(p))
            elif st > 1:
                assert rem < st, (cid, str(p))


def test_conv1d_cases_reach_both_tiles_for_every_kernel_size():
    tiles = {(K, KC.conv1d_big_tile(T, C, B)) for _, C, K, dil, T, B, res, acc in KC.CONV1D_CASES}
    assert tiles == {(K, big) for K in (3, 7, 11) for big in (False, True)}, sorted(tiles)
    assert {c[3] for c in KC.CONV1D_CASES} == {1, 3, 5} and {c[1] for c in KC.CONV1D_CASES} == {16, 64, 256}
    assert any(c[6] for c in KC.CONV1D_CASES) and any(c[7] for c in KC.CONV1D_CASES)  # the residual, the running sum with 1/3
