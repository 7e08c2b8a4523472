"""The kernel case matrix runs every FP16 transformer-flow convolution at the (Cin, Cout, K) the engine gives it: the shapes come from the
model's parameter table, not from the case list (no GPU needed)."""
import kernel_cases as KC
import kernel_harness as KH
import flow_kernel_cases as FC
from bert_vits2_b200 import spec


def _flow_conv_shapes(cfg):
    """(Cin, Cout, K) of every tensor-core convolution of one transformer coupling layer, as the engine packs it: q, k and v fused into
    one 3H-column projection (engine.cu encoder_from), conv_o, FFN conv_1 and conv_2 with K from their weights."""
    w = {p.key: p.shape for p in spec.param_specs(cfg)}
    enc = "flow.flows.0.enc"
    q = w[f"{enc}.attn_layers.0.conv_q.weight"]
    shapes = {"qkv": (q[1], 3 * q[0], q[2])}
    for name, key in (("conv_o", "attn_layers.0.conv_o"), ("ffn1", "ffn_layers.0.conv_1"), ("ffn2", "ffn_layers.0.conv_2")):
        co, ci, k = w[f"{enc}.{key}.weight"]
        shapes[name] = (ci, co, k)
    return shapes


def test_fp16_flow_families_cover_the_engine_shapes():
    cfg = spec.ModelConfig()
    assert cfg.use_transformer_flow and cfg.flow_kernel_size == 5
    fams = {**KC.FAMILIES, **FC.FAMILIES}
    have = {(f["Cin"], f["Cout"], f["K"]) for n, f in fams.items() if n.startswith("f16.")}
    cases = {fam for _, fam, *_ in KC.conv_cases()} | {fam for _, fam, *_ in FC.conv_cases()}
    for name, shape in _flow_conv_shapes(cfg).items():
        assert shape in have, f"flow {name} {shape} has no FP16 kernel family"
        assert any((fams[f]["Cin"], fams[f]["Cout"], fams[f]["K"]) == shape for f in cases if f.startswith("f16.")), (name, shape)


def test_flow_ffn_k5_cases_plan_what_they_state():
    KH.load()
    for cid, fam, B, T, lens, sms, expect in FC.conv_cases():
        p = KH.tc_plan(FC.family_args(fam, B, T, lens, sms))
        if expect:
            assert KH.KIND_NAMES[p.kind] == expect["kind"], (cid, str(p))
