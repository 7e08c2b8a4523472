"""Pin the CPU oracle (oracle/vits2_oracle.py) against fixtures produced by the UNMODIFIED reference
(tests/golden/make_golden.py, run in the build container where /root/reference exists).
The reference itself ships no tests or golden vectors for this path (SURVEY.md §4)."""
import json
import os

import pytest
import torch

from oracle import vits2_oracle as O
from util import GOLDEN_CASES, GOLDEN_DIR, case_inputs, load_golden, rms

# fp32, same ATen kernels, different op grouping (banded rel-pos attention, dense spline): tolerance 2e-5 abs
TOL = 2e-5
STAGES = ["x", "m_p_tok", "logs_p_tok", "logw_sdp", "logw_dp", "m_p", "logs_p", "z_p", "z", "o", "y_mask"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_matches_reference_golden(name):
    meta, gold = load_golden(name)
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)
    assert torch.equal(st["w_ceil"], gold["w_ceil"]), "durations (ceil) must match exactly"
    assert torch.equal(st["y_lengths"], gold["y_lengths"])
    for k in STAGES:
        assert st[k].shape == gold[k].shape, k
        err = float((st[k] - gold[k]).abs().max())
        assert err < TOL, (k, err)
    assert rms(st["o"], gold["o"]) < 1e-6


def test_attn_path_is_monotonic_one_hot():
    meta, gold = load_golden("tflow_b3")
    cfg, sd, inp, nw, nz, kw = case_inputs(meta)
    o, attn, y_mask, _ = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, **kw)
    assert attn.shape[1] == 1
    # every valid frame maps to exactly one token, and durations sum to y_lengths (commons.py:126-140)
    assert torch.equal(attn.sum(3).squeeze(1), y_mask.squeeze(1))
    assert torch.equal(attn.sum(2), gold["w_ceil"])


def test_spline_identity_outside_tails():
    x = torch.tensor([[-7.0, -5.0, 0.3, 5.0, 6.5]])
    uw = torch.randn(1, 5, 10)
    uh = torch.randn(1, 5, 10)
    ud = torch.randn(1, 5, 9)
    y = O.rq_spline_inverse(x, uw, uh, ud)
    assert y[0, 0] == -7.0 and y[0, 4] == 6.5  # linear tails: identity (transforms.py:61-74)
    assert abs(float(y[0, 1]) + 5.0) < 1e-4 and abs(float(y[0, 3]) - 5.0) < 1e-4  # knots map to knots
    assert -5.0 < float(y[0, 2]) < 5.0


@pytest.mark.parametrize("flow", ["tflow", "wnflow"])
def test_spec_matches_reference_state_dict_keys(flow):
    from bert_vits2_b200.spec import ModelConfig, param_specs
    ref = json.load(open(os.path.join(GOLDEN_DIR, f"state_dict_keys_{flow}.json")))
    cfg = ModelConfig(use_transformer_flow=(flow == "tflow"))
    mine = [[p.key, list(p.shape)] for p in param_specs(cfg)]
    assert mine == ref


def test_oracle_vs_live_reference_fresh_seeds():
    """The oracle against the UNMODIFIED reference's stages on seeds and shapes no other fixture covers (stored in
    tests/golden/fresh_cases.npz by oracle/validate_against_reference.py --store), every stage compared."""
    from oracle.validate_against_reference import validate
    for ci, errs, dur_ok in validate():
        assert dur_ok, f"case {ci}: ceil(durations) differ"
        for k, e in errs.items():
            assert e < TOL, (ci, k, e)
