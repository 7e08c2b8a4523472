#!/usr/bin/env python
"""Pin the oracle against the unmodified reference on seeds no other fixture uses (not the committed golden cases).

TEST INFRASTRUCTURE ONLY.
    python oracle/validate_against_reference.py            # live: reference vs oracle, max-abs error per stage (needs the reference)
    python oracle/validate_against_reference.py --store    # write the reference's stages of FRESH_CASES to tests/golden/fresh_cases.npz
tests/test_oracle_golden.py::test_oracle_vs_live_reference_fresh_seeds runs `validate()` against the stored reference stages, so a
drift between the restatement (oracle/vits2_oracle.py) and reference models.py:1026-1074 shows up in the CPU suite on inputs the
other fixtures do not cover (different lengths, languages, sdp_ratio, length_scale, max_len, spline tails, n_flow_layer).
"""
import importlib.util
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bert_vits2_b200 import synth  # noqa: E402
from bert_vits2_b200.spec import ModelConfig  # noqa: E402
from oracle import ref_import, vits2_oracle as O  # noqa: E402

STAGES = ["x", "m_p_tok", "logs_p_tok", "logw_sdp", "logw_dp", "m_p", "logs_p", "z_p", "z", "o", "y_mask"]

#: (use_transformer_flow, lengths, languages, infer kwargs, seeds (weights, inputs, noise))
FRESH_CASES = [
    (True, [13, 20], [1, 0], dict(sdp_ratio=0.2, noise_scale=0.667, noise_scale_w=0.8, length_scale=1.1), (5, 6, 7)),
    (False, [18], [2], dict(sdp_ratio=1.0, noise_scale=0.3, noise_scale_w=0.5, length_scale=0.9), (8, 9, 10)),
    (True, [1], [0], dict(sdp_ratio=0.0, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0), (11, 12, 13)),
    # train_ms.evaluate-style call: the decoder input is cut to max_len frames (models.py:1073)
    (False, [15, 11], [0, 1], dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0, max_len=20), (14, 15, 16)),
    # spline tails: noise_scale_w = 8 pushes the SDP latent beyond the +-5 tail bound (identity branch, transforms.py:61-74) and onto
    # the outermost bins; sdp_ratio = 0 keeps exp(logw_sdp) out of the durations (the logw_sdp stage itself is compared)
    (True, [24, 9], [0, 2], dict(sdp_ratio=0.0, noise_scale=0.6, noise_scale_w=8.0, length_scale=1.0), (17, 18, 19)),
    # WN flow with n_flow_layer != 4: ResidualCouplingBlock receives n_flow_layer as n_layers, n_flows stays 4 (models.py:918-919)
    (False, [14], [1], dict(sdp_ratio=0.5, noise_scale=0.6, noise_scale_w=0.9, length_scale=1.0), (20, 21, 22), dict(n_flow_layer=3)),
]


def _golden_tools():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(ROOT, "tests", "golden", "make_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


GOLDEN = os.path.join(ROOT, "tests", "golden", "fresh_cases.npz")
REF_ARGS = os.path.join(ROOT, "tests", "golden", "reference_get_net_g_args.json")


def _case(case, f_cap):
    tflow, lengths, langs, kw, (ws, is_, ns) = case[:5]
    model_kw = case[5] if len(case) > 5 else {}
    hps_model = json.load(open(REF_ARGS))["model"]  # the reference's configs/config.json model section, recorded
    cfg = ModelConfig.from_hps_model(dict(hps_model, **model_kw), use_transformer_flow=tflow)
    sd = synth.synthetic_state_dict(cfg, ws)
    inp = synth.synthetic_inputs(cfg, lengths, langs, seed=is_)
    nw, nz = synth.synthetic_noise(cfg, len(lengths), max(lengths), f_cap, seed=ns)
    return tflow, model_kw, kw, cfg, sd, inp, nw, nz


def reference_stages(cases=FRESH_CASES, f_cap=512):
    """The live reference's stages of every case (needs the reference tree)."""
    mg = _golden_tools()
    out = []
    for case in cases:
        tflow, model_kw, kw, cfg, sd, inp, nw, nz = _case(case, f_cap)
        net, hps = ref_import.build_reference_net(tflow, **model_kw)
        missing, unexpected = net.load_state_dict(sd, strict=False)
        assert not unexpected and all(k.startswith("enc_q.") for k in missing)
        ref = mg.run_reference(net, inp, nw, nz, **kw)
        out.append({k: ref[k] for k in STAGES + ["w_ceil"]})
    return out


SAMPLE = 4096  # stages with more elements are stored as a fixed, seeded sample of this many elements (the file stays small)


def _sample_idx(ci, k, size):
    """Flat indices of the stored sample of stage k of case ci (None: the whole stage is stored)."""
    if size <= SAMPLE:
        return None
    rng = np.random.default_rng(1000 * ci + (STAGES + ["w_ceil"]).index(k))
    return np.sort(rng.choice(size, SAMPLE, replace=False))


def store(path=GOLDEN):
    arrs = {}
    for ci, ref in enumerate(reference_stages()):
        for k, v in ref.items():
            a = v.detach().cpu().float().numpy()
            idx = _sample_idx(ci, k, a.size)
            arrs[f"c{ci}_{k}"] = a if idx is None else a.reshape(-1)[idx]
            arrs[f"c{ci}_{k}_shape"] = np.array(a.shape, dtype=np.int64)
    np.savez_compressed(path, **arrs)


def stored_stages(path=GOLDEN, n=len(FRESH_CASES)):
    """[{stage: (shape, flat indices or None, values)}] of the stored reference stages."""
    z = np.load(path)
    out = []
    for ci in range(n):
        d = {}
        for k in STAGES + ["w_ceil"]:
            shape = tuple(int(x) for x in z[f"c{ci}_{k}_shape"])
            d[k] = (shape, _sample_idx(ci, k, int(np.prod(shape))), torch.from_numpy(z[f"c{ci}_{k}"]))
        out.append(d)
    return out


def validate(cases=FRESH_CASES, f_cap=512, live=False):
    """Returns [(case index, {stage: max abs error}, durations_equal)] of the oracle against the reference's stages: the stored
    ones (tests/golden/fresh_cases.npz: whole small stages, a seeded sample of large ones) or, with live=True, the reference run now."""
    if live:
        refs = [{k: (tuple(v.shape), None, v) for k, v in r.items()} for r in reference_stages(cases, f_cap)]
    else:
        refs = stored_stages(n=len(cases))
    out = []
    for ci, (case, ref) in enumerate(zip(cases, refs)):
        tflow, model_kw, kw, cfg, sd, inp, nw, nz = _case(case, f_cap)
        st = O.infer(sd, cfg, **inp, noise_w=nw, noise_z=nz, return_stages=True, **kw)

        def pick(k):
            shape, idx, val = ref[k]
            assert tuple(st[k].shape) == shape, (ci, k, tuple(st[k].shape), shape)
            mine = st[k].detach().float()
            if idx is not None:
                mine = mine.reshape(-1)[torch.from_numpy(idx)]
            return mine, val.float().reshape(mine.shape)

        errs = {}
        for k in STAGES:
            a, r = pick(k)
            errs[k] = float((a - r).abs().max())
        a, r = pick("w_ceil")
        out.append((ci, errs, bool(torch.equal(a, r))))
    return out


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("reference not present at " + ref_import.REF)
    if "--store" in sys.argv:
        store()
        sys.exit(0)
    for ci, errs, dur_ok in validate(live=True):
        print(f"case {ci}: durations equal={dur_ok}  " + "  ".join(f"{k}={v:.1e}" for k, v in errs.items()))
