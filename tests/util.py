"""Shared helpers for the parity tests (golden loading, synthetic model/case regeneration, the kernel tests' error report)."""
import ast
import functools
import os

import numpy as np
import pytest
import torch

from bert_vits2_b200 import synth
from bert_vits2_b200.spec import ModelConfig

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_CASES = ["tflow_b1", "wnflow_b1", "tflow_b3", "wnflow_b3"]


def load_golden(name):
    d = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    meta = ast.literal_eval(str(d["meta"]))
    arrays = {k: torch.from_numpy(d[k]) for k in d.files if k != "meta"}
    return meta, arrays


@functools.lru_cache(maxsize=4)
def model_for(use_transformer_flow: bool, weight_seed: int = 0):
    cfg = ModelConfig(use_transformer_flow=use_transformer_flow)
    sd = synth.synthetic_state_dict(cfg, weight_seed)
    return cfg, sd


def case_inputs(meta):
    cfg, sd = model_for(meta["use_transformer_flow"], meta["weight_seed"])
    inp = synth.synthetic_inputs(cfg, meta["lengths"], meta["languages"], seed=meta["input_seed"])
    nw, nz = synth.synthetic_noise(cfg, len(meta["lengths"]), max(meta["lengths"]), meta["f_cap"], seed=meta["noise_seed"])
    kw = {k: meta[k] for k in ("sdp_ratio", "noise_scale", "noise_scale_w", "length_scale")}
    return cfg, sd, inp, nw, nz, kw


def rms(a, b):
    return float((a.double() - b.double()).pow(2).mean().sqrt())


def report(cid, plan, err, tol, mag, ok_mask, coords):
    """prints the case line (plan, worst err/mag) and fails with the location and plan of the worst element"""
    ratio = np.where(ok_mask, err / np.maximum(tol, 1e-30), 0.0)
    bad = ok_mask & ~(err <= tol)
    emag = float(np.max(np.where(ok_mask & (mag > 0), err / np.maximum(mag, 1e-30), 0.0))) if ok_mask.any() else 0.0
    print(f"\n  {cid}: {plan} | worst err/mag {emag:.2e}, worst err/tol {float(ratio.max()) if ratio.size else 0.0:.3f}")
    if bad.any():
        idx = np.unravel_index(np.argmax(ratio), ratio.shape)
        pytest.fail(f"{cid}: {int(bad.sum())} element(s) out of bound; worst at {coords}={tuple(int(i) for i in idx)}: "
                    f"err {float(err[idx]):.3e} > tol {float(tol[idx]):.3e} (mag {float(mag[idx]):.3e}); plan {plan}")
