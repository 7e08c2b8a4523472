"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/bv2.h
declares (no compute without a GPU), and the Python class mirrors the reference's state_dict interface."""
import json
import os
import re

import pytest
import torch

from bert_vits2_b200 import _lib
from util import GOLDEN_DIR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    _lib.build()
    return _lib.load()


def test_library_exports_every_header_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "bv2.h")).read()
    declared = set(re.findall(r"\b(bv2_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"bv2_engine", "bv2_config", "bv2_status"}
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.bv2_version()


def test_create_fails_loudly_without_gpu(lib):
    import ctypes as C
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = C.c_void_p()
    cfg = _lib.Bv2Config()
    assert lib.bv2_create(C.byref(h), C.byref(cfg), 0) != 0 and not h.value  # no CPU fallback exists


def test_config_struct_layout_matches_header():
    import ctypes as C
    # 20 scalars + 2*8 + 2 + 4 + 16 + 5 + float + 4 + n_flows = 70 int32-sized fields
    assert C.sizeof(_lib.Bv2Config) == 4 * (20 + 16 + 2 + 4 + 16 + 5 + 1 + 4 + 1)


@pytest.mark.parametrize("flow", ["tflow", "wnflow"])
def test_dropin_state_dict_matches_reference_keys(flow):
    from bert_vits2_b200.models import SynthesizerTrn
    ref = json.load(open(os.path.join(GOLDEN_DIR, f"state_dict_keys_{flow}.json")))
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=850, gin_channels=512, use_transformer_flow=(flow == "tflow"),
                         init_seed=None)
    got = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    assert got == ref
    # utils.load_checkpoint semantics (reference utils.py:85-114): extra enc_q.* keys are tolerated with strict=False
    sd = net.state_dict()
    sd["enc_q.pre.weight"] = torch.zeros(192, 1025, 1)
    r = net.load_state_dict(sd, strict=False)
    assert r.unexpected_keys == ["enc_q.pre.weight"] and not r.missing_keys


def test_unsupported_configurations_raise():
    from bert_vits2_b200.models import SynthesizerTrn
    args = (112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512, [16, 16, 8, 2, 2])
    with pytest.raises(ValueError):
        SynthesizerTrn(*args, n_speakers=0, gin_channels=512, init_seed=None)
    with pytest.raises(ValueError):
        SynthesizerTrn(*args, n_speakers=4, gin_channels=512, flow_share_parameter=True, init_seed=None)


def _mk(**kw):
    from bert_vits2_b200.models import SynthesizerTrn
    args = dict(n_speakers=850, gin_channels=512, init_seed=None)
    args.update(kw)
    return SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                          [16, 16, 8, 2, 2], **args)


def test_dropin_error_behaviour_without_gpu():
    """Unsupported configurations raise ValueError at construction like the reference's own checks; a CPU module refuses to
    infer (no CPU path exists) and forward() is out of scope."""
    from bert_vits2_b200.engine import Bv2Error
    with pytest.raises(ValueError):
        _mk(n_speakers=0)
    with pytest.raises(ValueError):
        _mk(flow_share_parameter=True)
    with pytest.raises(ValueError):
        _mk(use_spk_conditioned_encoder=False)
    net = _mk().eval()
    T = 5
    x = torch.zeros(1, T, dtype=torch.int64)
    f = torch.zeros(1, 1024, T)
    with pytest.raises(Bv2Error):
        net.infer(x, torch.tensor([T]), torch.zeros(1, dtype=torch.int64), x, x, f, f, f)
    with pytest.raises(NotImplementedError):
        net(x)
