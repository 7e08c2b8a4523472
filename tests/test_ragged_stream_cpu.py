"""Host side of ragged streams (no GPU needed): the C-ABI entry point is declared, typed and exported; Engine.infer_finish_stream picks
it for ragged=True with the arguments of the bounded stream; SynthesizerTrn.infer_stream(ragged=True) rejects fp32 / TF32 modules
before anything else, and an FP16 module on the CPU refuses like any other infer_stream()."""
import os
import re
import types

import pytest
import torch

from bert_vits2_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ragged_stream_symbol_declared_typed_and_exported():
    _lib.build()
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "bv2.h")).read()
    name = "bv2_infer_finish_stream_ragged"
    m = re.search(r"\b" + name + r"\s*\(([^;]*)\);", hdr)
    assert m, name
    args = [a.strip() for a in m.group(1).split(",")]
    bounded = re.search(r"\bbv2_infer_finish_stream_bounded\s*\(([^;]*)\);", hdr)
    assert args == [a.strip() for a in bounded.group(1).split(",")]  # the bounded stream's arguments
    assert len(args) == 14 == len(_lib.SYMBOLS[name][1])
    assert _lib.SYMBOLS[name] == _lib.SYMBOLS["bv2_infer_finish_stream_bounded"]
    assert hasattr(lib, name)
    # null engine / missing output are rejected before anything touches a device
    assert lib.bv2_infer_finish_stream_ragged(None, None, 0, 0.0, -1, 0, None, None, None, None, None, None, None, None) != 0


class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("bv2_infer_finish_stream"):
            raise AttributeError(name)
        return lambda *a: self.calls.append((name, a)) or 0


@pytest.mark.parametrize("ragged", [False, True])
def test_engine_infer_finish_stream_picks_the_ragged_entry(ragged):
    from bert_vits2_b200.engine import Engine
    eng = Engine.__new__(Engine)
    eng.lib, eng.cfg, eng.device, eng._h = _FakeLib(), types.SimpleNamespace(inter_channels=4, hop=8), torch.device("cpu"), None
    eng._stream = lambda: None
    o, attn, y_mask, aux = eng.infer_finish_stream(2, 3, 10, torch.zeros(2, 4, 12), 0.6, 7, want_attn=False, max_chunk_frames=5, ragged=ragged)
    assert o.shape == (2, 1, 7 * 8) and attn is None
    (name, a), = eng.lib.calls
    assert name == ("bv2_infer_finish_stream_ragged" if ragged else "bv2_infer_finish_stream_bounded")
    assert a[2:6] == (12, 0.6, 7, 5)  # noise_ld, noise_scale, max_len, max_chunk_frames


@pytest.mark.parametrize("precision", ["fp16", "fp16g", "fp32", "tf32"])
def test_module_infer_stream_ragged_checks_without_gpu(precision):
    from bert_vits2_b200.engine import Bv2Error
    from bert_vits2_b200.models import SynthesizerTrn
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=4, gin_channels=512, precision=precision, init_seed=None).eval()
    x = torch.zeros(1, 5, dtype=torch.int64)
    f = torch.zeros(1, 1024, 5)
    with pytest.raises(ValueError if precision in ("fp32", "tf32") else Bv2Error):
        next(net.infer_stream(x, torch.tensor([5]), torch.zeros(1, dtype=torch.int64), x, x, f, f, f, ragged=True))
    with pytest.raises(Bv2Error):  # the default stays padded, and is refused on the CPU like before
        next(net.infer_stream(x, torch.tensor([5]), torch.zeros(1, dtype=torch.int64), x, x, f, f, f))
