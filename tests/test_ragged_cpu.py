"""Host side of ragged batches (no GPU needed): infer_batch forwards `ragged` to the module's infer() and trims each utterance as
before; the two C-ABI entry points are declared, typed and exported; a CPU module refuses like any other infer()."""
import ctypes as C
import os
import re
import types

import numpy as np
import pytest
import torch

from bert_vits2_b200 import _lib
from bert_vits2_b200.infer_api import infer_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _FakeNet(torch.nn.Module):
    """2 frames per phone; each sample is the phone id of its token, and -1 past the utterance's own frames when ragged (so a trim
    that kept a ragged utterance's zero tail, or dropped its samples, would show)."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.cfg = types.SimpleNamespace(hop=4)
        self.kw = []

    def infer(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, **kw):
        self.kw.append(kw)
        B, T = x.shape
        F = 2 * T
        tok = torch.arange(F) // 2
        val = x[:, tok].float()
        y_mask = (torch.arange(F)[None, :] < (2 * x_lengths)[:, None]).float()
        if kw.get("ragged"):
            val = torch.where(y_mask > 0, val, torch.full_like(val, -1.0))
        return val.repeat_interleave(self.cfg.hop, dim=1).unsqueeze(1), None, y_mask.unsqueeze(1), None


def _item(t, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(8, t, generator=g), torch.randn(8, t, generator=g), torch.randn(8, t, generator=g),
            torch.randint(1, 100, (t,), generator=g), torch.randint(0, 5, (t,), generator=g), torch.zeros(t, dtype=torch.int64))


@pytest.mark.parametrize("ragged", [False, True])
def test_infer_batch_forwards_ragged_and_trims(ragged):
    lens = [11, 3, 7, 3, 12, 6, 1]
    items = [_item(t, 20 + i) for i, t in enumerate(lens)]
    net = _FakeNet()
    outs = infer_batch(net, items, sid=1, batch_size=3, ragged=ragged)
    assert len(net.kw) == 3 and all(kw["ragged"] is ragged for kw in net.kw)
    for it, t, o in zip(items, lens, outs):
        assert o.dtype == np.float32 and o.shape == (2 * t * 4,)
        assert np.array_equal(o, it[3].float().repeat_interleave(8).numpy())


def test_infer_batch_default_is_padded():
    net = _FakeNet()
    infer_batch(net, [_item(4, 0), _item(9, 1)], sid=0)
    assert net.kw[0]["ragged"] is False


def test_ragged_symbols_declared_typed_and_exported():
    _lib.build()
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "bv2.h")).read()
    for name, nargs in (("bv2_infer_finish_ragged", 14), ("bv2_generator_ragged", 8)):
        m = re.search(r"\b" + name + r"\s*\(([^;]*)\);", hdr)
        assert m, name
        assert len(m.group(1).split(",")) == nargs == len(_lib.SYMBOLS[name][1])
        assert hasattr(lib, name)
    # null engine / missing arrays are rejected before anything touches a device
    assert lib.bv2_generator_ragged(None, 1, 1, None, None, None, None, None) != 0
    assert lib.bv2_infer_finish_ragged(None, None, 0, 0.0, -1, None, None, None, None, None, None, None, None, None) != 0


@pytest.mark.parametrize("precision", ["fp16", "fp16g", "fp32", "tf32"])
def test_module_ragged_checks_without_gpu(precision):
    """fp32 / TF32 modules reject ragged=True as an argument error before anything else; an FP16 module on CPU refuses like any
    infer() (no CPU path)."""
    from bert_vits2_b200.engine import Bv2Error
    from bert_vits2_b200.models import SynthesizerTrn
    net = SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                         [16, 16, 8, 2, 2], n_speakers=4, gin_channels=512, precision=precision, init_seed=None).eval()
    x = torch.zeros(1, 5, dtype=torch.int64)
    f = torch.zeros(1, 1024, 5)
    with pytest.raises(ValueError if precision in ("fp32", "tf32") else Bv2Error):
        net.infer(x, torch.tensor([5]), torch.zeros(1, dtype=torch.int64), x, x, f, f, f, ragged=True)
