"""Per-utterance synthesis settings on CPU: the C entry point is declared, typed and exported; SynthesizerTrn normalises and
validates the four settings without a GPU; infer_batch carries per-item speakers and settings through length-only buckets."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from bert_vits2_b200 import _lib
from bert_vits2_b200.infer_api import infer_batch
from bert_vits2_b200.models import item_settings
from test_infer_api_cpu import _FakeNet, _item

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_begin_items_declared_typed_and_exported():
    hdr = open(os.path.join(ROOT, "include", "bv2.h")).read()
    decl = re.search(r"int bv2_infer_begin_items\(([^)]*)\)", hdr)
    assert decl, "bv2_infer_begin_items is not declared"
    params = [p.strip() for p in decl.group(1).split(",")]
    restype, argtypes = _lib.SYMBOLS["bv2_infer_begin_items"]
    assert restype is C.c_int and len(argtypes) == len(params) == 20
    # bv2_infer_begin's arguments with the three setting scalars replaced by arrays, then the per-item noise scale
    assert [p.split()[-1].lstrip("*") for p in params[12:16]] == ["noise_scale_w", "length_scale", "sdp_ratio", "noise_scale"]
    assert all(p.startswith("const float*") for p in params[12:16])
    _lib.build()
    assert hasattr(_lib.load(), "bv2_infer_begin_items")


def test_item_settings_normalisation():
    B = 3
    s = item_settings(B, noise_scale=0.667, length_scale=1, noise_scale_w=torch.tensor(0.8), sdp_ratio=np.float32(0.25))
    assert s == {"noise_scale": 0.667, "length_scale": 1.0, "noise_scale_w": float(torch.tensor(0.8)), "sdp_ratio": 0.25}
    assert all(type(v) is float for v in s.values())
    s = item_settings(B, noise_scale=[0.1, 0.2, 0.3], length_scale=(1, 2, 3), noise_scale_w=np.array([0.5, 0.6, 0.7]),
                      sdp_ratio=torch.tensor([0.0, 0.5, 1.0], dtype=torch.float64))
    for k, v in s.items():
        assert isinstance(v, torch.Tensor) and v.dtype == torch.float32 and v.shape == (B,), k
    # fp32 rounding happens once, as a float passed to the scalar call rounds
    assert s["noise_scale"].tolist() == [float(np.float32(v)) for v in (0.1, 0.2, 0.3)]
    assert s["noise_scale_w"].tolist() == [float(np.float32(v)) for v in (0.5, 0.6, 0.7)]


@pytest.mark.parametrize("bad", [[1.0, 2.0], [1.0] * 4, [[1.0]] * 3, torch.ones(3, 1), torch.ones(2), np.ones((3, 2)), "fast", [1.0, "x", 2.0]])
def test_item_settings_rejects_wrong_length_or_rank(bad):
    with pytest.raises(ValueError):
        item_settings(3, length_scale=bad)


def _mk():
    from bert_vits2_b200.models import SynthesizerTrn
    return SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                          [16, 16, 8, 2, 2], n_speakers=850, gin_channels=512, init_seed=None)


def test_module_validates_settings_before_it_needs_a_gpu():
    """a wrong length or rank is a ValueError even on a CPU module (which cannot infer: Bv2Error once the settings are valid)"""
    from bert_vits2_b200.engine import Bv2Error
    net = _mk()
    T = 5
    x = torch.zeros(2, T, dtype=torch.int64)
    f = torch.zeros(2, 1024, T)
    args = (x, torch.tensor([T, T]), torch.zeros(2, dtype=torch.int64), x, x, f, f, f)
    for bad in (dict(noise_scale=[0.5]), dict(sdp_ratio=torch.zeros(2, 2)), dict(length_scale=[1.0, 1.0, 1.0])):
        with pytest.raises(ValueError):
            net.infer(*args, **bad)
        with pytest.raises(ValueError):
            next(net.infer_stream(*args, **bad))
    with pytest.raises(Bv2Error):
        net.infer(*args, noise_scale=[0.5, 0.6], length_scale=torch.tensor([1.0, 1.2]))


class _RecordingNet(_FakeNet):
    """_FakeNet that records the sid and settings of every call, per item in the order of its rows"""

    def infer(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, **kw):
        self.seen = getattr(self, "seen", [])
        self.seen.append((x[:, 0].tolist(), sid.tolist(), kw))
        return super().infer(x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, **kw)


def test_infer_batch_per_item_sid_and_settings():
    lens = [11, 3, 7, 3, 12, 6, 1]
    items = [_item(t, 10 + i) for i, t in enumerate(lens)]
    for i, it in enumerate(items):
        it[3][0] = 200 + i  # tells the items apart in the calls
    n = len(items)
    sids = [5, 1, 2, 1, 0, 7, 3]
    per = dict(sdp_ratio=[0.1 * i for i in range(n)], noise_scale=np.linspace(0.3, 0.9, n), noise_scale_w=0.8,
               length_scale=torch.tensor([1.0 + 0.05 * i for i in range(n)]))
    net, ref_net = _RecordingNet(), _FakeNet()
    outs = infer_batch(net, items, sid=sids, batch_size=3, **per)
    ref = infer_batch(ref_net, items, sid=3, batch_size=3)
    assert net.calls == ref_net.calls  # the buckets depend on the lengths alone
    assert len(outs) == n and all(np.array_equal(a, b) for a, b in zip(outs, ref))  # input order kept
    first_token = [int(it[3][0]) for it in items]
    seen_items = 0
    for row_tokens, row_sids, kw in net.seen:
        idx = [first_token.index(t) for t in row_tokens]  # which items this call holds, in row order
        seen_items += len(idx)
        assert row_sids == [sids[i] for i in idx]
        assert kw["sdp_ratio"] == [per["sdp_ratio"][i] for i in idx]
        assert kw["noise_scale"] == [per["noise_scale"][i] for i in idx]
        assert [float(v) for v in kw["length_scale"]] == [float(per["length_scale"][i]) for i in idx]
        assert kw["noise_scale_w"] == 0.8  # a setting given once still goes as a float
    assert seen_items == n
    assert any(len(set(s)) > 1 for _, s, _ in net.seen)  # items with different speakers share a call


def test_infer_batch_scalars_forward_as_before():
    items = [_item(t, i) for i, t in enumerate([4, 9, 2])]
    net = _RecordingNet()
    infer_batch(net, items, sid=3, batch_size=2, sdp_ratio=0.2, noise_scale=0.6, noise_scale_w=0.8, length_scale=1.0)
    for _, row_sids, kw in net.seen:
        assert set(row_sids) == {3}
        assert kw == dict(sdp_ratio=0.2, noise_scale=0.6, noise_scale_w=0.8, length_scale=1.0, ragged=False)


@pytest.mark.parametrize("arg", ["sid", "length_scale"])
def test_infer_batch_rejects_wrong_per_item_length(arg):
    items = [_item(t, i) for i, t in enumerate([4, 9, 2])]
    with pytest.raises(ValueError):
        infer_batch(_FakeNet(), items, **{"sid": 0, arg: [1, 1]})
