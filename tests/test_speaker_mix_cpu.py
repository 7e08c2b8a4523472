"""Speaker mixes on CPU: the C entry point is declared, typed and exported; speaker_mixes normalises and validates a mix without a
GPU; SynthesizerTrn rejects a sid together with a mix; infer_batch carries per-item mixes into the right rows of each bucket."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from bert_vits2_b200 import _lib
from bert_vits2_b200.infer_api import infer_batch
from bert_vits2_b200.models import speaker_mixes
from test_infer_api_cpu import _FakeNet, _item

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_begin_mix_declared_typed_and_exported():
    hdr = open(os.path.join(ROOT, "include", "bv2.h")).read()
    decl = re.search(r"int bv2_infer_begin_mix\(([^)]*)\)", hdr)
    assert decl, "bv2_infer_begin_mix is not declared"
    params = [p.strip() for p in decl.group(1).split(",")]
    restype, argtypes = _lib.SYMBOLS["bv2_infer_begin_mix"]
    assert restype is C.c_int and len(argtypes) == len(params) == 22
    # bv2_infer_begin_items' arguments with sid replaced by (K, mix_sid, mix_weight)
    items = _lib.SYMBOLS["bv2_infer_begin_items"][1]
    assert argtypes[:5] == items[:5] and argtypes[8:] == items[6:]
    assert [p.split()[-1].lstrip("*") for p in params[5:8]] == ["K", "mix_sid", "mix_weight"]
    assert params[5] == "int K" and params[6].startswith("const int64_t*") and params[7].startswith("const float*")
    assert argtypes[5] is C.c_int
    _lib.build()
    assert hasattr(_lib.load(), "bv2_infer_begin_mix")


def test_speaker_mixes_one_dict_for_every_utterance():
    ids, w = speaker_mixes(3, {4: 0.25, 7: 0.75})
    assert ids.dtype == torch.int64 and w.dtype == torch.float32 and ids.shape == w.shape == (3, 2)
    assert ids.tolist() == [[4, 7]] * 3
    assert w.tolist() == [[0.25, 0.75]] * 3


def test_speaker_mixes_sequence_order_and_padding():
    mixes = [{5: 1.0}, {9: 0.2, 2: -0.3}, {np.int64(3): np.float32(0.5), 0: 0.5, 849: 2.0}]
    ids, w = speaker_mixes(3, mixes)
    assert ids.shape == w.shape == (3, 3)
    # dict order is summation order; a shorter mix is padded at the end with (its first id, 0.0)
    assert ids.tolist() == [[5, 5, 5], [9, 2, 9], [3, 0, 849]]
    assert w[0].tolist() == [1.0, 0.0, 0.0]
    assert w[1].tolist() == [float(np.float32(0.2)), float(np.float32(-0.3)), 0.0]
    assert w[2].tolist() == [0.5, 0.5, 2.0]
    # weights are used as given (no normalisation), and a tuple of dicts is a sequence too
    ids, w = speaker_mixes(2, ({1: 3.0, 2: -5.0}, {7: 0.0}))
    assert w.tolist() == [[3.0, -5.0], [0.0, 0.0]] and ids.tolist() == [[1, 2], [7, 7]]


@pytest.mark.parametrize("bad", [
    {}, [{}, {1: 1.0}], {"1": 1.0}, {1.0: 1.0}, {True: 1.0}, {np.bool_(False): 1.0}, {1: math.nan}, {1: math.inf}, {1: -math.inf},
    {1: 1e39}, {1: "x"}, [{1: 1.0}], [{1: 1.0}] * 3, [{1: 1.0}, 1], 5, "ab"])
def test_speaker_mixes_rejects(bad):
    with pytest.raises(ValueError):
        speaker_mixes(2, bad)


def _mk():
    from bert_vits2_b200.models import SynthesizerTrn
    return SynthesizerTrn(112, 1025, 32, 192, 192, 768, 2, 6, 3, 0.1, "1", [3, 7, 11], [[1, 3, 5]] * 3, [8, 8, 2, 2, 2], 512,
                          [16, 16, 8, 2, 2], n_speakers=850, gin_channels=512, init_seed=None)


def test_module_rejects_sid_with_mix_before_it_needs_a_gpu():
    """a sid together with a mix, or a malformed mix, is a ValueError even on a CPU module (which cannot infer: Bv2Error once the
    arguments are valid)"""
    from bert_vits2_b200.engine import Bv2Error
    net = _mk()
    T = 5
    x = torch.zeros(2, T, dtype=torch.int64)
    f = torch.zeros(2, 1024, T)
    sid = torch.zeros(2, dtype=torch.int64)
    args = lambda s: (x, torch.tensor([T, T]), s, x, x, f, f, f)  # noqa: E731
    for s, mix in ((sid, {1: 1.0}), (None, {}), (None, [{1: 1.0}]), (None, {1: math.nan})):
        with pytest.raises(ValueError):
            net.infer(*args(s), speaker_mix=mix)
        with pytest.raises(ValueError):
            next(net.infer_stream(*args(s), speaker_mix=mix))
    with pytest.raises(Bv2Error):
        net.infer(*args(None), speaker_mix=[{1: 0.5, 2: 0.5}, {3: 1.0}])


class _RecordingNet(_FakeNet):
    """_FakeNet that records the sid and speaker mix of every call, per item in the order of its rows"""

    def infer(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, **kw):
        self.seen = getattr(self, "seen", [])
        self.seen.append((x[:, 0].tolist(), sid, kw))
        if sid is None:
            sid = torch.zeros(x.shape[0], dtype=torch.int64)
        return super().infer(x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, **kw)


def test_infer_batch_routes_per_item_mixes():
    lens = [11, 3, 7, 3, 12, 6, 1]
    items = [_item(t, 30 + i) for i, t in enumerate(lens)]
    for i, it in enumerate(items):
        it[3][0] = 200 + i  # tells the items apart in the calls
    n = len(items)
    mixes = [{i: 1.0} if i % 2 else {i: 0.5, 100 + i: 0.25, 3: 0.25} for i in range(n)]
    net, ref_net = _RecordingNet(), _FakeNet()
    outs = infer_batch(net, items, batch_size=3, speaker_mix=mixes, noise_scale=[0.1 * i for i in range(n)])
    ref = infer_batch(ref_net, items, sid=3, batch_size=3)
    assert net.calls == ref_net.calls  # the buckets depend on the lengths alone
    assert len(outs) == n and all(np.array_equal(a, b) for a, b in zip(outs, ref))  # input order kept
    first_token = [int(it[3][0]) for it in items]
    seen_items = 0
    for row_tokens, sid, kw in net.seen:
        idx = [first_token.index(t) for t in row_tokens]  # which items this call holds, in row order
        seen_items += len(idx)
        assert sid is None
        assert kw["speaker_mix"] == [mixes[i] for i in idx]
        assert kw["noise_scale"] == [0.1 * i for i in idx]
    assert seen_items == n
    # one dict goes to every item
    net = _RecordingNet()
    infer_batch(net, items, batch_size=4, speaker_mix={2: 0.5, 5: 0.5})
    assert all(kw["speaker_mix"] == [{2: 0.5, 5: 0.5}] * len(rows) for rows, _, kw in net.seen)


@pytest.mark.parametrize("kw", [dict(sid=0, speaker_mix={1: 1.0}), dict(), dict(speaker_mix=[{1: 1.0}] * 2), dict(speaker_mix={})])
def test_infer_batch_rejects_bad_mix_before_any_call(kw):
    items = [_item(t, i) for i, t in enumerate([4, 9, 2])]
    net = _RecordingNet()
    with pytest.raises(ValueError):
        infer_batch(net, items, **kw)
    assert not net.calls
