"""Host logic of the batched caller-side API (SURVEY.md section 8f item 2) on CPU: bucketing, padding, order and trimming
of infer_batch, with a stand-in module that has the reference's .infer() signature (no compute path is exercised)."""
import os
import types

import numpy as np
import torch

from bert_vits2_b200.infer_api import infer_batch, pad_items


class _FakeNet(torch.nn.Module):
    """Emits, per utterance, 2 frames per phone; sample value = phone id of the frame's token (+ 0.5 where the BERT row 0
    is positive) so that order, padding and trimming are all visible in the output."""

    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.cfg = types.SimpleNamespace(hop=4)
        self.calls = []

    def infer(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, **kw):
        B, T = x.shape
        self.calls.append((B, T, sorted(x_lengths.tolist())))
        assert bert.shape == (B, 8, T) and tone.shape == (B, T) and sid.shape == (B,)
        F = 2 * T
        tok = torch.arange(F) // 2
        val = x[:, tok].float() + 0.5 * (bert[:, 0, tok] > 0).float()
        o = val.repeat_interleave(self.cfg.hop, dim=1).unsqueeze(1)           # [B,1,F*hop]
        y_mask = (torch.arange(F)[None, :] < (2 * x_lengths)[:, None]).float().unsqueeze(1)
        return o, None, y_mask, None


def _item(t, seed):
    g = torch.Generator().manual_seed(seed)
    ph = torch.randint(1, 100, (t,), generator=g)
    return (torch.randn(8, t, generator=g), torch.randn(8, t, generator=g), torch.randn(8, t, generator=g), ph,
            torch.randint(0, 5, (t,), generator=g), torch.zeros(t, dtype=torch.int64))


def test_pad_items_shapes_and_zero_padding():
    items = [_item(5, 0), _item(9, 1), _item(7, 2)]
    d = pad_items(items, "cpu")
    assert d["x"].shape == (3, 9) and d["bert"].shape == (3, 8, 9) and d["x_lengths"].tolist() == [5, 9, 7]
    assert (d["x"][0, 5:] == 0).all() and (d["bert"][0, :, 5:] == 0).all() and torch.equal(d["x"][1], items[1][3])


def test_infer_batch_order_bucketing_and_trimming():
    lens = [11, 3, 7, 3, 12, 6, 1]
    items = [_item(t, 10 + i) for i, t in enumerate(lens)]
    net = _FakeNet()
    outs = infer_batch(net, items, sid=3, batch_size=3)
    assert len(outs) == len(items) and len(net.calls) == 3
    # buckets hold utterances of similar length (sorted dealing), every utterance exactly once
    assert sorted(sum((c[2] for c in net.calls), [])) == sorted(lens)
    assert all(max(c[2]) == c[1] for c in net.calls)
    for it, t, o in zip(items, lens, outs):
        assert isinstance(o, np.ndarray) and o.dtype == np.float32 and o.shape == (2 * t * 4,)
        expect = (it[3].float() + 0.5 * (it[0][0] > 0).float()).repeat_interleave(8).numpy()
        assert np.array_equal(o, expect)


def test_dropin_constructs_like_get_net_g_and_loads_a_checkpoint(tmp_path):
    """Build container only: the drop-in class, constructed exactly as the reference's infer.get_net_g does (infer.py:95-101) from
    the reference's own hps (tests/golden/reference_get_net_g_args.json, recorded from the unmodified reference config), exposes
    the reference model's state_dict keys (tests/golden/state_dict_keys_tflow.json) and ends up with exactly a checkpoint's tensors
    when loaded the way utils.load_checkpoint does (model entry of the file, strict=False; enc_q.* keys of un-compressed
    checkpoints are ignored, as compress_model.py drops them)."""
    import json
    import torch
    from bert_vits2_b200 import synth
    from bert_vits2_b200.models import SynthesizerTrn
    from bert_vits2_b200.spec import ModelConfig
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    a = json.load(open(os.path.join(gold, "reference_get_net_g_args.json")))
    ref_shapes = {k: list(shape) for k, shape in json.load(open(os.path.join(gold, "state_dict_keys_tflow.json")))}
    net = SynthesizerTrn(a["n_symbols"], a["spec_channels"], a["segment_frames"], n_speakers=a["n_speakers"], **a["model"])
    cfg = ModelConfig.from_hps_model(a["model"])
    sd = synth.synthetic_state_dict(cfg, 3)
    assert set(net.state_dict()) == set(sd) == set(ref_shapes)
    assert all(list(v.shape) == ref_shapes[k] for k, v in sd.items())
    ck = dict(sd)
    ck["enc_q.pre.weight"] = torch.zeros(192, 1025, 1)  # training-only module still present in un-compressed checkpoints
    path = str(tmp_path / "G_0.pth")
    torch.save({"model": ck, "iteration": 7, "optimizer": None, "learning_rate": 2e-4}, path)
    saved = torch.load(path, map_location="cpu")["model"]
    own = net.state_dict()
    net.load_state_dict({k: saved.get(k, v) for k, v in own.items()}, strict=False)
    got = net.state_dict()
    for k, v in sd.items():
        assert torch.equal(got[k], v), k


def test_oracle_pcm16_restatement():
    """The restated gradio conversion (oracle.convert_to_16_bit_wav): peak maps to +-32767, truncation toward zero."""
    import numpy as np
    from oracle import vits2_oracle as O
    x = np.array([0.0, 0.25, -0.5, 0.1234567, -0.49999], dtype=np.float32)
    y = O.convert_to_16_bit_wav(x)
    assert y.dtype == np.int16 and y[2] == -32767 and y[0] == 0 and y[1] == 16383 and y[4] == int(np.float32(-0.49999) / np.float32(0.5) * np.float32(32767))
