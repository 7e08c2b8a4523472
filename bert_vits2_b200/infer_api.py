"""Caller-side batching for the reference's glue (SURVEY.md §8f item 2).

The reference serves one text slice per `net_g.infer` call (B is always 1 on the webui path: webui.py:65-87,
infer.py:302-318) and syncs + empties the CUDA cache after each.  `infer_batch` takes a list of `get_text()` outputs
(reference infer.py:107-148: bert, ja_bert, en_bert, phones, tones, lang_ids), length-buckets them, pads each bucket
and calls the engine once per bucket; results come back in the input order, trimmed to their own length.
Padding semantics follow the reference exactly (SURVEY.md §7 H4: the flow/Generator run over the padded length), so an
utterance's samples can differ from its B=1 result only in its last ~14 frames.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from .models import speaker_mixes
from .sharding import deal_buckets


def pad_items(items: Sequence[Tuple[torch.Tensor, ...]], device) -> dict:
    """items: (bert [1024,T], ja_bert, en_bert, phones [T], tones [T], lang_ids [T]) per utterance."""
    B = len(items)
    T = max(int(it[3].shape[0]) for it in items)
    D = int(items[0][0].shape[0])
    out = {
        "x": torch.zeros(B, T, dtype=torch.int64), "tone": torch.zeros(B, T, dtype=torch.int64),
        "language": torch.zeros(B, T, dtype=torch.int64), "x_lengths": torch.zeros(B, dtype=torch.int64),
        "bert": torch.zeros(B, D, T), "ja_bert": torch.zeros(B, D, T), "en_bert": torch.zeros(B, D, T),
    }
    for b, (bert, ja, en, ph, tn, lg) in enumerate(items):
        t = int(ph.shape[0])
        assert bert.shape[-1] == t and ja.shape[-1] == t and en.shape[-1] == t, "bert features must match the phone count (infer.py:124)"
        out["x"][b, :t] = ph; out["tone"][b, :t] = tn; out["language"][b, :t] = lg; out["x_lengths"][b] = t
        out["bert"][b, :, :t] = bert; out["ja_bert"][b, :, :t] = ja; out["en_bert"][b, :, :t] = en
    return {k: v.to(device, non_blocking=True) for k, v in out.items()}


def _per_item(name, v, n):
    """v as a list of n per-item values, or None when it is one value for every item"""
    if np.ndim(v) == 0:
        return None
    vals = v.tolist() if hasattr(v, "tolist") else list(v)
    if len(vals) != n or any(np.ndim(x) != 0 for x in vals):
        raise ValueError(f"{name}: expected one value or {n} per-item values in item order")
    return vals


@torch.no_grad()
def infer_batch(net, items: Sequence[Tuple[torch.Tensor, ...]], sid=None, batch_size: int = 32, sdp_ratio=0.2, noise_scale=0.6,
                noise_scale_w=0.8, length_scale=1.0, ragged=False, speaker_mix=None) -> List[np.ndarray]:
    """Returns one float32 waveform per item (same order), as infer.infer returns for a single slice (infer.py:315-318).
    `ragged=True` is passed to net.infer: the Generator then runs each utterance at its own length, so no utterance pays for the
    longest one of its bucket and none sees the padding in its last frames (FP16 Generator only; see SynthesizerTrn.infer).
    `sid` and each setting take one value for every item or a sequence of per-item values in item order (a webui dialogue whose
    sentences have their own speaker and speed).  Buckets depend on the lengths alone, so items with different speakers or settings
    share a call, each synthesised with its own values (SynthesizerTrn.infer).
    `speaker_mix` replaces `sid` (ValueError with both, or with neither): one dict {speaker_id: weight} for every item or one dict
    per item in item order, each item conditioned on its own weighted mix of speakers (models.speaker_mixes)."""
    dev = next(net.parameters()).device
    lengths = [int(it[3].shape[0]) for it in items]
    settings = dict(sdp_ratio=sdp_ratio, noise_scale=noise_scale, noise_scale_w=noise_scale_w, length_scale=length_scale)
    per_item = {k: _per_item(k, v, len(items)) for k, v in settings.items()}
    if (sid is None) == (speaker_mix is None):
        raise ValueError("infer_batch takes either sid or speaker_mix")
    if speaker_mix is None:
        sid_items = _per_item("sid", sid, len(items))
    else:
        speaker_mixes(len(items), speaker_mix)  # validates every mix before the first call
        mixes = [speaker_mix] * len(items) if isinstance(speaker_mix, dict) else list(speaker_mix)
    plan = deal_buckets(lengths, world_size=1, batch_size=batch_size)[0]
    hop = net.cfg.hop
    results: List[np.ndarray] = [None] * len(items)
    for bucket in plan:
        d = pad_items([items[i] for i in bucket], dev)
        kw = {k: v if per_item[k] is None else [per_item[k][i] for i in bucket] for k, v in settings.items()}
        if speaker_mix is not None:
            sids = None
            kw["speaker_mix"] = [mixes[i] for i in bucket]
        elif sid_items is None:
            sids = torch.full((len(bucket),), int(sid), dtype=torch.int64, device=dev)
        else:
            sids = torch.tensor([int(sid_items[i]) for i in bucket], dtype=torch.int64, device=dev)
        o, _, y_mask, _ = net.infer(d["x"], d["x_lengths"], sids, d["tone"], d["language"], d["bert"], d["ja_bert"], d["en_bert"],
                                    **kw, ragged=ragged)
        n = (y_mask.sum((1, 2)).long() * hop).cpu()
        wav = o[:, 0].float().cpu().numpy()
        for k, i in enumerate(bucket):
            results[i] = wav[k, : int(n[k])].copy()
    return results
