"""Drop-in for the reference `models.SynthesizerTrn` on the inference path.

Mirrors (names, argument meaning, return values, error behaviour):
  * constructor: reference models.py:816-935 as called by infer.get_net_g (infer.py:95-101):
        SynthesizerTrn(len(symbols), filter_length // 2 + 1, segment_size // hop_length,
                       n_speakers=hps.data.n_speakers, **hps.model)
  * .to(device) / .eval() / .state_dict() / .load_state_dict(): the parameters are registered under the
    reference's state_dict keys (spec.py), so utils.load_checkpoint (reference utils.py:65-120) works
    unmodified; `enc_q.*` keys in a checkpoint are ignored (strict=False there), as compress_model.py drops them.
  * .infer(...): reference models.py:1026-1074, same signature, returns
        (o [B,1,L], attn [B,1,F,T], y_mask [B,1,F], (z, z_p, m_p, logs_p))

Only tensor plumbing happens here.  All arithmetic runs in libbv2.so (CUDA, sm_90a); there is no PyTorch or
CPU fallback — calling .infer() on a CPU module raises.
"""
from __future__ import annotations

import contextlib
import threading
from typing import Optional

import numpy as np
import torch
from torch import nn

from . import synth
from .engine import Bv2Error, Engine
from .pool import EnginePool
from .spec import ModelConfig, param_specs

_ENGINE_LOCK = threading.Lock()  # builds a module's engine and pool once when several threads make its first call together


def item_settings(B: int, **settings):
    """Each synthesis setting of infer() / infer_stream() as a float, or as an fp32 [B] tensor (on the device it came from) when
    it is given per utterance as a 1-D sequence or tensor of B values.  A 0-d tensor counts as a float.  Another length or rank
    raises ValueError."""
    out = {}
    for name, v in settings.items():
        try:
            if np.ndim(v) == 0:
                out[name] = float(v)
                continue
            t = v.to(torch.float32) if isinstance(v, torch.Tensor) else torch.as_tensor(v, dtype=torch.float32)
        except (TypeError, ValueError, RuntimeError) as e:
            raise ValueError(f"{name}: expected a float or {B} per-utterance values") from e
        if t.dim() != 1 or t.shape[0] != B:
            raise ValueError(f"{name}: expected a float or {B} per-utterance values, got shape {list(t.shape)}")
        out[name] = t
    return out


def speaker_mixes(B: int, mix):
    """A speaker mix of infer() / infer_stream() as the (ids [B,K] int64, weights [B,K] fp32) CPU tensors Engine.infer_begin takes.
    `mix`: one dict {speaker_id: weight} for every utterance, or a sequence of B such dicts.  Dict order is summation order; a
    shorter mix is padded at the end to the batch's K with (its first id, 0.0).  Weights are used as given.  An empty dict, a
    non-integer or bool key, a non-finite weight or a sequence whose length is not B raises ValueError."""
    if isinstance(mix, dict):
        mixes = [mix] * B
    else:
        try:
            mixes = list(mix)
        except TypeError as e:
            raise ValueError("speaker_mix: expected a dict {speaker_id: weight} or a sequence of one per utterance") from e
        if len(mixes) != B:
            raise ValueError(f"speaker_mix: expected one dict or {B} dicts, got {len(mixes)}")
    rows = []
    for m in mixes:
        if not isinstance(m, dict) or not m:
            raise ValueError("speaker_mix: each mix must be a non-empty dict {speaker_id: weight}")
        ids = list(m.keys())
        if any(isinstance(i, (bool, np.bool_)) or not isinstance(i, (int, np.integer)) for i in ids):
            raise ValueError(f"speaker_mix: speaker ids must be integers, got {ids}")
        try:
            w = torch.tensor([float(v) for v in m.values()], dtype=torch.float32)
        except (TypeError, ValueError) as e:
            raise ValueError("speaker_mix: weights must be numbers") from e
        if not torch.isfinite(w).all():
            raise ValueError(f"speaker_mix: weights must be finite in fp32, got {list(m.values())}")
        rows.append(([int(i) for i in ids], w))
    K = max(len(ids) for ids, _ in rows)
    out_ids = torch.empty(B, K, dtype=torch.int64)
    out_w = torch.zeros(B, K, dtype=torch.float32)
    for b, (ids, w) in enumerate(rows):
        out_ids[b] = torch.tensor(ids + [ids[0]] * (K - len(ids)))
        out_w[b, :len(ids)] = w
    return out_ids, out_w


class _Lane:
    """Where a leased engine's work runs.  Without an own stream (concurrency=1): on the caller's current stream, as a single engine
    always ran.  With one: on the engine's own stream, which waits for the caller's work before each step; after the step the caller's
    stream waits for it, and every result tensor is recorded on the caller's stream so that the caching allocator does not hand its
    memory to the engine's next request while the caller still reads it."""

    def __init__(self, eng, own_stream: bool):
        self.stream = None
        if own_stream:
            if getattr(eng, "serve_stream", None) is None:
                eng.serve_stream = torch.cuda.Stream(eng.device)
            self.stream, self.caller = eng.serve_stream, torch.cuda.current_stream(eng.device)

    @contextlib.contextmanager
    def step(self):
        """Yields a list: append the step's result tensors to it."""
        results = []
        if self.stream is None:
            yield results
            return
        self.stream.wait_stream(self.caller)
        try:
            with torch.cuda.stream(self.stream):
                yield results
        finally:
            self.caller.wait_stream(self.stream)
        for t in results:
            if t is not None:
                t.record_stream(self.caller)


class LazyAttn:
    """Stand-in for the `attn` tensor infer() returns (reference models.py:1074): the dense [B,1,F,T] one-hot path is only
    written when somebody reads it (the reference's own callers never do: infer.py:302-318 uses `o` alone).  Any attribute
    access, indexing or torch function materialises it once through bv2_attn_path; `.materialize()` returns the tensor.
    Materialising leases the engine that served the call, and raises if that engine has served another request since."""

    def __init__(self, engine, shape, token, pool: EnginePool):
        self._engine, self._shape, self._token, self._pool, self._t = engine, tuple(shape), token, pool, None

    def materialize(self) -> torch.Tensor:
        if self._t is None:
            with self._pool.lease(self._engine) as eng:
                if getattr(eng, "_attn_token", None) is not self._token:
                    raise RuntimeError("attn of an earlier infer() call: materialise it before the engine that served it serves the next "
                                       "request (with concurrency=1: before the next call on the same module)")
                with _Lane(eng, self._pool.concurrency > 1).step() as results:
                    self._t = eng.attn_path()
                    results.append(self._t)
        return self._t

    @property
    def shape(self):
        return torch.Size(self._shape)

    def size(self, *a):
        return self.shape if not a else self.shape[a[0]]

    def dim(self):
        return len(self._shape)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return getattr(self.materialize(), name)

    def __getitem__(self, idx):
        return self.materialize()[idx]

    def __len__(self):
        return self._shape[0]

    def __repr__(self):
        return f"LazyAttn(shape={self._shape}, materialized={self._t is not None})"

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        conv = lambda a: a.materialize() if isinstance(a, LazyAttn) else a  # noqa: E731
        return func(*[conv(a) for a in args], **{k: conv(v) for k, v in (kwargs or {}).items()})


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's dotted state_dict key tree."""


class SynthesizerTrn(nn.Module):
    def __init__(self, n_vocab, spec_channels, segment_size, inter_channels, hidden_channels, filter_channels, n_heads,
                 n_layers, kernel_size, p_dropout, resblock, resblock_kernel_sizes, resblock_dilation_sizes, upsample_rates,
                 upsample_initial_channel, upsample_kernel_sizes, n_speakers=256, gin_channels=256, use_sdp=True,
                 n_flow_layer=4, n_layers_trans_flow=4, flow_share_parameter=False, use_transformer_flow=True,
                 precision: str = "fp16", init_seed: Optional[int] = 0, concurrency: int = 1, **kwargs):
        super().__init__()
        if int(concurrency) < 1:
            raise ValueError("concurrency must be >= 1")
        if n_speakers < 1:
            raise ValueError("n_speakers == 0 (ReferenceEncoder path, models.py:752-808) is a training-only configuration")
        if flow_share_parameter:
            raise ValueError("flow_share_parameter=True references attentions.FFT, which does not exist in the reference")
        if not kwargs.get("use_spk_conditioned_encoder", True):
            raise ValueError("use_spk_conditioned_encoder=False is not supported")
        self.n_vocab, self.spec_channels, self.segment_size = n_vocab, spec_channels, segment_size
        self.inter_channels, self.hidden_channels, self.filter_channels = inter_channels, hidden_channels, filter_channels
        self.n_heads, self.n_layers, self.kernel_size, self.p_dropout = n_heads, n_layers, kernel_size, p_dropout
        self.n_speakers, self.gin_channels, self.use_sdp = n_speakers, gin_channels, use_sdp
        self.precision = precision
        self.concurrency = int(concurrency)
        self._tls = threading.local()
        model = dict(inter_channels=inter_channels, hidden_channels=hidden_channels, filter_channels=filter_channels,
                     n_heads=n_heads, n_layers=n_layers, kernel_size=kernel_size, resblock=resblock,
                     resblock_kernel_sizes=list(resblock_kernel_sizes),
                     resblock_dilation_sizes=[list(d) for d in resblock_dilation_sizes], upsample_rates=list(upsample_rates),
                     upsample_initial_channel=upsample_initial_channel, upsample_kernel_sizes=list(upsample_kernel_sizes),
                     gin_channels=gin_channels, use_sdp=use_sdp, n_flow_layer=n_flow_layer,
                     n_layers_trans_flow=n_layers_trans_flow, use_transformer_flow=use_transformer_flow)
        self.cfg = ModelConfig.from_hps_model(model, n_vocab=n_vocab, n_speakers=n_speakers)
        init = synth.synthetic_state_dict(self.cfg, init_seed) if init_seed is not None else None
        for p in param_specs(self.cfg):
            parts = p.key.split(".")
            node = self
            for name in parts[:-1]:
                if name not in node._modules:
                    node.add_module(name, _Node())
                node = node._modules[name]
            t = init[p.key] if init is not None else torch.zeros(p.shape)
            node.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))
        self._engines = {}
        self._pools = {}
        self._weights_version = 0
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._invalidate())

    @property
    def last_y_lengths(self):
        """y_lengths of the calling thread's latest infer() / infer_stream() (each thread reads its own request's)."""
        return self._tls.y_lengths

    @last_y_lengths.setter
    def last_y_lengths(self, v):
        self._tls.y_lengths = v

    # -- weight changes invalidate the packed device copy ------------------------------------------------
    def _invalidate(self):
        self._weights_version += 1
        self._engines.clear()
        self._pools.clear()

    def _apply(self, fn, *a, **kw):
        r = super()._apply(fn, *a, **kw)
        self._invalidate()
        return r

    def remove_weight_norm(self):
        """No-op: weight-norm is folded once when the engine packs its weights (the reference re-evaluates it on
        every forward because nobody calls this, SURVEY.md §2.2)."""

    def _engine(self, device: torch.device) -> Engine:
        key = (str(device), self._weights_version)
        eng = self._engines.get(key)
        if eng is None:
            sd = {k: v for k, v in self.state_dict().items()}
            eng = Engine(self.cfg, sd, device=device, precision=self.precision)
            self._engines = {key: eng}
        return eng

    def _pool(self, device: torch.device) -> EnginePool:
        """The engine pool of `device`: the primary engine of _engine() plus up to concurrency - 1 siblings, created when needed."""
        with _ENGINE_LOCK:
            eng = self._engine(device)
            key = (str(device), self._weights_version)
            pool = self._pools.get(key)
            if pool is None or pool.primary is not eng:
                pool = EnginePool(eng, self.concurrency, lambda primary: primary.sibling())
                self._pools = {key: pool}
            return pool

    def _cuda_device(self, what: str) -> torch.device:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise Bv2Error(f"SynthesizerTrn.{what}: module is on CPU; bert_vits2_b200 has no CPU path — call .to('cuda')")
        return dev

    def _begin(self, eng, dev, results, args, noise_w, settings, w_ceil_override, mix=None):
        """eng.infer_begin with `settings` (item_settings) and `mix` (speaker_mixes, or None) -> (y_lengths, F, the noise_scale
        infer_finish* takes).  Per-utterance settings and the mix go to the device and to `results`, and a per-utterance noise_scale
        becomes item_noise_scale (finish then takes 1.0)."""
        s = dict(settings)
        if mix is None and all(not isinstance(v, torch.Tensor) for v in s.values()):  # the scalar call
            y_lengths, F = eng.infer_begin(*args, noise_w, s["noise_scale_w"], s["length_scale"], s["sdp_ratio"], w_ceil_override)
            return y_lengths, F, s["noise_scale"]
        for k, v in s.items():
            if isinstance(v, torch.Tensor):
                s[k] = v.to(device=dev, dtype=torch.float32).contiguous()
                results.append(s[k])
        if mix is not None:
            mix = tuple(t.to(device=dev).contiguous() for t in mix)
            results += mix
        ns = s["noise_scale"]
        y_lengths, F = eng.infer_begin(*args, noise_w, s["noise_scale_w"], s["length_scale"], s["sdp_ratio"], w_ceil_override,
                                       item_noise_scale=ns if isinstance(ns, torch.Tensor) else None, speaker_mix=mix)
        return y_lengths, F, 1.0 if isinstance(ns, torch.Tensor) else ns

    @staticmethod
    def _mix(B, sid, speaker_mix):
        """speaker_mix as speaker_mixes gives it, or None; ValueError when it comes with a sid"""
        if speaker_mix is None:
            return None
        if sid is not None:
            raise ValueError("give either sid or speaker_mix, not both (pass sid=None with a speaker mix)")
        return speaker_mixes(B, speaker_mix)

    # ----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def infer(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, noise_scale=0.667, length_scale=1,
              noise_scale_w=0.8, max_len=None, sdp_ratio=0, y=None, *, noise_w=None, noise_z=None, w_ceil_override=None, pcm16=False,
              ragged=False, speaker_mix=None):
        """reference models.py:1026-1074.  Keyword-only extras (not in the reference): explicit noise tensors
        `noise_w` [B,2,T] / `noise_z` [B,inter,>=F] replacing the two in-model RNG draws (models.py:249, 1071), and
        `w_ceil_override` [B,T] to teacher-force durations in parity harnesses, `pcm16=True` to get `o` as int16 converted like
        the reference's callers do (gradio convert_to_16_bit_wav, webui.py:86).  `ragged=True` (precision fp16 / fp16g only,
        ValueError otherwise): the Generator runs each utterance at its own length instead of the padded one, so each waveform is
        what the utterance gives alone (its last frames do not see the padding) and 0 past its length; a different result from
        the reference's padded batch, not a faster route to it.  `attn` comes back as a LazyAttn (see above).
        noise_scale, length_scale, noise_scale_w and sdp_ratio each take a float, as in the reference, which only takes scalars, or a
        1-D sequence or tensor of B values, one per utterance (ValueError for another length or rank): utterance b then comes out
        bit-identical to a call of the same batch with its own values as floats, at the launches of one call.
        `speaker_mix` (with sid=None; ValueError with both): each utterance is conditioned on a weighted sum of speaker embeddings
        instead of one speaker, given as one dict {speaker_id: weight} for every utterance or a sequence of B dicts (speaker_mixes);
        utterance b is bit-identical to a plain call on a module whose emb_g holds b's mix as an extra row (bv2_infer_begin_mix).
        The call leases one engine of the module's pool from begin to finish (concurrency=N: up to N calls run at once)."""
        if ragged and self.precision not in ("fp16", "fp16g"):
            raise ValueError(f"ragged=True needs the FP16 Generator (precision fp16 or fp16g), not {self.precision}")
        settings = item_settings(x.shape[0], noise_scale=noise_scale, length_scale=length_scale, noise_scale_w=noise_scale_w,
                                 sdp_ratio=sdp_ratio)
        mix = self._mix(x.shape[0], sid, speaker_mix)
        dev = self._cuda_device("infer")
        if x.dim() != 2 or bert.dim() != 3 or bert.shape[-1] != x.shape[1]:
            raise ValueError("expected x [B,T] and bert features [B,1024,T]")
        pool = self._pool(dev)
        B, T = x.shape
        with pool.lease() as eng:
            with _Lane(eng, self.concurrency > 1).step() as results:
                if noise_w is None:  # same draw order/shape as the reference: SDP first (models.py:249)
                    noise_w = torch.randn(B, 2, T, device=dev, dtype=torch.float32)
                y_lengths, F, noise_scale = self._begin(eng, dev, results, (x, x_lengths, sid, tone, language, bert, ja_bert, en_bert),
                                                        noise_w, settings, w_ceil_override, mix)
                if noise_z is None:  # torch.randn_like(m_p), m_p: [B, inter, F] (models.py:1071)
                    noise_z = torch.randn(B, self.inter_channels, F, device=dev, dtype=torch.float32)
                extra = {"ragged": True} if ragged else {}
                o, _, y_mask, aux = eng.infer_finish(B, T, F, noise_z, noise_scale, max_len, want_attn=False, pcm16=pcm16, **extra)
                results += [o, y_mask, *aux]
            eng._attn_token = token = object()
        self.last_y_lengths = y_lengths
        return o, LazyAttn(eng, (B, 1, F, T), token, pool), y_mask, aux

    @torch.no_grad()
    def infer_stream(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, noise_scale=0.667, length_scale=1,
                     noise_scale_w=0.8, max_len=None, sdp_ratio=0, y=None, *, noise_w=None, noise_z=None, w_ceil_override=None,
                     first_chunk_frames=32, max_chunk_frames=None, ragged=False, speaker_mix=None):
        """Streaming infer(): a generator of waveform chunks o[:, :, a:b] (device tensors, views of one [B,1,Fg*hop] buffer) whose
        concatenation is bit-identical to infer(...)[0] with the same noise.  Encoder, durations and flow run whole first (the flow's
        attention spans the utterance); the Generator then runs as a wavefront, so the first chunk costs about first_chunk_frames
        + 14 frames of Generator work instead of all of it.  Chunks are first_chunk_frames frames, then double.  Each chunk is final
        when it is yielded (the host waits on an event recorded after its work) and no later chunk writes it.  Noise is drawn exactly
        as infer() draws it.  `last_y_lengths` is set before the first chunk.  There is no pcm16 option: the PCM conversion normalises by the peak of the whole utterance.
        The generator leases one engine of the module's pool from its first step until it is exhausted, closed or collected.
        `max_chunk_frames`: chunks double only up to this many frames, and the stream's Generator memory is then set by it, not by
        the utterance's length (bounded stream: Engine.stream_bytes).  It needs the FP16 Generator (precision fp16 or fp16g) when it
        is below the utterance's frame count; ValueError otherwise, and for max_chunk_frames < first_chunk_frames.  None: chunks
        double without limit and every Generator activation stays resident until the stream ends.
        `ragged=True` (precision fp16 / fp16g only, ValueError otherwise): the Generator runs each utterance at its own length, as
        infer(..., ragged=True) does, with the same chunks.  Utterance b's samples are final and complete once a chunk ends at or past
        last_y_lengths[b] * hop (max_len applied), and the concatenation is bit-identical to infer(..., ragged=True)[0]: 0 past its end.
        The four synthesis settings take a float (the reference only takes scalars) or B per-utterance values, and `speaker_mix` a
        speaker mix instead of sid, as in infer()."""
        if ragged and self.precision not in ("fp16", "fp16g"):
            raise ValueError(f"ragged=True needs the FP16 Generator (precision fp16 or fp16g), not {self.precision}")
        settings = item_settings(x.shape[0], noise_scale=noise_scale, length_scale=length_scale, noise_scale_w=noise_scale_w,
                                 sdp_ratio=sdp_ratio)
        mix = self._mix(x.shape[0], sid, speaker_mix)
        dev = self._cuda_device("infer_stream")
        if x.dim() != 2 or bert.dim() != 3 or bert.shape[-1] != x.shape[1]:
            raise ValueError("expected x [B,T] and bert features [B,1024,T]")
        if first_chunk_frames < 1:
            raise ValueError("first_chunk_frames must be >= 1")
        if max_chunk_frames is not None and max_chunk_frames < first_chunk_frames:
            raise ValueError("max_chunk_frames must be >= first_chunk_frames")
        pool = self._pool(dev)
        B, T = x.shape
        eng = pool.acquire()
        try:
            lane = _Lane(eng, self.concurrency > 1)
            with lane.step() as results:
                if noise_w is None:
                    noise_w = torch.randn(B, 2, T, device=dev, dtype=torch.float32)
                y_lengths, F, noise_scale = self._begin(eng, dev, results, (x, x_lengths, sid, tone, language, bert, ja_bert, en_bert),
                                                        noise_w, settings, w_ceil_override, mix)
                if noise_z is None:
                    noise_z = torch.randn(B, self.inter_channels, F, device=dev, dtype=torch.float32)
                extra = {} if max_chunk_frames is None else {"max_chunk_frames": max_chunk_frames}
                if ragged:
                    extra["ragged"] = True
                o, _, _, _ = eng.infer_finish_stream(B, T, F, noise_z, noise_scale, max_len, want_attn=False, **extra)
                results.append(o)
            eng._attn_token = object()  # a LazyAttn of an earlier infer() must not materialise this utterance's path
            self.last_y_lengths = y_lengths
            hop = self.cfg.hop
            Fg = o.shape[-1] // hop
            done, step = 0, int(first_chunk_frames)
            while done < Fg:
                target = min(done + step, Fg)
                with lane.step():
                    eng.stream_advance(target)
                    ev = torch.cuda.Event()
                    ev.record(torch.cuda.current_stream(dev))
                    ev.synchronize()
                yield o[:, :, done * hop:target * hop]
                done, step = target, 2 * step if max_chunk_frames is None else min(2 * step, int(max_chunk_frames))
        finally:
            pool.release(eng)

    def forward(self, *a, **kw):
        raise NotImplementedError("training forward (reference models.py:937-1024) is out of scope; use .infer()")
