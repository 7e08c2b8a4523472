"""Thin ctypes wrapper over libbv2 (include/bv2.h): tensor plumbing only, every FLOP runs in the CUDA library."""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from .spec import ModelConfig, is_infer_key


class Bv2Error(RuntimeError):
    pass


#: engine precision -> bv2_config.generator_precision (include/bv2.h)
PRECISIONS = {"fp32": 0, "tf32": 1, "fp16g": 2, "fp16": 3}  # fp16g: FP16 Generator + TF32 flow (A/B only)


def _cfg_struct(cfg: ModelConfig, precision: int) -> _lib.Bv2Config:
    c = _lib.Bv2Config()
    for n in ("n_vocab", "num_tones", "num_languages", "bert_dim", "inter_channels", "hidden_channels", "filter_channels",
              "n_heads", "n_layers", "kernel_size", "window_size", "gin_channels", "n_speakers", "n_flow_layer",
              "n_layers_trans_flow", "flow_kernel_size", "wn_layers", "upsample_initial_channel", "sdp_filter", "sdp_kernel",
              "sdp_n_flows", "sdp_dds_layers", "sdp_num_bins", "dp_filter", "dp_kernel", "cond_layer_idx"):
        setattr(c, n, int(getattr(cfg, n)))
    c.use_transformer_flow = int(bool(cfg.use_transformer_flow))
    c.sdp_tail_bound = float(cfg.sdp_tail_bound)
    c.n_ups = len(cfg.upsample_rates)
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        c.upsample_rates[i] = u
        c.upsample_kernel_sizes[i] = k
    c.n_resblock_kernels = len(cfg.resblock_kernel_sizes)
    c.n_dilations = len(cfg.resblock_dilation_sizes[0])
    for j, (k, ds) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
        c.resblock_kernel_sizes[j] = k
        for d, v in enumerate(ds):
            c.resblock_dilation_sizes[j][d] = v
    c.generator_precision = precision
    c.n_flows = int(cfg.n_flows)
    if cfg.resblock != "1":
        raise ValueError("only resblock='1' (ResBlock1) is supported, as configs/config.json sets")
    return c


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _cap(max_chunk_frames: Optional[int]) -> int:
    """max_chunk_frames as the C ABI takes it: 0 = unbounded"""
    return 0 if max_chunk_frames is None else max(0, int(max_chunk_frames))


class Engine:
    """An engine on one CUDA device; it serves one request at a time (sibling() gives another over the same weights).  precision: 'fp32' (SIMT FMA everywhere), 'tf32' (wgmma implicit-GEMM convs with TF32
    operands) or 'fp16' (wgmma with FP16 operands -- same 11-bit significand as TF32, twice the tensor rate, half the
    operand traffic; fp32 accumulate and fp32 activations in HBM).  Everything that feeds ceil(durations) is FP32 FMA in all three."""

    def __init__(self, cfg: ModelConfig, state_dict: Optional[Dict[str, torch.Tensor]], device="cuda:0", precision: str = "fp16",
                 packed_path: Optional[str] = None):
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise Bv2Error("bert_vits2_b200 has no CPU path: a CUDA (sm_90) device is required")
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        self.precision = PRECISIONS[precision]
        self._h = C.c_void_p()
        cs = _cfg_struct(cfg, self.precision)
        rc = self.lib.bv2_create(C.byref(self._h), C.byref(cs), idx)
        if rc != 0:
            raise Bv2Error(f"bv2_create failed ({rc}): needs an sm_90 CUDA device, there is no fallback")
        if packed_path is not None:  # pre-folded, pre-packed weight file written by save_packed(): load = one cudaMemcpy
            self._check(self.lib.bv2_load_packed(self._h, os.fsencode(packed_path)))
            return
        for k, v in state_dict.items():
            if not is_infer_key(k):
                continue
            t = v.detach().to("cpu")
            dt = 1 if t.dtype == torch.float16 else 0
            if dt == 0:
                t = t.to(torch.float32)
            t = t.contiguous()
            shape = (C.c_int64 * max(1, t.dim()))(*t.shape)
            self._check(self.lib.bv2_set_weight(self._h, k.encode(), C.c_void_p(t.data_ptr()), shape, t.dim(), dt))
        self._check(self.lib.bv2_finalize(self._h))

    def sibling(self) -> "Engine":
        """A second engine over this engine's device weights (bv2_create_sibling: nothing is copied).  It has its own workspace,
        per-call state and mutex, so it can serve a request on another CUDA stream while this one serves another."""
        sib = Engine.__new__(Engine)
        sib.lib, sib.cfg, sib.device, sib.precision = self.lib, self.cfg, self.device, self.precision
        sib._h = C.c_void_p()
        self._check(self.lib.bv2_create_sibling(C.byref(sib._h), self._h))
        return sib

    @property
    def workspace_bytes(self) -> int:
        """Bytes of workspace (both arenas) this engine holds."""
        return int(self.lib.bv2_workspace_bytes(self._h))

    def save_packed(self, path: str):
        """Dump the finalized weight arena (folded + packed for this config and precision); reload with Engine(cfg, None, packed_path=path)."""
        self._check(self.lib.bv2_save_packed(self._h, os.fsencode(path)))

    def _check(self, rc):
        if rc != 0:
            msg = self.lib.bv2_last_error(self._h).decode(errors="replace")
            if rc == -1:
                if "index out of range" in msg:
                    raise IndexError(msg)  # the reference raises IndexError from nn.Embedding
                raise ValueError(msg)
            raise Bv2Error(f"libbv2 error {rc}: {msg}")

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.bv2_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _i64(self, t):
        return t.to(device=self.device, dtype=torch.int64).contiguous()

    def _f32(self, t):
        return t.to(device=self.device, dtype=torch.float32).contiguous()

    @property
    def launch_count(self) -> int:
        return int(self.lib.bv2_launch_count(self._h))

    @property
    def workspace_grows(self) -> int:
        """(Re)allocations of the workspace arenas since creation (0 on the hot path once `reserve` covered the shapes)."""
        return int(self.lib.bv2_workspace_grows(self._h))

    def reserve(self, B: int, T: int, F_cap: int):
        """Size the workspace up front for batches up to (B, T tokens, F_cap frames): no allocation / device sync afterwards."""
        self._check(self.lib.bv2_reserve(self._h, int(B), int(T), int(F_cap)))

    def reserve_stream(self, B: int, T: int, F_cap: int, max_chunk_frames: Optional[int]):
        """reserve() plus room for one stream with chunks of at most max_chunk_frames (None: an unbounded stream) over up to F_cap
        frames: afterwards no call and no such stream within those bounds grows the workspace."""
        self._check(self.lib.bv2_reserve_stream(self._h, int(B), int(T), int(F_cap), _cap(max_chunk_frames)))

    def stream_bytes(self, B: int, Fg: int, max_chunk_frames: Optional[int]) -> int:
        """Workspace bytes of the Generator tensors of a stream over Fg frames with chunks of at most max_chunk_frames (computed, not
        measured): for a cap below Fg the bounded storage, which does not depend on Fg; else what an unbounded stream allocates."""
        n = int(self.lib.bv2_stream_bytes(self._h, int(B), int(Fg), _cap(max_chunk_frames)))
        if n < 0:
            raise ValueError(f"stream_bytes(B={B}, Fg={Fg}, max_chunk_frames={max_chunk_frames}): rejected ({n}); a cap below Fg needs "
                             "the FP16 Generator")
        return n

    def set_profiling(self, on: bool = True):
        self._check(self.lib.bv2_set_profiling(self._h, int(on)))

    def stage_ms(self, stage: str) -> float:
        return float(self.lib.bv2_stage_ms(self._h, stage.encode()))

    # ---- whole path ---------------------------------------------------------------------------------
    def infer_begin(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert, noise_w, noise_scale_w, length_scale,
                    sdp_ratio, w_ceil_override=None, *, item_noise_scale=None, speaker_mix=None):
        """noise_scale_w, length_scale and sdp_ratio: a float, or a [B] tensor of per-utterance values.  `item_noise_scale` [B]: each
        utterance's prior-noise scale, multiplied (rounded once) into the noise_scale every infer_finish* takes, so pass 1.0 there.
        With any tensor this is bv2_infer_begin_items (floats broadcast to [B], item_noise_scale 1.0 when None), and utterance b comes
        out bit-identical to a call with its own values as floats; with floats alone it is bv2_infer_begin.
        `speaker_mix` (ids [B,K] int64, weights [B,K] fp32), with sid None: utterance b is conditioned on sum_k weights[b,k] *
        emb_g[ids[b,k]] in k order instead of one speaker's row (bv2_infer_begin_mix, the settings broadcast as for
        bv2_infer_begin_items)."""
        B, T = x.shape
        if (sid is None) == (speaker_mix is None):
            raise ValueError("infer_begin takes either sid or speaker_mix")
        self._keep = [self._i64(x), self._i64(x_lengths), None if sid is None else self._i64(sid), self._i64(tone), self._i64(language),
                      self._f32(bert), self._f32(ja_bert), self._f32(en_bert), self._f32(noise_w),
                      None if w_ceil_override is None else self._f32(w_ceil_override)]
        k = self._keep
        ylen = (C.c_int64 * B)()
        fmax = C.c_int32(0)
        head = (self._h, B, T, *(_ptr(t) for t in k[:9]))
        tail = (_ptr(k[9]), self._stream(), ylen, C.byref(fmax))
        settings = (noise_scale_w, length_scale, sdp_ratio, item_noise_scale)
        if speaker_mix is None and all(not isinstance(v, torch.Tensor) for v in settings):
            self._check(self.lib.bv2_infer_begin(*head, float(noise_scale_w), float(length_scale), float(sdp_ratio), *tail))
            return np.frombuffer(ylen, dtype=np.int64).copy(), int(fmax.value)
        arrays = [self._items(v, B) for v in settings[:3]] + [self._items(1.0 if item_noise_scale is None else item_noise_scale, B)]
        self._keep += arrays
        if speaker_mix is None:
            self._check(self.lib.bv2_infer_begin_items(*head, *(_ptr(a) for a in arrays), *tail))
        else:
            ids, w = self._i64(speaker_mix[0]), self._f32(speaker_mix[1])
            if ids.dim() != 2 or ids.shape[0] != B or ids.shape != w.shape:
                raise ValueError(f"speaker_mix: expected ids and weights of one shape [{B}, K], got {list(ids.shape)} and {list(w.shape)}")
            self._keep += [ids, w]
            self._check(self.lib.bv2_infer_begin_mix(self._h, B, T, _ptr(k[0]), _ptr(k[1]), ids.shape[1], _ptr(ids), _ptr(w),
                                                     *(_ptr(t) for t in k[3:9]), *(_ptr(a) for a in arrays), *tail))
        return np.frombuffer(ylen, dtype=np.int64).copy(), int(fmax.value)

    def _items(self, v, B):
        """a setting as the fp32 [B] device array bv2_infer_begin_items takes: a float broadcast, or a tensor of B values"""
        if not isinstance(v, torch.Tensor):
            return torch.full((B,), float(v), device=self.device, dtype=torch.float32)
        if v.shape != (B,):
            raise ValueError(f"a per-utterance setting must have shape [{B}], got {list(v.shape)}")
        return self._f32(v)

    def infer_finish(self, B, T, F, noise_z, noise_scale, max_len=None, want_attn=True, out_ptr: Optional[int] = None, pcm16: bool = False,
                     ragged: bool = False):
        """`out_ptr`: raw device address that receives the waveform batch [B,1,Fg*hop] instead of a fresh tensor -- e.g. a
        slice of a peer-mapped slab (sharding.PeerWaveSlab) so the Generator epilogue stores straight into the root GPU's
        memory over NVLink; the returned `o` is then None.  `want_attn=False` skips the O(F*T) attn write (use `attn_path()`
        later if it is needed after all).  `pcm16=True`: `o` is int16, peak-normalised exactly as the reference's callers
        convert every infer() result (gradio convert_to_16_bit_wav, webui.py:86).  `ragged=True` (FP16 Generator only, ValueError
        otherwise): the Generator runs each utterance at its own length, so its samples are those of a run of it alone and 0 past
        its length (bv2_infer_finish_ragged), instead of the padded batch's."""
        I, hop = self.cfg.inter_channels, self.cfg.hop
        noise_z = self._f32(noise_z)
        assert noise_z.shape[0] == B and noise_z.shape[1] == I and noise_z.shape[2] >= F
        Fg = F if (max_len is None or max_len >= F) else int(max_len)
        dev = self.device
        o = torch.empty(B, 1, Fg * hop, device=dev, dtype=torch.int16 if pcm16 else torch.float32) if out_ptr is None else None
        attn = torch.empty(B, 1, F, T, device=dev, dtype=torch.float32) if want_attn else None
        y_mask = torch.empty(B, 1, F, device=dev, dtype=torch.float32)
        z, z_p, m_p, logs_p = (torch.empty(B, I, F, device=dev, dtype=torch.float32) for _ in range(4))
        self._last = (B, T, F)
        dst = _ptr(o) if out_ptr is None else C.c_void_p(int(out_ptr))
        tail = (_ptr(attn), _ptr(y_mask), _ptr(z), _ptr(z_p), _ptr(m_p), _ptr(logs_p), self._stream())
        head = (self._h, _ptr(noise_z), noise_z.shape[2], float(noise_scale), -1 if max_len is None else int(max_len))
        if ragged:
            self._check(self.lib.bv2_infer_finish_ragged(*head, None if pcm16 else dst, dst if pcm16 else None, *tail))
        else:
            fn = self.lib.bv2_infer_finish_pcm16 if pcm16 else self.lib.bv2_infer_finish
            self._check(fn(*head, dst, *tail))
        return o, attn, y_mask, (z, z_p, m_p, logs_p)

    def infer_finish_stream(self, B, T, F, noise_z, noise_scale, max_len=None, want_attn=True, max_chunk_frames: Optional[int] = None,
                            ragged: bool = False):
        """infer_finish up to and including the flow, then open a Generator stream over the returned `o` [B,1,Fg*hop]; its samples become
        final as stream_advance() is called.  Returns (o, attn, y_mask, (z, z_p, m_p, logs_p)) like infer_finish.  Every precision;
        no pcm16 (its peak normalisation needs the whole utterance).  `max_chunk_frames`: a cap on how far one stream_advance may
        move the frontier; below Fg it bounds the stream's Generator memory (stream_bytes) and needs the FP16 Generator (ValueError
        otherwise).  `ragged=True` (FP16 Generator only, ValueError otherwise): the Generator runs each utterance at its own length
        L_b = min(y_lengths[b], Fg), so once the frontier reaches L_b its samples are those of infer_finish(..., ragged=True) and 0
        past L_b*hop (bv2_infer_finish_stream_ragged); same chunks, launches and workspace as the padded stream."""
        I, hop = self.cfg.inter_channels, self.cfg.hop
        noise_z = self._f32(noise_z)
        assert noise_z.shape[0] == B and noise_z.shape[1] == I and noise_z.shape[2] >= F
        Fg = F if (max_len is None or max_len >= F) else int(max_len)
        dev = self.device
        o = torch.empty(B, 1, Fg * hop, device=dev, dtype=torch.float32)
        attn = torch.empty(B, 1, F, T, device=dev, dtype=torch.float32) if want_attn else None
        y_mask = torch.empty(B, 1, F, device=dev, dtype=torch.float32)
        z, z_p, m_p, logs_p = (torch.empty(B, I, F, device=dev, dtype=torch.float32) for _ in range(4))
        self._last = (B, T, F)
        fn = self.lib.bv2_infer_finish_stream_ragged if ragged else self.lib.bv2_infer_finish_stream_bounded
        self._check(fn(self._h, _ptr(noise_z), noise_z.shape[2], float(noise_scale), -1 if max_len is None else int(max_len),
                       _cap(max_chunk_frames), _ptr(o), _ptr(attn), _ptr(y_mask), _ptr(z), _ptr(z_p), _ptr(m_p), _ptr(logs_p), self._stream()))
        self._stream_o = o  # the stream writes into o until it closes
        return o, attn, y_mask, (z, z_p, m_p, logs_p)

    def stream_advance(self, frames: int) -> int:
        """Enqueue the Generator work that makes o[..., :min(frames, Fg)*hop] final on the current stream; returns that sample count.
        Raises Bv2Error if no stream is open or `frames` does not exceed the frames already final, and ValueError if the chunk exceeds a
        bounded stream's max_chunk_frames (the stream stays open and unchanged)."""
        n = C.c_int64(0)
        self._check(self.lib.bv2_stream_advance(self._h, int(frames), self._stream(), C.byref(n)))
        return int(n.value)

    def attn_path(self) -> torch.Tensor:
        """attn [B,1,F,T] of the last infer_begin/infer_finish, materialised on demand (valid until the next infer_begin)."""
        B, T, F = self._last
        attn = torch.empty(B, 1, F, T, device=self.device, dtype=torch.float32)
        self._check(self.lib.bv2_attn_path(self._h, _ptr(attn), self._stream()))
        return attn

    def wave_to_pcm16(self, wave: torch.Tensor, n_valid: Optional[torch.Tensor] = None) -> torch.Tensor:
        """wave [B,1,L] or [B,L] fp32 -> int16 of the same shape, as gradio's convert_to_16_bit_wav does per utterance."""
        w = self._f32(wave)
        B, L = w.shape[0], w.shape[-1]
        nv = None if n_valid is None else self._i64(n_valid)
        out = torch.empty(w.shape, device=self.device, dtype=torch.int16)
        self._check(self.lib.bv2_wave_to_pcm16(self._h, B, L, _ptr(w), _ptr(nv), _ptr(out), self._stream()))
        return out

    # ---- per-stage entry points (parity tests, microbenchmarks) -----------------------------------------
    def text_encoder(self, x, x_lengths, sid, tone, language, bert, ja_bert, en_bert):
        B, T = x.shape
        H, I = self.cfg.hidden_channels, self.cfg.inter_channels
        k = [self._i64(x), self._i64(x_lengths), self._i64(sid), self._i64(tone), self._i64(language), self._f32(bert),
             self._f32(ja_bert), self._f32(en_bert)]
        xo = torch.empty(B, H, T, device=self.device)
        m = torch.empty(B, I, T, device=self.device)
        logs = torch.empty(B, I, T, device=self.device)
        self._check(self.lib.bv2_text_encoder(self._h, B, T, *[_ptr(t) for t in k], _ptr(xo), _ptr(m), _ptr(logs), self._stream()))
        return xo, m, logs

    def duration(self, x, x_lengths, sid, noise_w, noise_scale_w):
        B, H, T = x.shape
        k = [self._f32(x), self._i64(x_lengths), self._i64(sid), self._f32(noise_w)]
        a = torch.empty(B, 1, T, device=self.device)
        b = torch.empty(B, 1, T, device=self.device)
        self._check(self.lib.bv2_duration(self._h, B, T, _ptr(k[0]), _ptr(k[1]), _ptr(k[2]), _ptr(k[3]), float(noise_scale_w),
                                          _ptr(a), _ptr(b), self._stream()))
        return a, b

    def flow_reverse(self, z_p, y_lengths, sid):
        B, I, F = z_p.shape
        k = [self._f32(z_p), self._i64(y_lengths), self._i64(sid)]
        z = torch.empty(B, I, F, device=self.device)
        self._check(self.lib.bv2_flow_reverse(self._h, B, F, _ptr(k[0]), _ptr(k[1]), _ptr(k[2]), _ptr(z), self._stream()))
        return z

    def generator(self, z, g, out: Optional[torch.Tensor] = None, lengths=None):
        """z [B,inter,F], g [B,gin(,1)] -> [B,1,F*hop].  `lengths` [B] (frames; FP16 Generator only, ValueError otherwise): a ragged
        batch, item b run at its own length clamped to [1, F], with zeros past it (bv2_generator_ragged)."""
        B, I, F = z.shape
        z = self._f32(z)
        g = self._f32(g.reshape(B, -1))
        if out is None:
            out = torch.empty(B, 1, F * self.cfg.hop, device=self.device)
        if lengths is None:
            self._check(self.lib.bv2_generator(self._h, B, F, _ptr(z), _ptr(g), _ptr(out), self._stream()))
        else:
            lens = self._i64(torch.as_tensor(lengths)).reshape(B)
            self._check(self.lib.bv2_generator_ragged(self._h, B, F, _ptr(z), _ptr(g), _ptr(lens), _ptr(out), self._stream()))
        return out

    def debug_read(self, name: str, shape) -> torch.Tensor:
        n = int(np.prod(shape))
        buf = np.empty(n, dtype=np.float32)
        got = self.lib.bv2_debug_read(self._h, name.encode(), C.c_void_p(buf.ctypes.data), n)
        if got < 0:
            self._check(int(got))
        return torch.from_numpy(buf[:got].reshape(shape))
