"""Multi-GPU plumbing for the infer path: utterances are independent (no cross-batch op anywhere in reference
models.py:1026-1074), so the path shards embarrassingly -- one process per GPU, full weight replica per rank, no
data-path collective.  The single exchange step is the collection of the finished waveforms on one rank (SURVEY.md
§8e); the reference has no equivalent (inference is single-device, webui.py:31, 397-399).  Two implementations:
`PeerWaveSlab` (the Generator's conv_post+tanh epilogue stores into the root GPU's memory over
NVLink/NVSwitch through a CUDA-IPC mapped slab, NCCL carries only a 4-byte completion flag) and `gather_waveforms`
(backend-agnostic padded gather; gloo in the CPU tests).

`deal_buckets` reuses the length-bucketing idea of the reference's training sampler (data_utils.py:305-335):
sort by token count, cut into per-rank batches of similar length so padding (and the padded-tail work the
reference semantics require, SURVEY.md §7 H4) is minimal, and deal batches to ranks so that every rank gets the
same number of batches and a balanced token count.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def deal_buckets(lengths: Sequence[int], world_size: int, batch_size: int) -> List[List[List[int]]]:
    """Returns plan[rank] = list of batches, each a list of utterance indices (sorted by length inside a batch).
    Every utterance appears exactly once; ranks differ by at most one batch."""
    order = sorted(range(len(lengths)), key=lambda i: (lengths[i], i))
    batches = [order[i:i + batch_size] for i in range(0, len(order), batch_size)]
    # longest batches first, greedy onto the least-loaded rank (load = padded tokens), ties -> lowest rank
    batches.sort(key=lambda b: -max(lengths[i] for i in b) * len(b))
    plan: List[List[List[int]]] = [[] for _ in range(world_size)]
    load = [0] * world_size
    cap = -(-len(batches) // world_size)
    for b in batches:
        cands = [r for r in range(world_size) if len(plan[r]) < cap]
        r = min(cands, key=lambda q: (load[q], q))
        plan[r].append(b)
        load[r] += max(lengths[i] for i in b) * len(b)
    return plan


def gather_waveforms(wave: torch.Tensor, n_samples: torch.Tensor, dst: int = 0) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """Gather per-rank padded waveform batches [B_r, 1, L_r] (+ valid sample counts [B_r]) to rank `dst`.
    Works on any backend (nccl over NVLink on the GPU box, gloo in CPU tests).  Shapes may differ per rank, so the
    sizes are exchanged first and the payload is padded to the maximum."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return [wave], [n_samples]
    rank = dist.get_rank()
    shape = torch.tensor([wave.shape[0], wave.shape[-1]], dtype=torch.int64, device=wave.device)
    shapes = [torch.zeros_like(shape) for _ in range(world)]
    dist.all_gather(shapes, shape)
    Bm = int(max(s[0] for s in shapes)); Lm = int(max(s[1] for s in shapes))
    pad = torch.zeros(Bm, 1, Lm, dtype=wave.dtype, device=wave.device)
    pad[: wave.shape[0], :, : wave.shape[-1]] = wave
    ns = torch.zeros(Bm, dtype=torch.int64, device=wave.device)
    ns[: n_samples.shape[0]] = n_samples.to(torch.int64)
    outs = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
    nss = [torch.empty_like(ns) for _ in range(world)] if rank == dst else None
    dist.gather(pad, outs, dst=dst)
    dist.gather(ns, nss, dst=dst)
    if rank != dst:
        return [], []
    waves = [o[: int(s[0]), :, : int(s[1])] for o, s in zip(outs, shapes)]
    counts = [n[: int(s[0])] for n, s in zip(nss, shapes)]
    return waves, counts


class _DevMem:
    """Minimal __cuda_array_interface__ holder so torch can view library-owned device memory."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


class PeerWaveSlab:
    """Root-owned output slab for the multi-GPU exchange step, written by peer stores over NVLink/NVSwitch.

    Layout (fp32 payload, then int64 meta):  wave[rank][slot][b_cap * l_cap]   meta[rank][slot][2 + b_cap] = (B, L, n_samples[B])
    The slab is cudaMalloc'ed by libbv2 on rank `dst` and exported with CUDA IPC (bv2_peer_slab_alloc / _open,
    include/bv2.h); every rank gets the address of its own slice (`wave_ptr`) and hands it to the engine as the output
    pointer of `infer_finish`, so the waveform never exists in the producer's memory and no NCCL payload moves.
    `publish` adds the per-batch meta record (one small peer copy) and a 1-element all-reduce as the completion signal: when
    it completes on `dst`, every rank's stores of that slot are done.  `slots` >= 2 lets step i+1 be produced while
    the root consumes step i.  Back-pressure: `release(slot)` (collective, every rank calls it once per publish of that slot, the
    root AFTER it has copied what `collect` returned) posts a 1-element broadcast from the root; `wait(slot)` orders the next
    producer after both the completion flag and that release, so a peer can never overwrite a slot the root is still reading.
    With world_size 1 (or torch.distributed not initialised) everything stays local.
    """

    def __init__(self, device, b_cap: int, l_cap: int, dst: int = 0, slots: int = 2):
        import ctypes as C
        from . import _lib
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.dst, self.slots, self.b_cap, self.l_cap = dst, slots, int(b_cap), int(l_cap)
        self.meta_len = 2 + self.b_cap
        self.wave_bytes = self.world * slots * self.b_cap * self.l_cap * 4
        self.meta_bytes = self.world * slots * self.meta_len * 8
        self.owner = self.rank == dst
        handle = torch.zeros(64, dtype=torch.uint8)
        p = C.c_void_p()
        self.base = 0
        rc = 0
        if self.owner:
            buf = (C.c_ubyte * 64)()
            rc = self.lib.bv2_peer_slab_alloc(self.dev_index, self.wave_bytes + self.meta_bytes, C.byref(p), buf)
            if rc == 0:
                handle = torch.tensor(list(buf), dtype=torch.uint8)
        if self.world > 1:
            # construction is collective: every rank reaches the broadcast and the status exchange even when a step failed,
            # so a missing IPC capability raises on ALL ranks instead of hanging the others
            h = handle.to(self.device)
            dist.broadcast(h, src=dst)
            handle = h.cpu()
            if not self.owner and bool(handle.any()):
                buf = (C.c_ubyte * 64)(*handle.tolist())
                rc = self.lib.bv2_peer_slab_open(self.dev_index, buf, C.byref(p))
            elif not self.owner:
                rc = -3
            bad = torch.tensor([1.0 if rc != 0 else 0.0], device=self.device)
            dist.all_reduce(bad)
            if float(bad) > 0:
                if rc == 0 and p.value:
                    (self.lib.bv2_peer_slab_free if self.owner else self.lib.bv2_peer_slab_close)(self.dev_index, p)
                raise RuntimeError(f"PeerWaveSlab: CUDA IPC slab setup failed on {int(bad)} rank(s) (local status {rc})")
        self._check(rc, "alloc")
        self.base = int(p.value)
        self._flag = [torch.zeros(1, device=self.device) for _ in range(slots)]
        self._work = [None] * slots
        self._rel = [torch.zeros(1, device=self.device) for _ in range(slots)]
        self._rel_work = [None] * slots
        self._keep = [None] * slots
        self._meta_host = [torch.zeros(self.meta_len, dtype=torch.int64).pin_memory() for _ in range(slots)]
        self._meta_dev = [torch.zeros(self.meta_len, dtype=torch.int64, device=self.device) for _ in range(slots)]
        self._meta_ev = [None] * slots

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"PeerWaveSlab {what} failed with status {rc} (CUDA IPC / peer access unavailable?)")

    def _stream(self):
        import ctypes as C
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def wave_ptr(self, slot: int, rank: int = None) -> int:
        r = self.rank if rank is None else rank
        return self.base + ((r * self.slots + slot) * self.b_cap * self.l_cap) * 4

    def _meta_ptr(self, slot: int, rank: int) -> int:
        return self.base + self.wave_bytes + ((rank * self.slots + slot) * self.meta_len) * 8

    def fits(self, B: int, L: int) -> bool:
        return B <= self.b_cap and B * L <= self.b_cap * self.l_cap

    def publish(self, slot: int, B: int, L: int, n_samples, wave: torch.Tensor = None):
        """Record (B, L, n_samples[B] -- host sequence / array) for this rank's slot and signal completion.  `wave` (optional, [B,1,L] on this device) is
        copied into the slot first -- the API-level variant for callers that already hold the tensor; the fused variant
        passes `wave_ptr(slot)` to Engine.infer_finish instead and leaves `wave` None."""
        import ctypes as C
        if not self.fits(B, L):
            raise ValueError(f"batch [{B}, {L}] exceeds the slab slot capacity [{self.b_cap}, {self.l_cap}]")
        if self._meta_ev[slot] is not None:
            self._meta_ev[slot].synchronize()  # the previous H2D out of this slot's pinned record has long finished
        mh = self._meta_host[slot]
        mh.zero_()
        mh[0], mh[1] = B, L
        mh[2:2 + B] = torch.as_tensor(n_samples).to(device="cpu", dtype=torch.int64)
        meta = self._meta_dev[slot]
        meta.copy_(mh, non_blocking=True)
        ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(self.device)); self._meta_ev[slot] = ev
        st = self._stream()
        if wave is not None:
            w = wave.contiguous()
            self._check(self.lib.bv2_peer_write(self.dev_index, C.c_void_p(self.wave_ptr(slot)), C.c_void_p(w.data_ptr()), B * L * 4, st), "write")
        self._check(self.lib.bv2_peer_write(self.dev_index, C.c_void_p(self._meta_ptr(slot, self.rank)), C.c_void_p(meta.data_ptr()),
                                            self.meta_len * 8, st), "write")
        self._keep[slot] = (meta, wave)  # sources stay alive until the slot is reused
        if self.world > 1:
            self._work[slot] = dist.all_reduce(self._flag[slot], async_op=True)

    def wait(self, slot: int):
        """Order the current stream after every rank's stores into `slot` and after the root's release of it (no host block)."""
        w = self._work[slot]
        if w is not None:
            w.wait()
            self._work[slot] = None
        r = self._rel_work[slot]
        if r is not None:
            r.wait()
            self._rel_work[slot] = None

    def release(self, slot: int):
        """Collective: the root declares `slot` consumed (call it after copying out what collect() returned -- the broadcast is
        enqueued behind that work on the root's stream); producers only post the matching receive.  Views returned by collect()
        for this slot are invalid afterwards."""
        if self.world > 1:
            self._rel_work[slot] = dist.broadcast(self._rel[slot], src=self.dst, async_op=True)

    def collect(self, slot: int) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
        """Root only: per-rank waveform views [B_r,1,L_r] into the slab + sample counts, valid until release(slot): copy them out,
        then call release(slot) on every rank."""
        w = self._work[slot]
        if w is not None:
            w.wait()
            self._work[slot] = None
        if not self.owner:
            return [], []
        torch.cuda.current_stream(self.device).synchronize()
        waves, counts = [], []
        for r in range(self.world):
            m = torch.as_tensor(_DevMem(self._meta_ptr(slot, r), (self.meta_len,), "<i8"), device=self.device).cpu()
            B, L = int(m[0]), int(m[1])
            w = torch.as_tensor(_DevMem(self.wave_ptr(slot, r), (B, 1, L), "<f4"), device=self.device) if B * L else \
                torch.empty(0, 1, 0, device=self.device)
            waves.append(w)
            counts.append(m[2:2 + B].clone())
        return waves, counts

    def close(self):
        import ctypes as C
        if getattr(self, "base", 0):
            torch.cuda.synchronize(self.device)
            if self.world > 1:
                dist.barrier()  # nobody frees/unmaps while a peer may still store
            if self.owner:
                self.lib.bv2_peer_slab_free(self.dev_index, C.c_void_p(self.base))
            else:
                self.lib.bv2_peer_slab_close(self.dev_index, C.c_void_p(self.base))
            self.base = 0
