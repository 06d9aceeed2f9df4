"""NVSwitch symmetric-memory engine: the per-group state behind every fused collective kernel.

There is no counterpart in the reference — its communicators are NCCL handles
(rust/bagua-core/bagua-core-internal/src/communicators/mod.rs:26-73).  On an HGX H100 every GPU reaches every
peer at full NVLink 4 bandwidth through NVSwitch, so a group's "communicator" here is:

* symmetric device memory: identical allocations on every rank, each mapped into every peer's address space
  (+ an NVLS multicast alias when the fabric offers it).  Allocation/handle exchange is bootstrapped with
  ``torch.distributed._symmetric_memory`` (CUDA VMM + fd passing); the kernels are ours.
* a signal pad (epoch flags) in that memory + an abort flag → ``_C.PeerComm``.
* a slab allocator handing out slices for bucket storage, peer replicas and quantised in/out boxes.
"""
from __future__ import annotations

import logging
import os
from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.distributed as dist

from .. import env
from ..core import dtype_code, native

logger = logging.getLogger(__name__)

_ALIGN = 1024                       # slice alignment (bytes); ≥ 16 B vectors, keeps TMA/128 B lines happy
_SLAB_BYTES = 256 * 1024 ** 2       # symmetric memory is requested in slabs of this size (or larger on demand)
ONE_SHOT_SLOT = 512 * 1024          # staging slot per (parity, rank) of the one-shot allreduce


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


class _Slab:
    def __init__(self, engine: "PeerEngine", nbytes: int):
        self.nbytes = nbytes
        ptrs, mc = None, 0
        if engine.world > 1 or engine.self_peer_symm:
            try:
                import torch.distributed._symmetric_memory as symm_mem

                self.tensor = symm_mem.empty(nbytes, dtype=torch.uint8, device=engine.device)
                self.tensor.zero_()
                self.handle = symm_mem.rendezvous(self.tensor, engine.torch_pg)
                ptrs = [int(p) for p in self.handle.buffer_ptrs]
                if engine.use_multicast:
                    try:
                        mc = int(self.handle.multicast_ptr or 0)
                    except Exception:  # noqa: BLE001
                        mc = 0
            except Exception:  # noqa: BLE001
                if engine.world > 1:
                    raise
                engine.self_peer_symm = False  # a 1-rank group that torch's allocator will not rendezvous: plain memory below
                ptrs = None
        if ptrs is None:
            # self-peer mode (world == 1): "every peer" is this GPU, ordinary device memory is symmetric by definition
            self.tensor = torch.zeros(nbytes, dtype=torch.uint8, device=engine.device)
            self.handle = None
            ptrs = [self.tensor.data_ptr()]
        self.ptrs = ptrs
        self.mc = mc
        self.buf = native().SymmBuf(ptrs, mc, nbytes)
        self.free_list: List[List[int]] = [[0, nbytes]]  # [offset, size], kept sorted and coalesced

    def alloc(self, nbytes: int) -> Optional[int]:
        for i, (off, size) in enumerate(self.free_list):
            if size >= nbytes:
                if size == nbytes:
                    self.free_list.pop(i)
                else:
                    self.free_list[i] = [off + nbytes, size - nbytes]
                return off
        return None

    def free(self, off: int, nbytes: int):
        self.free_list.append([off, nbytes])
        self.free_list.sort()
        merged: List[List[int]] = []
        for o, s in self.free_list:
            if merged and merged[-1][0] + merged[-1][1] == o:
                merged[-1][1] += s
            else:
                merged.append([o, s])
        self.free_list = merged


@dataclass
class SymmSlice:
    """``nbytes`` of symmetric memory: ``tensor`` is this rank's view; ``buf``/``offset`` address the same bytes on peers."""

    slab: _Slab
    offset: int
    nbytes: int
    tensor: torch.Tensor

    @property
    def buf(self):
        return self.slab.buf

    @property
    def has_multicast(self) -> bool:
        return self.slab.mc != 0

    def view(self, dtype: torch.dtype, numel: Optional[int] = None) -> torch.Tensor:
        t = self.tensor.view(dtype)
        return t if numel is None else t[:numel]

    def free(self):
        if self.slab is not None:
            self.slab.free(self.offset, self.nbytes)
            self.slab = None


class PeerEngine:
    """Owns the symmetric memory, signal pads and kernel-variant policy of one process group."""

    @classmethod
    def create(cls, group) -> Optional["PeerEngine"]:
        if not torch.cuda.is_available() or os.environ.get("BAGUA_FORCE_CPU", "0") == "1":
            return None
        if env.get_allreduce_variant() == "nccl":
            return None
        n = len(group.ranks)
        # n == 1: nothing to exchange — but BAGUA_SELF_PEER=1 still builds the engine with this GPU as its only peer, so the very
        # same kernels / ops / bucket programs run (slices, barriers, optimizer epilogue) on a single-GPU box: used by smoke(),
        # the 1-GPU tests and `ncu` captures of the peer kernels (ncu cannot wrap a multi-rank job).
        if n == 1 and os.environ.get("BAGUA_SELF_PEER", "0") != "1":
            return None
        if n > native().MAX_PEERS or group.nnodes != 1:
            return None
        if dist.get_rank() not in group.ranks:
            return None
        return cls(group)

    def __init__(self, group):
        C = native()
        self.group = group
        self.torch_pg = group.torch_group
        self.world = len(group.ranks)
        self.rank = group.ranks.index(dist.get_rank())
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.use_multicast = os.environ.get("BAGUA_DISABLE_MULTICAST", "0") != "1"
        self.self_peer_symm = self.world == 1 and os.environ.get("BAGUA_SELF_PEER_SYMM", "0") == "1"  # torch symm_mem also works alone, but a 1-device multicast object is refused by the driver (measured): plain memory by default
        self._slabs: List[_Slab] = []
        # signal pads first: their own tiny symmetric allocation, zeroed before anybody can signal
        pad = self._new_slab(_round_up(C.signal_pad_bytes(), 4096), track=False)
        self._pad_slab = pad
        self.comm = C.PeerComm(self.rank, self.world, self.device.index, pad.ptrs, env.get_peer_kernel_timeout_s())
        # The blocking API (bagua.allreduce_inplace & co, SyncBatchNorm) is driven by the TRAINING thread while the scheduler's worker
        # issues bucket kernels: two issue orders that are not the same on every rank. They therefore get their own signal pad
        # (barriers pair only with their own kind), their own staging / workspace and their own stream (one kind can never queue
        # behind a spinning kernel of the other kind).
        pad2 = self._new_slab(_round_up(C.signal_pad_bytes(), 4096), track=False)
        self._pad_slab2 = pad2
        self.comm_blocking = C.PeerComm(self.rank, self.world, self.device.index, pad2.ptrs, env.get_peer_kernel_timeout_s())
        self.blocking_stream = torch.cuda.Stream(device=self.device, priority=-1)
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=self.torch_pg)
        self.has_multicast = pad.mc != 0
        self._staging: Optional[SymmSlice] = None
        self._workspace: Optional[SymmSlice] = None
        self.sm_count = torch.cuda.get_device_properties(self.device).multi_processor_count
        logger.info("bagua_b200 PeerEngine: group %s rank %d/%d multicast=%s", group.group_name, self.rank, self.world, self.has_multicast)
        self.variant_table = None
        if os.environ.get("BAGUA_PEER_CALIBRATE", "0") == "1":
            self.calibrate()

    # -- allocation ------------------------------------------------------------------------------------------------
    def _new_slab(self, nbytes: int, track: bool = True) -> _Slab:
        slab = _Slab(self, nbytes)
        if track:
            self._slabs.append(slab)
        return slab

    def alloc(self, nbytes: int) -> SymmSlice:
        """Collective: every rank of the group must request the same sizes in the same order."""
        nbytes = _round_up(max(int(nbytes), 1), _ALIGN)
        for slab in self._slabs:
            off = slab.alloc(nbytes)
            if off is not None:
                return SymmSlice(slab, off, nbytes, slab.tensor[off : off + nbytes])
        slab = self._new_slab(max(_SLAB_BYTES, _round_up(nbytes, 2 * 1024 ** 2)))
        off = slab.alloc(nbytes)
        return SymmSlice(slab, off, nbytes, slab.tensor[off : off + nbytes])

    # -- policy ------------------------------------------------------------------------------------------------------
    def calibrate(self, sizes=(64 * 1024, 1024 ** 2, 16 * 1024 ** 2, 128 * 1024 ** 2), iters: int = 10, dtype: torch.dtype = torch.bfloat16):
        """Measure every allreduce variant (and a few CTA counts) at a handful of message sizes on THIS fabric and keep, per
        size class, the fastest one — "variant per message size from measured bus bandwidth".  Collective; times are
        CUDA-event durations reduced with MAX over ranks, so every rank derives the identical table.  Enabled with
        ``BAGUA_PEER_CALIBRATE=1`` (or called explicitly); the table is also handed to the autotune service as the prior."""
        C = native()
        stream = torch.cuda.current_stream()
        table = []
        for nbytes in sizes:
            sl = self.alloc(nbytes)
            sl.view(dtype).normal_()
            best = None
            cands = ([("one_shot", b) for b in (4, 8)] if nbytes <= ONE_SHOT_SLOT else []) + [("two_shot", b) for b in (8, 16, 32)]
            if self.has_multicast:
                cands += [("multimem", b) for b in (8, 16)]
            for variant, blocks in cands:
                op, chosen = self.make_allreduce_op(sl, sl, nbytes, dtype, True, variant, blocks=blocks)
                for _ in range(2):
                    C.run_op(op, stream.cuda_stream, self.device.index)
                stream.synchronize()
                dist.barrier(group=self.torch_pg)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record(stream)
                for _ in range(iters):
                    C.run_op(op, stream.cuda_stream, self.device.index)
                e.record(stream)
                stream.synchronize()
                t = torch.tensor([s.elapsed_time(e) / iters], device=self.device)
                dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.torch_pg)
                ms = float(t.item())
                busbw = nbytes / ms / 1e6 * 2 * (self.world - 1) / self.world
                if best is None or ms < best["ms"]:
                    best = {"bytes": nbytes, "variant": chosen, "blocks": blocks, "ms": ms, "busbw_GBs": busbw}
            sl.free()
            table.append(best)
        self.variant_table = table
        logger.info("bagua_b200 allreduce calibration: %s", table)
        return table

    def _from_table(self, nbytes: int):
        table = getattr(self, "variant_table", None)
        if not table:
            return None
        # nearest calibrated size on a log scale
        import math

        return min(table, key=lambda r: abs(math.log2(max(nbytes, 1)) - math.log2(r["bytes"])))

    def choose_variant(self, nbytes: int, requested: str = "auto") -> str:
        v = requested if requested not in (None, "", "auto") else env.get_allreduce_variant()
        if v in ("one_shot", "two_shot"):
            return v
        if v == "multimem":
            return "multimem" if self.has_multicast else "two_shot"
        row = self._from_table(nbytes)
        if row is not None and not (row["variant"] == "one_shot" and nbytes > ONE_SHOT_SLOT):
            return row["variant"]
        if nbytes <= ONE_SHOT_SLOT // 2:
            return "one_shot"
        # with 2 ranks each GPU pulls half the bucket either way, so the in-switch reduction saves nothing and the peer-load two-shot
        # kernel is used; from 4 ranks on multimem moves ~N/2 x fewer bytes over each GPU's links
        if self.world <= 2:
            return "two_shot"
        return "multimem" if self.has_multicast else "two_shot"

    def launch_cfg(self, variant: str, nbytes: int, blocks: int = 0):
        C = native()
        env_blocks = int(os.environ.get("BAGUA_COMM_BLOCKS", "0"))
        if blocks <= 0:
            blocks = env_blocks
        if blocks <= 0:
            row = self._from_table(nbytes)
            if row is not None and row["variant"] == variant:
                blocks = row["blocks"]
        if blocks <= 0:
            vecs = max(nbytes // 16, 1)
            if variant == "one_shot":
                blocks = max(1, min(8, vecs // 512))
            elif variant == "multimem":
                blocks = max(1, min(8, vecs // (self.world * 2048)))  # 8 CTAs of 512 threads keep enough NVLS requests in flight
            else:
                blocks = max(1, min(32, vecs // (self.world * 2048)))
        return C.LaunchCfg(int(min(blocks, C.MAX_COMM_BLOCKS)), 512)

    def staging(self, blocking: bool = False) -> SymmSlice:
        """One-shot staging area (double-buffered by call parity); the blocking communicator has its own."""
        if blocking:
            if getattr(self, "_staging_blocking", None) is None:
                self._staging_blocking = self.alloc(2 * self.world * ONE_SHOT_SLOT)
            return self._staging_blocking
        if self._staging is None:
            self._staging = self.alloc(2 * self.world * ONE_SHOT_SLOT)
        return self._staging

    # -- op factories ----------------------------------------------------------------------------------------------
    def make_allreduce_op(self, src: SymmSlice, dst: SymmSlice, nbytes: int, dtype: torch.dtype, average: bool, variant: str = "auto",
                          src_off: int = 0, dst_off: int = 0, blocks: int = 0, comm=None):
        """Native op reducing ``nbytes`` at ``src``(+off) over all ranks into ``dst``(+off) on all ranks."""
        C = native()
        comm = comm if comm is not None else self.comm
        blocking = comm is not self.comm
        v = self.choose_variant(nbytes, variant)
        scale = 1.0 / self.world if average else 1.0
        nbytes16 = _round_up(nbytes, 16)
        if v == "one_shot" and nbytes16 <= ONE_SHOT_SLOT:
            st = self.staging(blocking)
            return C.AllReduceOneShotOp(comm, st.buf, st.offset, ONE_SHOT_SLOT, src.tensor.data_ptr() + src_off, dst.tensor.data_ptr() + dst_off,
                                        nbytes16, dtype_code(dtype), scale, self.launch_cfg("one_shot", nbytes16, blocks)), "one_shot"
        if v == "one_shot":
            v = "multimem" if self.has_multicast else "two_shot"
        if v == "multimem" and not (src.has_multicast and dst.has_multicast):
            v = "two_shot"
        code = C.AR_MULTIMEM if v == "multimem" else C.AR_TWO_SHOT
        op = C.AllReduceOp(comm, src.buf, dst.buf, src.offset + src_off, dst.offset + dst_off, nbytes16, dtype_code(dtype), scale, code,
                           self.launch_cfg(v, nbytes16, blocks))
        return op, v

    # -- blocking-API fast path --------------------------------------------------------------------------------------
    class _BlockingRegion:
        """Work of the blocking API: ordered after the caller's current stream, executed on the engine's own blocking stream with
        the blocking communicator, and finished (host wait) on exit — never queued behind a bucket kernel of the comm stream."""

        def __init__(self, eng: "PeerEngine"):
            self.eng = eng

        def __enter__(self):
            self.eng.comm_blocking.check_fatal("a blocking collective")
            bs = self.eng.blocking_stream
            bs.wait_stream(torch.cuda.current_stream())
            self.ctx = torch.cuda.stream(bs)
            self.ctx.__enter__()
            return bs

        def __exit__(self, *exc):
            self.ctx.__exit__(*exc)
            self.eng.blocking_stream.synchronize()
            if exc[0] is None:
                self.eng.comm_blocking.check_fatal("this blocking collective")
            return False

    def blocking_region(self):
        return PeerEngine._BlockingRegion(self)

    def allreduce_tensor(self, tensor: torch.Tensor, average: bool) -> bool:
        """Blocking all-reduce of an arbitrary contiguous CUDA tensor through the peer kernels (see :meth:`blocking_region`)."""
        C = native()
        nbytes = tensor.numel() * tensor.element_size()
        if nbytes == 0:
            return True
        scale = 1.0 / self.world if average else 1.0
        with self.blocking_region() as bs:
            stream = bs.cuda_stream
            if nbytes % 16 == 0 and tensor.data_ptr() % 16 == 0 and nbytes <= ONE_SHOT_SLOT:
                st = self.staging(blocking=True)
                op = C.AllReduceOneShotOp(self.comm_blocking, st.buf, st.offset, ONE_SHOT_SLOT, tensor.data_ptr(), tensor.data_ptr(), nbytes,
                                          dtype_code(tensor.dtype), scale, self.launch_cfg("one_shot", nbytes))
                C.run_op(op, stream, self.device.index)
                return True
            padded = _round_up(nbytes, 16 * self.world)
            ws = self._ensure_workspace(padded)
            flat = ws.tensor[:nbytes].view(tensor.dtype)
            flat.copy_(tensor.reshape(-1))
            if padded > nbytes:
                ws.tensor[nbytes:padded].zero_()
            op, _ = self.make_allreduce_op(ws, ws, padded, tensor.dtype, average, "auto", comm=self.comm_blocking)
            C.run_op(op, stream, self.device.index)
            tensor.reshape(-1).copy_(flat)
        return True

    def _ensure_workspace(self, nbytes: int) -> "SymmSlice":
        if self._workspace is None or self._workspace.nbytes < nbytes:
            self._workspace = self.alloc(max(nbytes, 64 * 1024 ** 2))  # collective growth: every rank sees the same message sizes
        return self._workspace

    def allgather_tensor(self, send: torch.Tensor, recv: torch.Tensor) -> bool:
        """``recv`` = concatenation of every rank's ``send`` (any dtype, moved as 16-byte vectors): own chunk → symmetric
        workspace → ``all_gather_kernel`` (peer stores / multimem.st) → ``recv``.  False when the shape is not eligible."""
        C = native()
        sb = send.numel() * send.element_size()
        if sb == 0 or sb % 16 or recv.numel() * recv.element_size() != sb * self.world or not (send.is_contiguous() and recv.is_contiguous()):
            return False
        total = sb * self.world
        with self.blocking_region() as bs:
            ws = self._ensure_workspace(total)
            ws.tensor[self.rank * sb: (self.rank + 1) * sb].copy_(send.reshape(-1).view(torch.uint8))
            use_mc = bool(ws.has_multicast and self.has_multicast)
            op = C.AllGatherOp(self.comm_blocking, ws.buf, ws.offset, total, dtype_code(torch.float32), use_mc,
                               self.launch_cfg("multimem" if use_mc else "two_shot", total))
            C.run_op(op, bs.cuda_stream, self.device.index)
            recv.reshape(-1).view(torch.uint8).copy_(ws.tensor[:total])
        return True

    def reduce_scatter_tensor(self, send: torch.Tensor, recv: torch.Tensor, average: bool) -> bool:
        """``recv`` = sum (or mean) over ranks of chunk ``rank`` of ``send``: ``send`` → symmetric workspace →
        ``reduce_scatter_kernel`` (peer loads / multimem.ld_reduce) → ``recv``."""
        C = native()
        rb = recv.numel() * recv.element_size()
        if (rb == 0 or rb % 16 or send.numel() != recv.numel() * self.world or send.dtype != recv.dtype
                or send.dtype not in (torch.float32, torch.float16, torch.bfloat16) or not (send.is_contiguous() and recv.is_contiguous())):
            return False
        total = rb * self.world
        with self.blocking_region() as bs:
            ws = self._ensure_workspace(total)
            ws.tensor[:total].view(send.dtype).copy_(send.reshape(-1))
            use_mc = bool(ws.has_multicast and self.has_multicast)
            op = C.ReduceScatterOp(self.comm_blocking, ws.buf, ws.offset, total, dtype_code(send.dtype), (1.0 / self.world) if average else 1.0, use_mc,
                                   self.launch_cfg("multimem" if use_mc else "two_shot", total))
            C.run_op(op, bs.cuda_stream, self.device.index)
            recv.reshape(-1).copy_(ws.tensor[self.rank * rb: (self.rank + 1) * rb].view(recv.dtype))
        return True

    def barrier(self, stream: Optional[torch.cuda.Stream] = None):
        s = (stream or torch.cuda.current_stream()).cuda_stream
        self.comm.barrier(s)

    def check_error(self):
        """Raise if a kernel of this engine has failed (non-synchronising: reads the host-mapped error mirrors)."""
        self.comm.check_fatal("further communication")
        self.comm_blocking.check_fatal("further communication")
