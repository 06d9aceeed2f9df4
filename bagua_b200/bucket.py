"""Buckets: groups of tensors fused into one flat message plus the communication program that runs on it.

Reference: ``bagua/torch_api/bucket.py:18-366`` (API parity: padding/alignment, flatten, ``append_*_op``).

H100-first: when the group has a :class:`~bagua_b200.parallel.symm.PeerEngine`, the flat storage of a bucket is a
slice of NVSwitch *symmetric memory* — the gradients (or weights) autograd/optimizers write are directly loadable
by every peer GPU, so a bucket's op is a single fused kernel (no staging copy, no NCCL).  Without an engine
(CPU/gloo, multi-node, ``BAGUA_ALLREDUCE_VARIANT=nccl``) the same ops run on ``torch.distributed``.
"""
from __future__ import annotations

import os
from typing import Callable, List, Optional

import torch
import torch.distributed as dist

from . import communication as comm_mod
from .core import dtype_code, native
from .ops import quant
from .tensor import dense_strides
from .utils import check_contiguous

__all__ = ["BaguaBucket", "BucketArena", "bucket_arena"]

_ARENA_ALIGN = 1024


class _ArenaSlice:
    """A window of a :class:`BucketArena`; same duck type as ``symm.SymmSlice`` (buf / offset / tensor / view)."""

    def __init__(self, arena: "BucketArena", offset: int, nbytes: int):
        self.arena = arena
        self.rel = offset
        self.nbytes = nbytes
        self.tensor = arena.tensor[offset : offset + nbytes]

    @property
    def buf(self):
        return self.arena.slice.buf if self.arena.slice is not None else None

    @property
    def offset(self) -> int:
        return (self.arena.slice.offset if self.arena.slice is not None else 0) + self.rel

    @property
    def has_multicast(self) -> bool:
        return self.arena.slice is not None and self.arena.slice.has_multicast

    @property
    def symmetric(self) -> bool:
        return self.arena.slice is not None

    def view(self, dtype, numel=None):
        t = self.tensor.view(dtype)
        return t if numel is None else t[:numel]

    def free(self):
        pass


class BucketArena:
    """One contiguous allocation holding every bucket of a model: NVSwitch symmetric memory when the group has a peer
    engine, ordinary device/host memory otherwise.  Contiguity is what lets the fused optimizer update the whole model
    with a single kernel launch."""

    def __init__(self, group, device: torch.device, capacity_bytes: int):
        eng = group.peer_engine() if device.type == "cuda" else None
        if eng is None and device.type == "cuda" and getattr(group, "nnodes", 1) > 1:
            hier = group.hier_engine()  # multi-node: the arena lives in the NODE's symmetric memory (intra-node kernels)
            eng = hier[0] if hier is not None else None
        capacity_bytes = max(int(capacity_bytes), _ARENA_ALIGN)
        self.engine = eng
        if eng is not None:
            self.slice = eng.alloc(capacity_bytes)
            self.tensor = self.slice.tensor
            self.tensor.zero_()
        else:
            self.slice = None
            self.tensor = torch.zeros(capacity_bytes, dtype=torch.uint8, device=device)
        self.capacity = capacity_bytes
        self.cursor = 0

    def take(self, nbytes: int) -> Optional[_ArenaSlice]:
        nbytes = (int(nbytes) + _ARENA_ALIGN - 1) // _ARENA_ALIGN * _ARENA_ALIGN
        if self.cursor + nbytes > self.capacity:
            return None
        s = _ArenaSlice(self, self.cursor, nbytes)
        self.cursor += nbytes
        return s

    def free(self):
        if self.slice is not None:
            self.slice.free()
            self.slice = None

    @staticmethod
    def required_bytes(bucket_bytes: List[int], slack: int = 2 * _ARENA_ALIGN) -> int:
        return sum((b + slack + _ARENA_ALIGN - 1) // _ARENA_ALIGN * _ARENA_ALIGN for b in bucket_bytes)


_current_arena: List[Optional[BucketArena]] = [None]


class bucket_arena:
    """``with bucket_arena(arena): ...`` — buckets flattened inside take their storage from ``arena``."""

    def __init__(self, arena: Optional[BucketArena]):
        self.arena = arena

    def __enter__(self):
        self.prev = _current_arena[0]
        _current_arena[0] = self.arena
        return self.arena

    def __exit__(self, *exc):
        _current_arena[0] = self.prev
        return False


class _DecentralizedOpHandle:
    """What ``append_decentralized_synchronous_op`` returns: lets the algorithm copy the averaged peer weights back."""

    def __init__(self, bucket: "BaguaBucket", peer_weight: torch.Tensor):
        self.bucket = bucket
        self.peer_weight = peer_weight

    def copy_back_peer_weight(self, bucket: Optional["BaguaBucket"] = None):
        b = bucket if bucket is not None else self.bucket
        flat = b.backend_tensor
        with torch.no_grad():
            if flat is not None:
                flat.copy_(self.peer_weight.view(-1)[: flat.numel()])
            else:
                off = 0
                for t in b._all_tensors:
                    eff = t.bagua_getter_closure()
                    eff.copy_(self.peer_weight.view(-1)[off : off + eff.numel()].view_as(eff))
                    off += eff.numel()


class BaguaBucket:
    """A group of bagua tensors communicated together (reference bagua/torch_api/bucket.py:18-366): optionally flattened into one
    contiguous slice of the model's bucket arena (NVSwitch symmetric memory on GPUs), carrying the ordered list of communication
    ops the scheduler runs once every tensor of the bucket is ready."""
    def __init__(self, tensors: List[torch.Tensor], name: str, flatten: bool, alignment: int = 1, group=None):
        """
        Args:
            tensors: bagua tensors (see :meth:`torch.Tensor.ensure_bagua_tensor`) of one dtype/device.
            name: unique bucket name.
            flatten: make the effective tensors views of one flat storage.
            alignment: pad with an always-ready zero tensor so that ``numel % alignment == 0``.
            group: process group whose symmetric memory backs the flat storage (default group if ``None``).
        """
        self.tensors = list(tensors)
        self.bagua_module_name = tensors[0].bagua_module_name
        for t in self.tensors:
            assert self.bagua_module_name == t.bagua_module_name, "every tensor in the same bucket should have the same model name"
        self._bagua_backend = comm_mod.get_backend(self.bagua_module_name)
        self.name = name
        self._group = group
        self.padding_tensor = None
        eff0 = self.tensors[0].bagua_getter_closure()
        kinds = {(t.bagua_getter_closure().dtype, t.bagua_getter_closure().device) for t in self.tensors}
        if len(kinds) > 1:   # the reference's backend rejects such a bucket as well (bagua-core-internal/src/datatypes/mod.rs:1135-1147)
            raise ValueError(f"bucket {name!r}: all tensors of a bucket must share one dtype and one device, got {sorted(str(k) for k in kinds)}")
        if alignment > 1:
            padding = sum(t.bagua_getter_closure().numel() for t in self.tensors) % alignment
            if padding > 0:
                padding = alignment - padding
                # the padding tensor never gets a ready mark: the scheduler treats it as always ready
                self.padding_tensor = torch.zeros(padding, dtype=eff0.dtype, device=eff0.device).ensure_bagua_tensor(
                    "bagua_padding_tensor_bucket_" + name, module_name=self.bagua_module_name
                )
        self._all_tensors = self.tensors + [self.padding_tensor] if self.padding_tensor is not None else list(self.tensors)
        self.backend_tensor: Optional[torch.Tensor] = None
        self._slice = None          # SymmSlice backing the flat storage (peer engine only)
        self._aux_slices = []       # symmetric scratch owned by the ops (quantised in/out boxes)
        self._companion_slices = []  # symmetric replicas handed to algorithms (peer_weight, ...)
        self._ops_keepalive = []
        self.flatten = flatten
        if self.flatten:
            self._flatten_()
        self.backend_bucket = native().Bucket(name, [t.bagua_backend_tensor() for t in self._all_tensors])
        if self.padding_tensor is not None:
            self.backend_bucket.mark_padding(len(self._all_tensors) - 1)
        for t in self._all_tensors:
            t._bagua_bucket = self
            t._bagua_backend = self._bagua_backend

    # ------------------------------------------------------------------------------------------------------------
    def _process_group(self, group=None):
        return group if group is not None else (self._group if self._group is not None else comm_mod._get_default_group())

    def _engine(self, group=None):
        eff = self._all_tensors[0].bagua_getter_closure()
        if eff.device.type != "cuda":
            return None
        return self._process_group(group).peer_engine()

    def flattened_tensor(self) -> torch.Tensor:
        """A new contiguous tensor with the data of all effective tensors (+ padding)."""
        effs = [t.bagua_getter_closure() for t in self._all_tensors]
        total = sum(e.numel() for e in effs)
        flat = torch.zeros(total, dtype=effs[0].dtype, device=effs[0].device)
        off = 0
        with torch.no_grad():
            for e in effs:
                flat[off : off + e.numel()].copy_(e.reshape(-1))
                off += e.numel()
        return flat

    def _flatten_(self):
        """Make every effective tensor a view of one flat storage (symmetric memory when available)."""
        effs = [t.bagua_getter_closure() for t in self._all_tensors]
        total = sum(e.numel() for e in effs)
        eng = self._engine()
        arena = _current_arena[0]
        taken = arena.take(total * effs[0].element_size()) if (arena is not None and arena.tensor.device == effs[0].device) else None
        with torch.no_grad():
            if taken is not None:
                flat = taken.view(effs[0].dtype, total)
                if taken.symmetric:
                    self._slice = taken
            elif eng is not None:
                self._slice = eng.alloc(total * effs[0].element_size())
                flat = self._slice.view(effs[0].dtype, total)
            elif self.check_flatten():
                flat = torch.empty(0, dtype=effs[0].dtype, device=effs[0].device).set_(
                    effs[0].untyped_storage(), effs[0].storage_offset(), (total,)
                )
                self.backend_tensor = flat
                return
            else:
                flat = torch.zeros(total, dtype=effs[0].dtype, device=effs[0].device)
            storage = flat.untyped_storage()
            off = flat.storage_offset()
            for t, e in zip(self._all_tensors, effs):
                # copy in *memory* order (dense permutations such as channels_last keep their strides)
                dst = torch.empty(0, dtype=e.dtype, device=e.device).set_(storage, off, e.shape, dense_strides(e))
                dst.copy_(e)
                t.bagua_set_storage(storage, off)
                off += e.numel()
        self.backend_tensor = flat
        assert self.check_flatten(), "flatten failed: effective tensors are not contiguous"

    def new_companion(self, init_from_bucket: bool = True, symmetric: bool = False, group=None) -> torch.Tensor:
        """A flat tensor shaped like the bucket (same dtype / numel incl. padding) for replicas such as ``peer_weight``.
        ``symmetric=True`` places it in NVSwitch symmetric memory when the group has a peer engine (collective call);
        the returned tensor then carries ``_bagua_symm_slice``."""
        ref = self.backend_tensor if self.backend_tensor is not None else self.flattened_tensor()
        eng = self._engine(group) if symmetric else None
        if eng is not None:
            sl = eng.alloc(ref.numel() * ref.element_size())
            self._companion_slices.append(sl)
            t = sl.view(ref.dtype, ref.numel())
            t._bagua_symm_slice = sl
        else:
            t = torch.empty_like(ref)
        with torch.no_grad():
            if init_from_bucket:
                t.copy_(ref if self.backend_tensor is not None else self.flattened_tensor())
            else:
                t.zero_()
        return t

    def check_flatten(self) -> bool:
        """True when the effective tensors are back to back in memory."""
        return check_contiguous([t.bagua_getter_closure() for t in self._all_tensors])

    def release(self):
        """Give symmetric slices back to the engine (called when buckets are rebuilt)."""
        for s in self._aux_slices + self._companion_slices:
            s.free()
        self._aux_slices = []
        self._companion_slices = []
        # the flat slice stays alive as long as tensors view it; it is recycled by the engine's allocator only
        # after the owning engine re-buckets (see BaguaDistributedDataParallel._reset_buckets)

    def bytes(self) -> int:
        """Bytes of the effective tensors (padding excluded), as the reference reports (bucket.py:362-366)."""
        return sum(t.bagua_getter_closure().numel() * t.bagua_getter_closure().element_size() for t in self.tensors)

    def numel(self) -> int:
        return sum(t.bagua_getter_closure().numel() for t in self._all_tensors)

    def clear_ops(self) -> "BaguaBucket":
        self.backend_bucket.clear_ops()
        self._ops_keepalive = []
        for s in self._aux_slices:
            s.free()
        self._aux_slices = []
        return self

    # ------------------------------------------------------------------------------------------------------------
    # op builders
    # ------------------------------------------------------------------------------------------------------------
    def _flat_or_gather(self):
        """(flat tensor, scatter_back) — zero-copy when flattened, else a staging copy (reference datatypes/mod.rs:1029-1087)."""
        if self.backend_tensor is not None:
            return self.backend_tensor, None
        flat = self.flattened_tensor()

        def scatter_back():
            off = 0
            with torch.no_grad():
                for t in self._all_tensors:
                    e = t.bagua_getter_closure()
                    e.copy_(flat[off : off + e.numel()].view_as(e))
                    off += e.numel()

        return flat, scatter_back

    def _stream_ctx(self, group):
        s = self._process_group(group).stream
        if s is not None and torch.cuda.is_available():
            return torch.cuda.stream(s)
        import contextlib

        return contextlib.nullcontext()

    def append_python_op(self, python_function: Callable[[str], None], group=None) -> "BaguaBucket":
        """Append a python callable ``fn(bucket_name)``; it runs on the comm worker thread, with the group's comm
        stream current (reference bucket.py:134-165)."""

        def wrapped(name: str):
            with self._stream_ctx(group):
                python_function(name)

        self.backend_bucket.append_python_op(wrapped, "python")
        return self

    def append_centralized_synchronous_op(
        self,
        hierarchical: bool = False,
        average: bool = True,
        scattergather: bool = False,
        compression: Optional[str] = None,
        group=None,
        variant: str = "auto",
        momentum_source=None,
    ) -> "BaguaBucket":
        """Allreduce (optionally MinMaxUInt8-compressed) of the bucket across the group
        (reference bucket.py:167-213; comm ops 1 and 2 of SURVEY §2.5).

        ``hierarchical`` is accepted for API parity; inside one NVSwitch domain the flat kernel is already optimal, and
        across nodes the intra-node / inter-node legs are composed from the group's intra/inter communicators.

        ``momentum_source=(grad_flat, beta1)`` (compressed ops only; QAdam): the bucket holds a first moment and
        ``m = beta1*m + (1-beta1)*grad_flat`` is applied before the exchange — inside the fused kernel's first pass on NVSwitch
        (the reference needs a python op on the comm thread for it, algorithms/q_adam.py:193-221)."""
        pg = self._process_group(group)
        eng = self._engine(group)
        n = pg.size()
        if compression is not None:
            assert compression == "MinMaxUInt8", f"unknown compression {compression}"
            total = self.numel()
            if eng is not None and self._slice is not None and total % (32 * n) == 0:
                C = native()
                box = C.ByteGradOp.box_bytes(total, n)
                inbox, outbox = eng.alloc(box), eng.alloc(box)
                self._aux_slices += [inbox, outbox]
                op = C.ByteGradOp(eng.comm, self.backend_tensor.data_ptr(), total, dtype_code(self.backend_tensor.dtype), inbox.buf, inbox.offset,
                                  outbox.buf, outbox.offset, average,
                                  eng.launch_cfg("two_shot", total, int(os.environ.get("BAGUA_BYTEGRAD_BLOCKS", "0")) or 64))   # measured on BERT-large: 32 CTAs 263, 64: 295-304, 128: 294 samples/s
                if momentum_source is not None:
                    gflat, beta1 = momentum_source
                    assert gflat.dtype == self.backend_tensor.dtype and gflat.numel() == total and gflat.is_contiguous()
                    op.set_momentum_source(gflat.data_ptr(), float(beta1))
                    self._ops_keepalive.append(gflat)
                self.backend_bucket.append_op(op)
                self._ops_keepalive.append(op)
                self.allreduce_variant = "bytegrad_fused" + ("+momentum" if momentum_source is not None else "")
                return self
            if momentum_source is not None:
                gflat, beta1 = momentum_source

                def momentum(_name: str):
                    flat, scatter_back = self._flat_or_gather()
                    with torch.no_grad():
                        flat.mul_(beta1).add_(gflat.view(-1)[: flat.numel()], alpha=1 - beta1)
                    if scatter_back is not None:
                        scatter_back()

                self.append_python_op(momentum, group=group)
            self.allreduce_variant = "bytegrad_pipeline"
            self.append_python_op(lambda _name: quant.bytegrad_allreduce_fallback(self, pg, average), group=group)
            return self
        if n == 1 and eng is None:
            self.allreduce_variant = "none(world=1)"
            return self  # nothing to reduce; the scheduler still orders the bucket (events only)
        # (n == 1 WITH an engine is the self-peer mode, BAGUA_SELF_PEER=1: the same kernels run with this GPU as the only peer)
        if eng is not None and self._slice is not None and self.backend_tensor.dtype in (torch.float32, torch.float16, torch.bfloat16):
            nbytes = self.backend_tensor.numel() * self.backend_tensor.element_size()
            v = "two_shot" if (scattergather and variant == "auto") else variant
            op, chosen = eng.make_allreduce_op(self._slice, self._slice, nbytes, self.backend_tensor.dtype, average, v)
            self.backend_bucket.append_op(op)
            self._ops_keepalive.append(op)
            self.allreduce_variant = chosen
            return self

        hier = pg.hier_engine() if (eng is None and self._slice is not None and pg.nnodes > 1) else None
        flat_t = self.backend_tensor
        if hier is not None and flat_t is not None and flat_t.dtype in (torch.float32, torch.float16, torch.bfloat16) and (flat_t.numel() * flat_t.element_size()) % 16 == 0:
            # several NVSwitch nodes: NVLink reduce-scatter kernel → inter-node all-reduce of my 1/L slice on my rail → NVLink all-gather kernel
            ieng, rail_pg, L, nodes = hier
            C = native()
            es = flat_t.element_size()
            nbytes = flat_t.numel() * es
            vecs = nbytes // 16
            vpr = (vecs + L - 1) // L
            lo, hi = ieng.rank * vpr * 16, min((ieng.rank + 1) * vpr * 16, nbytes)
            shard = flat_t.view(-1)[lo // es: max(lo, hi) // es]
            use_mc = bool(self._slice.has_multicast and ieng.has_multicast)
            cfg = ieng.launch_cfg("multimem" if use_mc else "two_shot", nbytes)
            rs = C.ReduceScatterOp(ieng.comm, self._slice.buf, self._slice.offset, nbytes, dtype_code(flat_t.dtype), (1.0 / (L * nodes)) if average else 1.0,
                                   use_mc, cfg)
            ag = C.AllGatherOp(ieng.comm, self._slice.buf, self._slice.offset, nbytes, dtype_code(flat_t.dtype), use_mc, cfg)

            def inter_node(_name: str):
                if shard.numel():
                    dist.all_reduce(shard, group=rail_pg)

            self.backend_bucket.append_op(rs)
            self.append_python_op(inter_node, group=group)
            self.backend_bucket.append_op(ag)
            self._ops_keepalive += [rs, ag]
            self.allreduce_variant = "hier:rs_" + ("multimem" if use_mc else "peer") + "+rail_allreduce+ag"
            return self

        def fallback(_name: str):
            flat, scatter_back = self._flat_or_gather()
            _torch_allreduce(flat, pg, average, hierarchical)
            if scatter_back is not None:
                scatter_back()

        self.allreduce_variant = "torch.distributed"
        self.append_python_op(fallback, group=group)
        return self

    def append_decentralized_synchronous_op(
        self,
        peer_weight: torch.Tensor,
        hierarchical: bool = True,
        peer_selection_mode: str = "all",
        group=None,
    ):
        """Average the bucket's weights with peers into ``peer_weight`` without touching the weights themselves
        (reference bucket.py:215-263; comm op 3).  Returns a handle with ``copy_back_peer_weight(bucket)``."""
        assert peer_selection_mode in ("all", "shift_one"), f"unsupported peer_selection_mode {peer_selection_mode}"
        pg = self._process_group(group)
        eng = self._engine(group)
        handle = _DecentralizedOpHandle(self, peer_weight)
        pw_slice = getattr(peer_weight, "_bagua_symm_slice", None)
        if eng is not None and self._slice is not None:
            C = native()
            flat = self.backend_tensor
            nbytes = flat.numel() * flat.element_size()
            if peer_selection_mode == "all" and pw_slice is not None:
                op, _ = eng.make_allreduce_op(self._slice, pw_slice, nbytes, flat.dtype, True, "auto")
                self.backend_bucket.append_op(op)
                self._ops_keepalive.append(op)
                return handle
            if peer_selection_mode == "shift_one" and nbytes % 16 == 0:
                op = C.PeerAverageOp(eng.comm, self._slice.buf, self._slice.offset, peer_weight.data_ptr(), nbytes, dtype_code(flat.dtype),
                                     eng.launch_cfg("two_shot", nbytes * pg.size()))
                self.backend_bucket.append_op(op)
                self._ops_keepalive.append(op)
                return handle
        state = {"step": 0}

        def fallback(_name: str):
            flat, _ = self._flat_or_gather()
            n = pg.size()
            c = pg.get_global_communicator()
            with torch.no_grad():
                if peer_selection_mode == "all":
                    peer_weight.view(-1)[: flat.numel()].copy_(flat)
                    dist.all_reduce(peer_weight, group=pg.torch_group)
                    peer_weight.div_(n)
                else:
                    assert n % 2 == 0, f"decentralized shift_one needs an even number of ranks, got {n}"
                    peer = native().PeerAverageOp.shift_one_peer(c.rank(), n, state["step"])
                    send_buf = flat.clone()
                    reqs = [dist.isend(send_buf, c._global(peer), group=pg.torch_group), dist.irecv(peer_weight, c._global(peer), group=pg.torch_group)]
                    for r in reqs:
                        r.wait()
                    peer_weight.add_(flat).div_(2)
            state["step"] += 1

        self.append_python_op(fallback, group=group)
        return handle

    def append_low_precision_decentralized_synchronous_op(
        self,
        weight: torch.Tensor,
        left_peer_weight: torch.Tensor,
        right_peer_weight: torch.Tensor,
        hierarchical: bool = True,
        compression: str = "MinMaxUInt8",
        group=None,
    ) -> "BaguaBucket":
        """Ring exchange of compressed weight differences (reference bucket.py:265-320; comm op 4)."""
        assert compression == "MinMaxUInt8"
        pg = self._process_group(group)
        eng = self._engine(group)
        total = self.numel()
        if eng is not None and self._slice is not None and total % 32 == 0:
            C = native()
            box = eng.alloc(C.LowPrecRingOp.box_bytes(total))
            self._aux_slices.append(box)
            flat = self.backend_tensor
            op = C.LowPrecRingOp(eng.comm, flat.data_ptr(), weight.data_ptr(), left_peer_weight.data_ptr(), right_peer_weight.data_ptr(), total,
                                 dtype_code(flat.dtype), box.buf, box.offset, eng.launch_cfg("two_shot", total * 4))
            self.backend_bucket.append_op(op)
            self._ops_keepalive.append(op)
            return self
        self.append_python_op(
            lambda _name: quant.low_precision_ring_fallback(self, pg, weight, left_peer_weight, right_peer_weight), group=group
        )
        return self

    def append_asynchronous_model_average_op(self, peer_selection_mode: str = "all", group=None):
        """Background model averaging step (reference bucket.py:322-352; comm op 5).  Returns the op object with
        ``lock_weight() / unlock_weight() / abort() / reset()``."""
        from .parallel.async_op import AsyncModelAverageOp, FusedAsyncModelAverageOp

        assert peer_selection_mode == "all", "only peer_selection_mode='all' is supported (as in the reference)"
        pg = self._process_group(group)
        op = FusedAsyncModelAverageOp.create(self, pg)   # one kernel per round over NVSwitch peer memory
        if op is not None:
            self.backend_bucket.append_op(op.native_op)
            self._ops_keepalive.append(op)
        else:
            op = AsyncModelAverageOp(self, pg)             # CPU / multi-node: torch.distributed
            self.backend_bucket.append_python_op(op.run, "async_model_average")
        self._async_op = op
        return op


def _torch_allreduce(flat: torch.Tensor, pg, average: bool, hierarchical: bool):
    """``torch.distributed`` allreduce of a flat tensor; hierarchical = intra reduce → inter allreduce → intra bcast
    (reference communicators/mod.rs:261-348)."""
    n = pg.size()
    if hierarchical and pg.nnodes > 1:
        intra = pg.get_intra_node_communicator()
        inter = pg.get_inter_node_communicator()
        dist.reduce(flat, intra._global(0), group=intra.pg)
        if intra.rank() == 0:
            dist.all_reduce(flat, group=inter.pg)
        dist.broadcast(flat, intra._global(0), group=intra.pg)
    else:
        dist.all_reduce(flat, group=pg.torch_group)
    if average:
        flat.div_(n)
