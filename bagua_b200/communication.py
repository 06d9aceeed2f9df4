"""Process groups, communicators and the blocking collective API.

Capability parity with ``bagua/torch_api/communication.py`` of the reference (init_process_group :446-548,
new_group :206-273, from_torch_group :279-309, the 20 blocking collectives :573-1401, ReduceOp :64-75).

H100-first design:

* one process per GPU; ``torch.distributed`` (NCCL on GPUs, gloo on CPU) is the *plumbing*: rendezvous, object
  exchange, the cold user-facing primitives and the fallback for every op.  The reference is GPU/NCCL only
  (communication.py:540-546, :585); the gloo path lets the whole engine run and be tested without a GPU.
* the *hot* paths (bucket allreduce, ByteGrad, decentralized averaging, MoE dispatch) do not go through this
  file at all: they are sm_90a kernels over NVSwitch symmetric memory owned by :class:`PeerEngine`
  (``bagua_b200/parallel/symm.py``), reached through ``BaguaProcessGroup.peer_engine()``.
* a communicator is (torch ProcessGroup, comm stream); blocking collectives keep the reference's stream
  protocol: current stream → event → comm stream runs the op → host waits for the comm stream.
"""
from __future__ import annotations

import io
import logging
import os
import pickle
import threading
import weakref
from enum import IntEnum
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import env

__all__ = [
    "ReduceOp",
    "BaguaProcessGroup",
    "Communicator",
    "init_process_group",
    "is_initialized",
    "new_group",
    "from_torch_group",
    "send",
    "recv",
    "broadcast",
    "broadcast_coalesced",
    "broadcast_object",
    "reduce",
    "reduce_inplace",
    "allreduce",
    "allreduce_inplace",
    "allreduce_coalesced_inplace",
    "allgather",
    "allgather_inplace",
    "gather",
    "gather_inplace",
    "scatter",
    "scatter_inplace",
    "reduce_scatter",
    "reduce_scatter_inplace",
    "alltoall",
    "alltoall_inplace",
    "alltoall_v",
    "alltoall_v_inplace",
    "barrier",
]

logger = logging.getLogger(__name__)


class ReduceOp(IntEnum):
    """Reduction operations; numbering identical to the reference (communication.py:64-75)."""

    SUM = 0
    PRODUCT = 1
    MIN = 2
    MAX = 3
    BOR = 7
    BAND = 8
    BXOR = 9
    AVG = 10


_TORCH_OP = {
    ReduceOp.SUM: dist.ReduceOp.SUM,
    ReduceOp.PRODUCT: dist.ReduceOp.PRODUCT,
    ReduceOp.MIN: dist.ReduceOp.MIN,
    ReduceOp.MAX: dist.ReduceOp.MAX,
    ReduceOp.BOR: dist.ReduceOp.BOR,
    ReduceOp.BAND: dist.ReduceOp.BAND,
    ReduceOp.BXOR: dist.ReduceOp.BXOR,
}


def _use_cuda() -> bool:
    return torch.cuda.is_available() and os.environ.get("BAGUA_FORCE_CPU", "0") != "1"


def _device_index() -> int:
    return torch.cuda.current_device() if _use_cuda() else -1


# ---------------------------------------------------------------------------------------------------------------
# communicator
# ---------------------------------------------------------------------------------------------------------------
class Communicator:
    """A (torch ProcessGroup, comm stream) pair with the collective methods of the reference's
    ``BaguaSingleCommunicatorPy`` (rust/bagua-core/bagua-core-py/src/lib.rs:43-236)."""

    def __init__(self, pg: Optional[dist.ProcessGroup], ranks: Sequence[int], stream, scope: str = "global", owner=None):
        self.pg = pg
        self.ranks = list(ranks)
        self.cuda_stream = stream
        self.scope = scope
        self._aborted = False
        self._owner = weakref.ref(owner) if owner is not None else None
        self._global_rank = dist.get_rank() if dist.is_initialized() else 0

    # -- identity ------------------------------------------------------------------------------------------
    def rank(self) -> int:
        return self.ranks.index(self._global_rank) if self._global_rank in self.ranks else -1

    def nranks(self) -> int:
        return len(self.ranks)

    def device_id(self) -> int:
        return _device_index()

    def abort(self):
        """Unblock in-flight peer kernels of this group (ncclCommAbort analogue, reference mod.rs:474-489)."""
        self._aborted = True
        owner = self._owner() if self._owner else None
        if owner is not None and owner._peer_engine is not None:
            owner._peer_engine.comm.abort()
            owner._peer_engine.comm_blocking.abort()   # the blocking API's own communicator spins on its own flags

    def check_abort(self) -> bool:
        return self._aborted

    def _global(self, group_rank: int) -> int:
        return self.ranks[group_rank]

    # -- helpers -------------------------------------------------------------------------------------------
    def _reduce_op(self, op):
        op = ReduceOp(int(op))
        if op == ReduceOp.AVG:
            return None
        return _TORCH_OP[op]

    def _finish_avg(self, tensor: torch.Tensor, op):
        if ReduceOp(int(op)) == ReduceOp.AVG:
            # AVG divides by the communicator size, not the world size (SURVEY Appendix C)
            if tensor.is_floating_point():
                tensor.div_(self.nranks())
            else:
                tensor.copy_(torch.div(tensor, self.nranks(), rounding_mode="floor"))

    # -- collectives (all in group-rank space like the reference) --------------------------------------------
    def send(self, tensor, dst: int):
        dist.send(tensor, self._global(dst), group=self.pg)

    def recv(self, tensor, src: int):
        dist.recv(tensor, self._global(src), group=self.pg)

    def broadcast(self, tensor, src: int = 0):
        dist.broadcast(tensor, self._global(src), group=self.pg)

    def reduce(self, send_tensor, recv_tensor, dst: int, op=ReduceOp.SUM):
        buf = send_tensor.clone()
        self.reduce_inplace(buf, dst, op)
        if self.rank() == dst:
            recv_tensor.copy_(buf)

    def reduce_inplace(self, tensor, dst: int, op=ReduceOp.SUM):
        top = self._reduce_op(op)
        dist.reduce(tensor, self._global(dst), op=top if top is not None else dist.ReduceOp.SUM, group=self.pg)
        if self.rank() == dst:
            self._finish_avg(tensor, op)

    def allreduce(self, send_tensor, recv_tensor, op=ReduceOp.SUM):
        if recv_tensor.data_ptr() != send_tensor.data_ptr():
            recv_tensor.copy_(send_tensor)
        self.allreduce_inplace(recv_tensor, op)

    def allreduce_inplace(self, tensor, op=ReduceOp.SUM):
        top = self._reduce_op(op)
        dist.all_reduce(tensor, op=top if top is not None else dist.ReduceOp.SUM, group=self.pg)
        self._finish_avg(tensor, op)

    def allgather(self, send_tensor, recv_tensor):
        n = self.nranks()
        assert recv_tensor.numel() == send_tensor.numel() * n, "allgather: recv must hold nranks * send elements"
        try:
            dist.all_gather_into_tensor(recv_tensor.view(-1), send_tensor.contiguous().view(-1), group=self.pg)
        except (RuntimeError, NotImplementedError):  # backends without the flat variant
            _allgather_list(self, send_tensor, recv_tensor)

    def allgather_inplace(self, tensor):
        n = self.nranks()
        assert tensor.numel() % n == 0, "allgather_inplace: tensor size must be divisible by nranks"
        chunk = tensor.view(-1).chunk(n)[self.rank()].clone()
        self.allgather(chunk, tensor)

    def gather(self, send_tensor, recv_tensor, dst: int):
        n = self.nranks()
        if self.rank() == dst:
            outs = list(recv_tensor.view(-1).chunk(n))
            tmp = [torch.empty_like(send_tensor.view(-1)) for _ in range(n)]
            dist.gather(send_tensor.contiguous().view(-1), tmp, dst=self._global(dst), group=self.pg)
            for o, t in zip(outs, tmp):
                o.copy_(t)
        else:
            dist.gather(send_tensor.contiguous().view(-1), None, dst=self._global(dst), group=self.pg)

    def gather_inplace(self, tensor, count: int, dst: int):
        chunk = tensor.view(-1)[self.rank() * count : (self.rank() + 1) * count].clone() if self.rank() == dst else tensor.view(-1)[:count].clone()
        if self.rank() == dst:
            self.gather(chunk, tensor.view(-1)[: count * self.nranks()], dst)
        else:
            self.gather(chunk, tensor, dst)

    def scatter(self, send_tensor, recv_tensor, src: int):
        n = self.nranks()
        if self.rank() == src:
            ins = [c.contiguous() for c in send_tensor.view(-1).chunk(n)]
            dist.scatter(recv_tensor.view(-1), ins, src=self._global(src), group=self.pg)
        else:
            dist.scatter(recv_tensor.view(-1), None, src=self._global(src), group=self.pg)

    def scatter_inplace(self, tensor, count: int, src: int):
        out = torch.empty(count, dtype=tensor.dtype, device=tensor.device)
        self.scatter(tensor.view(-1)[: count * self.nranks()] if self.rank() == src else tensor, out, src)
        tensor.view(-1)[:count].copy_(out)

    def reduce_scatter(self, send_tensor, recv_tensor, op=ReduceOp.SUM):
        n = self.nranks()
        assert send_tensor.numel() == recv_tensor.numel() * n, "reduce_scatter: send must hold nranks * recv elements"
        top = self._reduce_op(op)
        top = top if top is not None else dist.ReduceOp.SUM
        try:
            dist.reduce_scatter_tensor(recv_tensor.view(-1), send_tensor.contiguous().view(-1), op=top, group=self.pg)
        except (RuntimeError, NotImplementedError):
            # gloo has no reduce_scatter: allreduce a copy and keep the own slice
            buf = send_tensor.clone().view(-1)
            dist.all_reduce(buf, op=top, group=self.pg)
            recv_tensor.view(-1).copy_(buf.chunk(n)[self.rank()])
        self._finish_avg(recv_tensor, op)

    def reduce_scatter_inplace(self, tensor, op=ReduceOp.SUM):
        n = self.nranks()
        out = torch.empty(tensor.numel() // n, dtype=tensor.dtype, device=tensor.device)
        self.reduce_scatter(tensor, out, op)
        tensor.view(-1)[: out.numel()].copy_(out)

    def alltoall(self, send_tensor, recv_tensor):
        try:
            dist.all_to_all_single(recv_tensor.view(-1), send_tensor.contiguous().view(-1), group=self.pg)
        except (RuntimeError, NotImplementedError):
            _alltoall_p2p(self, send_tensor, recv_tensor)

    def alltoall_inplace(self, tensor):
        self.alltoall(tensor.clone(), tensor)

    def alltoall_v(self, send_tensor, send_counts, send_displs, recv_tensor, recv_counts, recv_displs):
        n = self.nranks()
        sends = [send_tensor.view(-1)[send_displs[i] : send_displs[i] + send_counts[i]].contiguous() for i in range(n)]
        recvs = [torch.empty(recv_counts[i], dtype=recv_tensor.dtype, device=recv_tensor.device) for i in range(n)]
        try:
            dist.all_to_all(recvs, sends, group=self.pg)
        except (RuntimeError, NotImplementedError):
            _alltoall_list_p2p(self, sends, recvs)
        flat = recv_tensor.view(-1)
        for i in range(n):
            flat[recv_displs[i] : recv_displs[i] + recv_counts[i]].copy_(recvs[i])

    def alltoall_v_inplace(self, tensor, counts, displs):
        self.alltoall_v(tensor.clone(), counts, displs, tensor, counts, displs)

    def barrier(self):
        # the reference's barrier is a 1-element allreduce (communication.py:1396-1398)
        t = torch.zeros(1, device="cuda" if _use_cuda() else "cpu")
        dist.all_reduce(t, group=self.pg)


def _allgather_list(comm: Communicator, send_tensor, recv_tensor):
    outs = [torch.empty_like(send_tensor.view(-1)) for _ in range(comm.nranks())]
    dist.all_gather(outs, send_tensor.contiguous().view(-1), group=comm.pg)
    for o, c in zip(outs, recv_tensor.view(-1).chunk(comm.nranks())):
        c.copy_(o)


def _alltoall_list_p2p(comm: Communicator, sends: List[torch.Tensor], recvs: List[torch.Tensor]):
    me = comm.rank()
    recvs[me].copy_(sends[me])
    reqs = []
    for p in range(comm.nranks()):
        if p == me:
            continue
        reqs.append(dist.isend(sends[p], comm._global(p), group=comm.pg))
        reqs.append(dist.irecv(recvs[p], comm._global(p), group=comm.pg))
    for r in reqs:
        r.wait()


def _alltoall_p2p(comm: Communicator, send_tensor, recv_tensor):
    n = comm.nranks()
    sends = [c.contiguous() for c in send_tensor.view(-1).chunk(n)]
    recvs = [torch.empty_like(s) for s in sends]
    _alltoall_list_p2p(comm, sends, recvs)
    for c, r in zip(recv_tensor.view(-1).chunk(n), recvs):
        c.copy_(r)


# ---------------------------------------------------------------------------------------------------------------
# process groups
# ---------------------------------------------------------------------------------------------------------------
class BaguaProcessGroup:
    """A set of ranks + the comm stream their collectives run on (reference communication.py:108-148).

    Communicators are created lazily: ``global`` (all ranks of the group), ``intra`` (ranks of the group on this
    node) and ``inter`` (ranks of the group with this process's local rank, one per node)."""

    def __init__(self, ranks: Sequence[int], stream, group_name: str, torch_pg: Optional[dist.ProcessGroup] = None):
        self.ranks = list(ranks)
        self.stream = stream
        self.group_name = group_name
        self._torch_pg = torch_pg
        self._comms: Dict[str, Communicator] = {}
        self._peer_engine = None
        self._peer_engine_failed = False
        self._lock = threading.Lock()
        mapping = _get_rank_mappings()
        node_of = {r: mapping[r][0] for r in self.ranks if r in mapping}
        local_of = {r: mapping[r][1] for r in self.ranks if r in mapping}
        me = dist.get_rank() if dist.is_initialized() else 0
        self.intra_ranks = [r for r in self.ranks if node_of.get(r) == node_of.get(me, env.get_node_rank())] or [me]
        # "rail" peers: the group members holding the same position inside their node (== same local rank when the group
        # takes the same local ranks on every node; still connects the nodes when it does not)
        by_node: Dict[object, List[int]] = {}
        for r in self.ranks:
            by_node.setdefault(node_of.get(r), []).append(r)
        pos = {r: sorted(members).index(r) for members in by_node.values() for r in members}
        self.inter_ranks = [r for r in self.ranks if pos.get(r) == pos.get(me, 0)] if me in pos else [me]
        self.nnodes = len(set(node_of.values())) if node_of else 1
        self._node_sizes = sorted(len(m) for m in by_node.values())
        self._local_of = local_of
        self._hier = None
        self._hier_failed = False
        _named_groups[group_name] = self

    # torch ProcessGroup accessors ----------------------------------------------------------------------------
    def _pg_for(self, scope: str) -> Optional[dist.ProcessGroup]:
        if scope == "global":
            return self._torch_pg
        ranks = self.intra_ranks if scope == "intra" else self.inter_ranks
        if ranks == self.ranks:
            return self._torch_pg
        key = (scope, tuple(ranks))
        pg = _subgroup_cache.get(key)
        if pg is None:
            pg = dist.new_group(ranks=ranks, use_local_synchronization=True)
            _subgroup_cache[key] = pg
        return pg

    def _get(self, scope: str) -> Communicator:
        with self._lock:
            c = self._comms.get(scope)
            if c is None:
                ranks = {"global": self.ranks, "intra": self.intra_ranks, "inter": self.inter_ranks}[scope]
                c = Communicator(self._pg_for(scope), ranks, self.stream, scope, owner=self)
                self._comms[scope] = c
            return c

    def get_global_communicator(self) -> Communicator:
        return self._get("global")

    def get_inter_node_communicator(self) -> Communicator:
        return self._get("inter")

    def get_intra_node_communicator(self) -> Communicator:
        return self._get("intra")

    @property
    def torch_group(self) -> Optional[dist.ProcessGroup]:
        return self._torch_pg

    def rank(self) -> int:
        return self.get_global_communicator().rank()

    def size(self) -> int:
        return len(self.ranks)

    # NVSwitch symmetric-memory engine ---------------------------------------------------------------------------
    def peer_engine(self):
        """The :class:`~bagua_b200.parallel.symm.PeerEngine` of this group, or ``None`` when the group cannot use
        peer kernels (CPU, multi-node, > 8 ranks, BAGUA_ALLREDUCE_VARIANT=nccl, or symmetric memory unavailable)."""
        if self._peer_engine is not None or self._peer_engine_failed:
            return self._peer_engine
        from .parallel import symm

        with self._lock:
            if self._peer_engine is None and not self._peer_engine_failed:
                try:
                    self._peer_engine = symm.PeerEngine.create(self)
                except Exception as e:  # noqa: BLE001
                    logger.warning("bagua_b200: peer (NVSwitch) engine unavailable for group %s: %s", self.group_name, e)
                    self._peer_engine = None
                if self._peer_engine is None:
                    self._peer_engine_failed = True
        return self._peer_engine


def _hier_engine(self):
    """Multi-node counterpart of :meth:`peer_engine`: ``(intra-node PeerEngine, rail torch group, ranks per node, nodes)`` for
    a CUDA group that spans several NVSwitch nodes with the same number (2…8) of ranks on each; ``None`` otherwise.
    Collective over the group on first use.  The hierarchical all-reduce built on it: reduce-scatter kernel inside the node →
    all-reduce of this rank's 1/L slice with its rail peers (NCCL; every NIC rail carries 1/L of the bucket) → all-gather kernel."""
    if self._hier is not None or self._hier_failed:
        return self._hier
    from .core import native

    with self._lock:
        if self._hier is None and not self._hier_failed:
            try:
                ok = (_use_cuda() and env.get_allreduce_variant() != "nccl" and self.nnodes > 1 and len(set(self._node_sizes)) == 1
                      and 2 <= self._node_sizes[0] <= native().MAX_PEERS and dist.get_rank() in self.ranks)
                if ok:
                    intra_pg = BaguaProcessGroup(self.intra_ranks, self.stream, self.group_name + ".intra", self._pg_for("intra"))
                    eng = intra_pg.peer_engine()
                    rail = self._pg_for("inter")
                    if eng is not None:
                        self._hier = (eng, rail, self._node_sizes[0], self.nnodes)
                        self._hier_intra_pg = intra_pg
            except Exception as e:  # noqa: BLE001
                logger.warning("bagua_b200: hierarchical peer engine unavailable for group %s: %s", self.group_name, e)
            if self._hier is None:
                self._hier_failed = True
    return self._hier


BaguaProcessGroup.hier_engine = _hier_engine
_subgroup_cache: Dict[tuple, dist.ProcessGroup] = {}
_default_pg: Optional[BaguaProcessGroup] = None
_group_count = 0
_rank_mappings: Optional[Dict[int, tuple]] = None
_pg_map: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()
_autotune_server = None
_autotune_service_port = None
_backends: Dict[str, object] = {}
_named_groups: "weakref.WeakValueDictionary" = weakref.WeakValueDictionary()


def _get_rank_mappings() -> Dict[int, tuple]:
    """global rank → (node_rank, local_rank), gathered once (reference communication.py:151-163)."""
    global _rank_mappings
    if _rank_mappings is not None:
        return _rank_mappings
    if not dist.is_initialized() or dist.get_world_size() == 1:
        _rank_mappings = {0: (env.get_node_rank(), env.get_local_rank())}
        return _rank_mappings
    objs: List[object] = [None] * dist.get_world_size()
    dist.all_gather_object(objs, (env.get_node_rank(), env.get_local_rank()))
    _rank_mappings = {r: tuple(o) for r, o in enumerate(objs)}
    return _rank_mappings


def is_initialized() -> bool:
    """Whether :func:`init_process_group` has been called."""
    return _default_pg is not None


def _get_default_group() -> BaguaProcessGroup:
    if _default_pg is None:
        raise RuntimeError("Default process group has not been initialized, please make sure to call init_process_group.")
    return _default_pg


def _rank_not_in_group(group: Optional[BaguaProcessGroup]) -> bool:
    if group is None:
        return False
    return dist.get_rank() not in group.ranks


def _make_stream(priority_high: bool = True):
    if not _use_cuda():
        return None
    return torch.cuda.Stream(priority=-1 if priority_high else 0)


def new_group(ranks: Optional[Sequence[int]] = None, stream=None) -> BaguaProcessGroup:
    """Create a new process group over ``ranks`` (default: all) whose collectives run on ``stream``.

    Must be entered by all processes of the job, in the same order (reference communication.py:206-273)."""
    global _group_count
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialized; call bagua_b200.init_process_group() first")
    world = dist.get_world_size()
    if ranks is None:
        ranks = list(range(world))
    ranks = sorted(int(r) for r in ranks)
    if len(ranks) == 0 or len(ranks) > world or any(r < 0 or r >= world for r in ranks):
        raise ValueError(f"invalid ranks {ranks} for a world of {world}")
    group_name = str(_group_count)
    _group_count += 1
    torch_pg = dist.new_group(ranks=ranks) if len(ranks) != world or _group_count > 1 else dist.group.WORLD
    if stream is None:
        stream = _make_stream()
    pg = BaguaProcessGroup(ranks, stream, group_name, torch_pg)
    return pg


def from_torch_group(group: dist.ProcessGroup, stream=None) -> BaguaProcessGroup:
    """Wrap an existing ``torch.distributed`` group (reference communication.py:279-309)."""
    global _group_count
    if not isinstance(group, dist.ProcessGroup):  # torch hands non-members the GroupMember.NON_GROUP_MEMBER sentinel
        raise ValueError("from_torch_group: this rank is not a member of the given torch.distributed group")
    cached = _pg_map.get(group)
    if cached is not None and (stream is None or cached.stream is stream):
        return cached
    ranks = sorted(dist.get_process_group_ranks(group))
    group_name = f"torch{_group_count}"
    _group_count += 1
    pg = BaguaProcessGroup(ranks, stream if stream is not None else _make_stream(), group_name, group)
    try:
        _pg_map[group] = pg
    except TypeError:
        pass
    return pg


class BaguaProcessGroupPatch:
    """Methods grafted onto ``torch.distributed.ProcessGroup`` (reference communication.py:78-105): ``pg.bagua_patch(stream)`` registers
    the torch group with the engine, ``pg.bagua_pg`` is its :class:`BaguaProcessGroup`, ``pg.bagua_get_*_communicator()`` its
    communicators.  The cache is weakly keyed on the torch group."""

    def bagua_patch(self, stream=None):
        from_torch_group(self, stream)
        return self

    @property
    def bagua_pg(self):
        return from_torch_group(self)

    def bagua_get_global_communicator(self):
        return from_torch_group(self).get_global_communicator()

    def bagua_get_inter_node_communicator(self):
        return from_torch_group(self).get_inter_node_communicator()

    def bagua_get_intra_node_communicator(self):
        return from_torch_group(self).get_intra_node_communicator()


def _patch_torch_process_group():
    """Install :class:`BaguaProcessGroupPatch` on ``torch.distributed.ProcessGroup``."""
    for name in ("bagua_patch", "bagua_pg", "bagua_get_global_communicator", "bagua_get_inter_node_communicator", "bagua_get_intra_node_communicator"):
        setattr(dist.ProcessGroup, name, BaguaProcessGroupPatch.__dict__[name])


def broadcast_nccl_unique_id(comm_key: str, root: int) -> str:
    """Publish a fresh NCCL unique id (base64 text) from ``root`` under ``comm_key`` in the default group's c10d store and return it on
    every rank (reference communication.py:551-560).  The engine itself never needs one — torch.distributed creates the NCCL
    communicators here — but code that brings its own ``ncclCommInitRank`` can keep using the helper."""
    from torch.distributed.distributed_c10d import _get_default_store

    store = _get_default_store()
    if dist.get_rank() == root:
        from bagua_core import BaguaSingleCommunicatorPy

        idstr = BaguaSingleCommunicatorPy.generate_nccl_unique_id_str()
        store.set(comm_key, idstr)
        return idstr
    return store.get(comm_key).decode("utf-8")


def get_backend(model_name: str):
    """One native scheduler (worker thread + ordered bucket list) per module name
    (reference communication.py:377-381), so several models can train in one process."""
    from .core import native

    be = _backends.get(model_name)
    if be is None:
        pg = _get_default_group()
        dev = _device_index()
        stream = pg.stream.cuda_stream if (dev >= 0 and pg.stream is not None) else 0
        be = native().Backend(100, dev, stream, env.get_comm_timeout_s())
        _backends[model_name] = be
    return be


def _shutdown_backends():
    for be in list(_backends.values()):
        try:
            be.shutdown()
        except Exception:  # noqa: BLE001
            pass
    _backends.clear()


def get_autotune_service_port() -> Optional[int]:
    return _autotune_service_port


_autotune_service_host: List[Optional[str]] = [None]


def get_autotune_service_host() -> str:
    """Host under which this process reaches the autotune service (decided by the health check in ``init_process_group``)."""
    return _autotune_service_host[0] or env.get_master_addr()


def _start_autotune_server(world_size: int):
    """Rank 0 hosts the autotune HTTP service in a daemon process (reference communication.py:384-443)."""
    global _autotune_server, _autotune_service_port
    from .service.autotune_service import start_autotune_server_process

    store = dist.distributed_c10d._get_default_store()
    if dist.get_rank() == 0:
        port = env.get_bagua_service_port()
        if port <= 0:
            port = env.find_free_network_port()
        _autotune_server = start_autotune_server_process(port, world_size)
        store.set("bagua_autotune_service_port", str(port))
    _autotune_service_port = int(store.get("bagua_autotune_service_port"))
    from .service.autotune_service import AutotuneClient
    import time

    # Where rank 0 is reachable: MASTER_ADDR normally — but the elastic launcher exports the node's *hostname* there, which
    # need not resolve inside a container; processes of rank 0's own node then reach the service through loopback.
    hosts = [env.get_master_addr()]
    if env.get_node_rank() == 0 and "127.0.0.1" not in hosts:
        hosts.append("127.0.0.1")
    deadline = time.time() + max(30, env.get_autotune_server_wait_time())
    while time.time() < deadline:
        for h in hosts:
            if AutotuneClient(h, _autotune_service_port, timeout=2.0).health_check():
                _autotune_service_host[0] = h
                os.environ["AUTO_TUNE_SERVER_ADDR"] = f"{h}:{_autotune_service_port}"
                return
        time.sleep(0.2)
    raise RuntimeError(f"autotune service did not come up in time (tried {hosts}, port {_autotune_service_port})")


def start_autotune_server(service_port: int = -1):
    """Start the autotune service on this process (reference communication.py:384-412; rank 0 calls it from
    :func:`init_process_group` when ``BAGUA_AUTOTUNE > 0``).  Returns the server process."""
    from .service.autotune_service import start_autotune_server_process

    port = service_port if service_port and service_port > 0 else env.find_free_network_port()
    return start_autotune_server_process(port, dist.get_world_size() if dist.is_initialized() else env.get_world_size())


def get_hyperparameters_service_client():
    """REST client of the running autotune service (reference communication.py:355-361)."""
    from .service.autotune_service import AutotuneClient

    port = _autotune_service_port if _autotune_service_port else env.get_bagua_service_port()
    return AutotuneClient(get_autotune_service_host(), port)


class comm(object):
    """``comm.WORLD``: "the default group's global communicator" (reference communication.py:563-565; ``None`` here, which every
    collective already treats that way)."""

    WORLD = None


class CommMember(object):
    """Sentinels of the reference API (communication.py:567-570)."""

    WORLD = comm.WORLD  # "use the default group's global communicator"
    NON_COMM_MEMBER = object()


def get_communicator(group_name: str, comm_name: str):
    """The ``global`` / ``inter`` / ``intra`` communicator of a named group, or ``CommMember.NON_COMM_MEMBER`` when this rank
    is not part of it (reference communication.py:313-352)."""
    pg = _named_groups.get(group_name)
    if pg is None:
        raise KeyError(f"unknown process group {group_name!r}")
    if comm_name not in ("global", "inter", "intra"):
        raise ValueError("comm_name should be one of ['global', 'inter', 'intra']")
    ranks = {"global": pg.ranks, "inter": pg.inter_ranks, "intra": pg.intra_ranks}[comm_name]
    if dist.get_rank() not in ranks:
        return CommMember.NON_COMM_MEMBER
    return pg._get(comm_name)


def init_process_group(store=None, rank: int = -1, world_size: int = -1, local_world_size: int = -1):
    """Initialise the default process group (reference communication.py:446-548).

    ``store is None`` → ``env://`` rendezvous (``MASTER_ADDR``/``MASTER_PORT``/``RANK``/``WORLD_SIZE``); otherwise the
    given c10d store with explicit ``rank``/``world_size``/``local_world_size``.  Backend is NCCL when a GPU is
    visible and gloo otherwise."""
    global _default_pg, _rank_mappings
    if _default_pg is not None:
        raise RuntimeError("trying to initialize the default process group twice!")
    if store is not None:
        assert rank >= 0 and world_size > 0 and local_world_size > 0, "rank, world_size and local_world_size are required with a store"
        os.environ["RANK"] = str(rank)
        os.environ["WORLD_SIZE"] = str(world_size)
        os.environ["LOCAL_WORLD_SIZE"] = str(local_world_size)
        os.environ.setdefault("LOCAL_RANK", str(rank % local_world_size))
    backend = "nccl" if _use_cuda() else "gloo"
    if not dist.is_initialized():
        kwargs = {}
        if backend == "nccl":
            kwargs["device_id"] = torch.device("cuda", torch.cuda.current_device())
        if store is not None:
            dist.init_process_group(backend=backend, store=store, rank=rank, world_size=world_size, **kwargs)
        else:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29500")
            # rank / world size come from the environment: passing them explicitly makes torch rewrite the env:// URL, which
            # breaks re-rendezvous of restarted gangs under the elastic launcher (stale store keys → connect refused).
            # A bare single-process run (no launcher) has neither variable: it is rank 0 of 1.
            os.environ.setdefault("RANK", str(env.get_rank()))
            os.environ.setdefault("WORLD_SIZE", str(env.get_world_size()))
            if os.environ.get("TORCHELASTIC_USE_AGENT_STORE", "") == "True" and int(os.environ.get("TORCHELASTIC_RESTART_COUNT", "0") or 0) > 0:
                # Elastic launcher: every attempt of the gang talks to the SAME agent-hosted TCPStore (MASTER_PORT does not change across
                # restarts), and torch's env:// handler adds no per-attempt prefix — a restarted rank then reads its peer's address of
                # the PREVIOUS attempt ("Gloo connectFullMesh failed … Connection refused", about every second restart on loopback).
                # The keys of every RESTARTED attempt are isolated here (attempt 0 finds a fresh store and takes the stock env:// path).
                from datetime import timedelta

                attempt = os.environ.get("TORCHELASTIC_RESTART_COUNT", "0")
                tcp = dist.TCPStore(env.get_master_addr(), env.get_master_port(), env.get_world_size(), False, timedelta(seconds=env.get_comm_timeout_s() + 600))
                dist.init_process_group(backend=backend, store=dist.PrefixStore(f"/bagua_b200/attempt_{attempt}", tcp), rank=env.get_rank(),
                                        world_size=env.get_world_size(), **kwargs)
            else:
                dist.init_process_group(backend=backend, **kwargs)
    _rank_mappings = None
    _patch_torch_process_group()
    _default_pg = new_group(stream=_make_stream())
    if env.get_autotune_level() > 0:
        _start_autotune_server(dist.get_world_size())
    import atexit

    atexit.register(_shutdown_backends)
    return _default_pg


def _reset_for_tests():
    """Tear down module state (used by the test-suite between in-process scenarios)."""
    global _default_pg, _group_count, _rank_mappings
    _shutdown_backends()
    _default_pg = None
    _group_count = 0
    _rank_mappings = None
    _subgroup_cache.clear()


# ---------------------------------------------------------------------------------------------------------------
# blocking collective API (module level, reference communication.py:573-1401)
# ---------------------------------------------------------------------------------------------------------------
def _comm(comm: Optional[Communicator]) -> Communicator:
    return comm if comm is not None else _get_default_group().get_global_communicator()


def _check(comm: Communicator, *tensors):
    if _use_cuda():
        for t in tensors:
            assert t.device.type == "cuda", "input tensors must be CUDA tensors when a GPU backend is active"


class _on_comm_stream:
    """current stream → event → comm stream runs the body → host waits for the comm stream."""

    def __init__(self, comm: Communicator):
        self.comm = comm
        self.ctx = None

    def __enter__(self):
        s = self.comm.cuda_stream
        if s is not None and _use_cuda():
            ev = torch.cuda.current_stream().record_event()
            s.wait_event(ev)
            self.ctx = torch.cuda.stream(s)
            self.ctx.__enter__()
        return self

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)
            self.comm.cuda_stream.synchronize()
        return False


def send(tensor: torch.Tensor, dst: int, comm: Optional[Communicator] = None):
    """Send ``tensor`` to group-rank ``dst`` (blocking)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.send(tensor, dst)


def recv(tensor: torch.Tensor, src: int, comm: Optional[Communicator] = None):
    """Receive into ``tensor`` from group-rank ``src`` (blocking)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.recv(tensor, src)


def broadcast(tensor: torch.Tensor, src: int = 0, comm: Optional[Communicator] = None):
    """Broadcast ``tensor`` from group-rank ``src`` to every rank of the communicator."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.broadcast(tensor, src)


def broadcast_coalesced(tensors: Sequence[torch.Tensor], src: int = 0, comm: Optional[Communicator] = None):
    """Broadcast a list of tensors as one flat message per dtype."""
    c = _comm(comm)
    _check(c, *tensors)
    with _on_comm_stream(c):
        by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
        for t in tensors:
            by_dtype.setdefault(t.dtype, []).append(t)
        for group in by_dtype.values():
            flat = torch.cat([t.reshape(-1) for t in group])
            c.broadcast(flat, src)
            off = 0
            for t in group:
                t.copy_(flat[off : off + t.numel()].view_as(t))
                off += t.numel()


def broadcast_object(obj: object, src: int = 0, comm: Optional[Communicator] = None) -> object:
    """Broadcast a picklable python object; returns it on every rank (reference communication.py:668-708)."""
    c = _comm(comm)
    dev = "cuda" if _use_cuda() else "cpu"
    if c.rank() == src:
        buf = io.BytesIO()
        pickle.dump(obj, buf)
        data = bytearray(buf.getvalue())
        length = torch.tensor([len(data)], dtype=torch.int64, device=dev)
        payload = torch.tensor(list(data), dtype=torch.uint8, device=dev) if len(data) else torch.empty(0, dtype=torch.uint8, device=dev)
        broadcast(length, src, c)
        broadcast(payload, src, c)
        return obj
    length = torch.zeros(1, dtype=torch.int64, device=dev)
    broadcast(length, src, c)
    payload = torch.empty(int(length.item()), dtype=torch.uint8, device=dev)
    broadcast(payload, src, c)
    return pickle.loads(bytes(payload.cpu().tolist()))


def reduce(send_tensor, recv_tensor, dst: int, op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """Reduce ``send_tensor`` across ranks into ``recv_tensor`` on group-rank ``dst``."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    with _on_comm_stream(c):
        c.reduce(send_tensor, recv_tensor, dst, op)


def reduce_inplace(tensor, dst: int, op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """In-place :func:`reduce`: ``tensor`` on ``dst`` becomes the reduction over all ranks (reference communication.py:792-813)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.reduce_inplace(tensor, dst, op)


def _peer_allreduce_eligible(c: Communicator, tensor: torch.Tensor, op):
    if not _use_cuda() or ReduceOp(int(op)) not in (ReduceOp.SUM, ReduceOp.AVG):
        return None
    if tensor.dtype not in (torch.float32, torch.float16, torch.bfloat16) or not tensor.is_contiguous():
        return None
    owner = c._owner() if c._owner else None
    if owner is None or c.scope != "global":
        return None
    return owner.peer_engine()


def _peer_allreduce(c: Communicator, tensor: torch.Tensor, op) -> bool:
    """Route eligible allreduces through the NVSwitch kernels; returns False when NCCL/gloo must do it.  Called from the
    caller's own stream (NOT under ``_on_comm_stream``): the engine orders the kernel after it on its blocking stream."""
    eng = _peer_allreduce_eligible(c, tensor, op)
    if eng is None:
        return False
    return eng.allreduce_tensor(tensor, average=ReduceOp(int(op)) == ReduceOp.AVG)


def allreduce(send_tensor, recv_tensor, op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """All-reduce ``send_tensor`` into ``recv_tensor`` (same shape) on every rank."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    assert send_tensor.numel() == recv_tensor.numel(), "send and recv tensors must have the same size"
    if _peer_allreduce_eligible(c, recv_tensor, op):
        # peer kernels: own communicator, own stream, ordered after the caller's stream (PeerEngine.blocking_region)
        if recv_tensor.data_ptr() != send_tensor.data_ptr():
            recv_tensor.copy_(send_tensor)
        if _peer_allreduce(c, recv_tensor, op):
            return
    with _on_comm_stream(c):
        if recv_tensor.data_ptr() != send_tensor.data_ptr():
            recv_tensor.copy_(send_tensor)
        c.allreduce_inplace(recv_tensor, op)


def allreduce_inplace(tensor, op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """In-place all-reduce of ``tensor`` over the communicator (``AVG`` divides by its size); CUDA tensors on one NVSwitch node
    take the peer kernels (reference communication.py:922-943)."""
    c = _comm(comm)
    _check(c, tensor)
    if _peer_allreduce(c, tensor, op):
        return
    with _on_comm_stream(c):
        c.allreduce_inplace(tensor, op)


def allreduce_coalesced_inplace(tensors: Sequence[torch.Tensor], op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """All-reduce a list of tensors as flat messages (one per dtype)."""
    c = _comm(comm)
    _check(c, *tensors)
    by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
    for t in tensors:
        by_dtype.setdefault(t.dtype, []).append(t)
    for group in by_dtype.values():
        flat = torch.cat([t.reshape(-1) for t in group])
        if not _peer_allreduce(c, flat, op):
            with _on_comm_stream(c):
                c.allreduce_inplace(flat, op)
        off = 0
        for t in group:
            t.copy_(flat[off : off + t.numel()].view_as(t))
            off += t.numel()


def _peer_engine_for(c: Communicator):
    """The NVSwitch engine behind a global communicator when the opt-in peer collectives are enabled
    (``BAGUA_PEER_COLLECTIVES=1``: all-gather / reduce-scatter through the peer kernels instead of NCCL)."""
    if not _use_cuda() or os.environ.get("BAGUA_PEER_COLLECTIVES", "0") != "1":
        return None
    owner = c._owner() if c._owner else None
    if owner is None or c.scope != "global":
        return None
    return owner.peer_engine()


def allgather(send_tensor, recv_tensor, comm: Optional[Communicator] = None):
    """``recv_tensor`` (``nranks × send_tensor.numel()``) = concatenation of every rank's ``send_tensor`` in rank order (reference communication.py:946-982)."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    eng = _peer_engine_for(c)
    if eng is not None and eng.allgather_tensor(send_tensor, recv_tensor):
        return
    with _on_comm_stream(c):
        c.allgather(send_tensor, recv_tensor)


def allgather_inplace(tensor, comm: Optional[Communicator] = None):
    """All-gather inside one buffer: chunk ``rank`` of ``tensor`` is this rank's contribution, all chunks are filled on return (reference communication.py:985-1005)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.allgather_inplace(tensor)


def gather(send_tensor, recv_tensor, dst: int, comm: Optional[Communicator] = None):
    """``recv_tensor`` on ``dst`` = concatenation of every rank's ``send_tensor``; untouched elsewhere (reference communication.py:1008-1046)."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    with _on_comm_stream(c):
        c.gather(send_tensor, recv_tensor, dst)


def gather_inplace(tensor, count: int, dst: int, comm: Optional[Communicator] = None):
    """In-place gather: the first ``count`` elements of ``tensor`` are sent; on ``dst`` ``tensor`` holds all ranks' pieces
    afterwards (reference communication.py:1049-1081)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.gather_inplace(tensor, count, dst)


def scatter(send_tensor, recv_tensor, src: int, comm: Optional[Communicator] = None):
    """Rank ``src`` splits ``send_tensor`` into ``nranks`` equal chunks; every rank receives its chunk in ``recv_tensor`` (reference communication.py:1084-1123)."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    with _on_comm_stream(c):
        c.scatter(send_tensor, recv_tensor, src)


def scatter_inplace(tensor, count: int, src: int, comm: Optional[Communicator] = None):
    """In-place scatter: chunk ``rank`` (``count`` elements) of ``src``'s ``tensor`` lands in the first ``count`` elements of
    ``tensor`` (reference communication.py:1126-1160)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.scatter_inplace(tensor, count, src)


def reduce_scatter(send_tensor, recv_tensor, op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """Reduce ``send_tensor`` over all ranks and leave chunk ``rank`` of the result in ``recv_tensor`` (reference communication.py:1163-1202)."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    eng = _peer_engine_for(c) if ReduceOp(int(op)) in (ReduceOp.SUM, ReduceOp.AVG) else None
    if eng is not None and eng.reduce_scatter_tensor(send_tensor, recv_tensor, ReduceOp(int(op)) == ReduceOp.AVG):
        return
    with _on_comm_stream(c):
        c.reduce_scatter(send_tensor, recv_tensor, op)


def reduce_scatter_inplace(tensor, op: ReduceOp = ReduceOp.SUM, comm: Optional[Communicator] = None):
    """In-place reduce-scatter: the FIRST ``numel / nranks`` elements of ``tensor`` hold this rank's chunk of the reduction
    afterwards (MPI_IN_PLACE placement, which is what the reference's Aluminum call does — rust/…/communicators/mod.rs:1026-1058 —
    not NCCL's chunk-``rank`` placement; reference communication.py:1205-1235)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.reduce_scatter_inplace(tensor, op)


def alltoall(send_tensor, recv_tensor, comm: Optional[Communicator] = None):
    """Chunk ``j`` of ``send_tensor`` goes to rank ``j``; chunk ``i`` of ``recv_tensor`` comes from rank ``i`` (equal chunks; reference communication.py:1238-1276)."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    with _on_comm_stream(c):
        c.alltoall(send_tensor, recv_tensor)


def alltoall_inplace(tensor, comm: Optional[Communicator] = None):
    """In-place :func:`alltoall` (reference communication.py:1279-1298)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.alltoall_inplace(tensor)


def alltoall_v(send_tensor, send_counts, send_displs, recv_tensor, recv_counts, recv_displs, comm: Optional[Communicator] = None):
    """All-to-all with per-peer element counts and displacements, MPI_Alltoallv style (reference communication.py:1301-1350)."""
    c = _comm(comm)
    _check(c, send_tensor, recv_tensor)
    with _on_comm_stream(c):
        c.alltoall_v(send_tensor, send_counts, send_displs, recv_tensor, recv_counts, recv_displs)


def alltoall_v_inplace(tensor, counts, displs, comm: Optional[Communicator] = None):
    """In-place :func:`alltoall_v` with identical send and receive layout (reference communication.py:1353-1374)."""
    c = _comm(comm)
    _check(c, tensor)
    with _on_comm_stream(c):
        c.alltoall_v_inplace(tensor, counts, displs)


def barrier(comm: Optional[Communicator] = None):
    """Block until every rank of the communicator has entered the barrier."""
    c = _comm(comm)
    with _on_comm_stream(c):
        c.barrier()
