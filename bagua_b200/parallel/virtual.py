"""Virtual peer worlds: run the NVSwitch peer kernels of P ranks on ONE GPU inside one process.

The fused collective kernels (``csrc/peer_kernels.cu``, ``csrc/bytegrad_kernels.cu``, ``csrc/moe_kernels.cu``) only see
pointers: ``PeerCtx.flags[p]`` (signal pads), ``PeerBuf.ptr[p]`` (one buffer per rank) and their own ``rank``.  Nothing in
them requires the P buffers to live on P different GPUs — so a *virtual world* gives every rank its own signal pad,
buffers and CUDA stream on the same device and launches the P kernels back to back on the P streams.  They become
co-resident (P × grid ≤ what the 132 SMs of an H100 hold), meet at the same epoch barriers and exchange data through the same
loads/stores as over NVLink; only the wires are missing.  That makes every P = 2…8 code path (slice arithmetic, rotation of
the peer order, barrier protocol, parity double-buffering, quantised in/out boxes, MoE row addressing) checkable against
fp32 oracles on a single-GPU box — which is what the CI box has (the reference can only test its collectives with ≥ 2
real GPUs: ``tests/comm/test_communicator.py``).

What it cannot cover: ``multimem`` (NVLS) instructions need a real multicast object — see ``self_multicast_buffer`` for
the world = 1 flavour — and link bandwidth.

Not a production path: ``bagua_doctor --kernels`` and the test-suite / ``smoke()`` use it.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch

from ..core import native

__all__ = ["VirtualPeerWorld", "VirtualBuf"]


class VirtualBuf:
    """One "symmetric" allocation of a virtual world: ``tensors[r]`` is rank r's copy, ``buf`` the native ``SymmBuf``."""

    def __init__(self, tensors: List[torch.Tensor]):
        self.tensors = tensors
        self.nbytes = tensors[0].numel() * tensors[0].element_size()
        self.buf = native().SymmBuf([t.data_ptr() for t in tensors], 0, self.nbytes)
        self.offset = 0

    def view(self, rank: int, dtype: torch.dtype, numel: Optional[int] = None) -> torch.Tensor:
        t = self.tensors[rank].view(dtype)
        return t if numel is None else t[:numel]


class VirtualPeerWorld:
    """``world`` virtual ranks on ``device``: per-rank ``PeerComm`` (own signal pad, epochs, error word) and stream."""

    def __init__(self, world: int, device: Optional[torch.device] = None, timeout_s: float = 20.0):
        C = native()
        assert 1 <= world <= C.MAX_PEERS
        self.world = world
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._pads = [torch.zeros(C.signal_pad_bytes(), dtype=torch.uint8, device=self.device) for _ in range(world)]
        torch.cuda.synchronize(self.device)
        ptrs = [p.data_ptr() for p in self._pads]
        self.comms = [C.PeerComm(r, world, self.device.index, ptrs, timeout_s) for r in range(world)]
        self.streams = [torch.cuda.Stream(device=self.device) for _ in range(world)]
        sm = torch.cuda.get_device_properties(self.device).multi_processor_count
        # every CTA of every rank must be resident at the same time (they spin on each other): 512-thread CTAs with
        # ≤ 64 registers fit two per SM; keep a margin
        self.max_blocks_per_rank = max(1, min(C.MAX_COMM_BLOCKS, (sm * 2 * 3 // 4) // world))

    def alloc(self, nbytes: int, fill: Optional[Callable[[int, torch.Tensor], None]] = None) -> VirtualBuf:
        nbytes = (int(nbytes) + 1023) // 1024 * 1024
        ts = [torch.zeros(nbytes, dtype=torch.uint8, device=self.device) for _ in range(self.world)]
        vb = VirtualBuf(ts)
        if fill is not None:
            for r, t in enumerate(ts):
                fill(r, t)
        return vb

    def cfg(self, blocks: int = 4, threads: int = 512):
        return native().LaunchCfg(int(min(blocks, self.max_blocks_per_rank)), threads)

    def run(self, make_op: Callable[[int], object], repeat: int = 1, ops: Optional[Sequence[object]] = None):
        """Launch rank r's op (``make_op(r)`` — built once — or ``ops[r]``) on rank r's stream, ``repeat`` times, and wait.
        Raises if any rank's kernel reported a barrier time-out / abort."""
        C = native()
        if ops is None:
            ops = [make_op(r) for r in range(self.world)]
        torch.cuda.synchronize(self.device)
        for _ in range(repeat):
            for r, op in enumerate(ops):
                C.run_op(op, self.streams[r].cuda_stream, self.device.index)
        torch.cuda.synchronize(self.device)
        self.check()
        return ops

    def launch_all(self, fn: Callable[[int, int], None]):
        """``fn(rank, stream_ptr)`` enqueues rank's kernel(s) itself (direct kernel entry points such as ``moe_scatter``)."""
        torch.cuda.synchronize(self.device)
        for r in range(self.world):
            fn(r, self.streams[r].cuda_stream)
        torch.cuda.synchronize(self.device)
        self.check()

    def check(self):
        for r, c in enumerate(self.comms):
            code = c.error_code()
            if code:
                raise RuntimeError(f"virtual rank {r}: peer kernel error {code} (1 timeout, 2 abort, 3 grid barrier timeout)")
