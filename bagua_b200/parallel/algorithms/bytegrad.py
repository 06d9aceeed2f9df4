"""ByteGrad: 8-bit MinMaxUInt8-compressed gradient allreduce (reference: bagua/torch_api/algorithms/bytegrad.py:1-82)."""
from __future__ import annotations

from typing import List

import torch

from ...bucket import BaguaBucket
from .base import Algorithm, AlgorithmImpl

__all__ = ["ByteGradAlgorithm", "ByteGradAlgorithmImpl"]


def bytegrad_min_bucket_bytes(tensors) -> int:
    """Lower bound on a ByteGrad bucket on GPUs (``BAGUA_BYTEGRAD_MIN_BUCKET_BYTES``, default 32 MiB; 0 on the host).  Every quantised
    exchange — the fused kernel as well as the 7-step torch.distributed pipeline — has a fixed cost per bucket (four grid-wide and two
    cross-GPU rendezvous in the kernel; 2·P+7 launches and two collectives in the pipeline) that does not shrink with the bucket, while
    NVSwitch moves 10 MiB in microseconds, so fewer, larger buckets pay where the rendezvous cross GPUs."""
    import os

    try:
        first = tensors[0][0].bagua_getter_closure()
        on_gpu = first.is_cuda
    except Exception:  # noqa: BLE001
        on_gpu = False
    return int(os.environ.get("BAGUA_BYTEGRAD_MIN_BUCKET_BYTES", str(32 * 1024 ** 2 if on_gpu else 0)))


def merge_small_buckets(tensors: List[List[torch.Tensor]], min_bytes: int) -> List[List[torch.Tensor]]:
    """Concatenate consecutive suggested buckets (same dtype) until each holds at least ``min_bytes``; order is preserved, so a merged
    bucket becomes ready when its last member would have."""
    if min_bytes <= 0:
        return tensors
    out, cur, size = [], [], 0
    for b in tensors:
        eff = b[0].bagua_getter_closure()
        if cur and cur[0].bagua_getter_closure().dtype != eff.dtype:
            out.append(cur)
            cur, size = [], 0
        cur = cur + list(b)
        size += sum(t.bagua_getter_closure().numel() * t.bagua_getter_closure().element_size() for t in b)
        if size >= min_bytes:
            out.append(cur)
            cur, size = [], 0
    if cur:
        if out and size < min_bytes // 4 and out[-1][0].bagua_getter_closure().dtype == cur[0].bagua_getter_closure().dtype:
            out[-1] = out[-1] + cur      # a small remainder joins its predecessor instead of paying a launch of its own
        else:
            out.append(cur)
    return out


class ByteGradAlgorithmImpl(AlgorithmImpl):
    def __init__(self, process_group, hierarchical: bool = True, average: bool = True):
        super().__init__(process_group)
        self.hierarchical = hierarchical
        self.average = average

    def tensors_to_buckets(self, tensors: List[List[torch.Tensor]], do_flatten: bool) -> List[BaguaBucket]:
        """Buckets are padded so every rank owns an equal chunk; the fused kernel additionally wants 32-element chunk
        granularity (16-byte payload vectors + 32-byte wire alignment), which is still a multiple of ``nranks``
        (reference pads to ``nranks``, bytegrad.py:33-45)."""
        n = self.process_group.size()
        tensors = merge_small_buckets(tensors, bytegrad_min_bucket_bytes(tensors))
        return [BaguaBucket(b, flatten=do_flatten, name=str(i), alignment=32 * n, group=self.process_group) for i, b in enumerate(tensors)]

    def init_operations(self, bagua_ddp, bucket):
        bucket.clear_ops()
        bucket.append_centralized_synchronous_op(
            hierarchical=self.hierarchical, average=self.average, scattergather=True, compression="MinMaxUInt8", group=self.process_group
        )


class ByteGradAlgorithm(Algorithm):
    def __init__(self, hierarchical: bool = True, average: bool = True):
        self.hierarchical = hierarchical
        self.average = average

    def reify(self, process_group) -> ByteGradAlgorithmImpl:
        return ByteGradAlgorithmImpl(process_group, hierarchical=self.hierarchical, average=self.average)
