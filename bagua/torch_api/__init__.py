"""``bagua.torch_api`` → :mod:`bagua_b200`; reference sub-module paths are aliased onto the new layout."""
import importlib as _importlib
import sys as _sys

import bagua_b200 as _b
from bagua_b200 import *  # noqa: F401,F403
from bagua_b200 import (  # noqa: F401
    ReduceOp, init_process_group, is_initialized, new_group, from_torch_group, get_rank, get_world_size, get_local_rank, get_local_size,
    send, recv, broadcast, broadcast_coalesced, broadcast_object, reduce, reduce_inplace, allreduce, allreduce_inplace,
    allreduce_coalesced_inplace, allgather, allgather_inplace, gather, gather_inplace, scatter, scatter_inplace, reduce_scatter,
    reduce_scatter_inplace, alltoall, alltoall_inplace, alltoall_v, alltoall_v_inplace, barrier, BaguaModule, DistributedDataParallel,
)

_ALIASES = {
    "env": "bagua_b200.env",
    "communication": "bagua_b200.communication",
    "tensor": "bagua_b200.tensor",
    "bucket": "bagua_b200.bucket",
    "utils": "bagua_b200.utils",
    "distributed": "bagua_b200.parallel.distributed",
    "algorithms": "bagua_b200.parallel.algorithms",
    "algorithms.base": "bagua_b200.parallel.algorithms.base",
    "algorithms.gradient_allreduce": "bagua_b200.parallel.algorithms.gradient_allreduce",
    "algorithms.bytegrad": "bagua_b200.parallel.algorithms.bytegrad",
    "algorithms.decentralized": "bagua_b200.parallel.algorithms.decentralized",
    "algorithms.q_adam": "bagua_b200.parallel.algorithms.q_adam",
    "algorithms.async_model_average": "bagua_b200.parallel.algorithms.async_model_average",
    "data_parallel": "bagua_b200.parallel.data_parallel",
    "data_parallel.distributed": "bagua_b200.parallel.data_parallel.distributed",
    "data_parallel.functional": "bagua_b200.parallel.data_parallel.functional",
    "data_parallel.bagua_distributed": "bagua_b200.parallel.bagua_distributed",
    "contrib": "bagua_b200.contrib",
    "contrib.fuse": "bagua_b200.contrib.fuse",
    "contrib.fuse.optimizer": "bagua_b200.contrib.fuse.optimizer",
    "contrib.sync_batchnorm": "bagua_b200.contrib.sync_batchnorm",
    "contrib.load_balancing_data_loader": "bagua_b200.contrib.load_balancing_data_loader",
    "contrib.cache_loader": "bagua_b200.contrib.cache_loader",
    "contrib.cached_dataset": "bagua_b200.contrib.cached_dataset",
    "contrib.utils": "bagua_b200.contrib.utils",
    "contrib.utils.store": "bagua_b200.contrib.utils.store",
    "contrib.utils.redis_store": "bagua_b200.contrib.utils.redis_store",
    "checkpoint": "bagua_b200.checkpoint",
    "checkpoint.checkpointing": "bagua_b200.checkpoint.checkpointing",
    "model_parallel": "bagua_b200.parallel",
    "model_parallel.moe": "bagua_b200.parallel.moe",
    "model_parallel.moe.layer": "bagua_b200.parallel.moe.layer",
    "model_parallel.moe.sharded_moe": "bagua_b200.parallel.moe.sharded_moe",
    "model_parallel.moe.experts": "bagua_b200.parallel.moe.experts",
    "model_parallel.moe.utils": "bagua_b200.parallel.moe.utils",
    "moe": "bagua_b200.parallel.moe",
    "ops": "bagua_b200.ops",
    "amp": "bagua_b200.amp",
}
for _k, _v in _ALIASES.items():
    _m = _importlib.import_module(_v)
    _sys.modules[f"{__name__}.{_k}"] = _m
    if "." not in _k:
        globals()[_k] = _m
