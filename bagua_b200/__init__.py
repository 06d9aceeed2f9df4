"""bagua_b200 — a Hopper-native (sm_90a, NVLink 4 / NVSwitch) data-parallel training engine with the capabilities
and public API of BaguaSys/bagua (``import bagua_b200 as bagua`` or, unchanged user code, ``import bagua.torch_api as bagua``).

Public surface mirrors ``bagua/torch_api/__init__.py:25-63`` of the reference."""
from __future__ import annotations

__version__ = "0.1.0"

import logging as _logging
import os as _os

# LOG_LEVEL (TRACE|DEBUG|INFO|WARN|ERROR) drives both the native core's stderr log (csrc/log.h) and this package's loggers
_lvl = {"TRACE": 5, "DEBUG": _logging.DEBUG, "INFO": _logging.INFO, "WARN": _logging.WARNING, "WARNING": _logging.WARNING,
        "ERROR": _logging.ERROR}.get(_os.environ.get("LOG_LEVEL", "").upper())
if _lvl is not None:
    _logging.getLogger(__name__).setLevel(_lvl)

from . import env  # noqa: F401
from .env import get_rank, get_world_size, get_local_rank, get_local_size, get_node_rank  # noqa: F401
from . import tensor as _tensor_patch  # noqa: F401  (installs torch.Tensor.*bagua* methods)
from . import communication  # noqa: F401
from .communication import (  # noqa: F401
    ReduceOp,
    init_process_group,
    is_initialized,
    new_group,
    from_torch_group,
    send,
    recv,
    broadcast,
    broadcast_coalesced,
    broadcast_object,
    reduce,
    reduce_inplace,
    allreduce,
    allreduce_inplace,
    allreduce_coalesced_inplace,
    allgather,
    allgather_inplace,
    gather,
    gather_inplace,
    scatter,
    scatter_inplace,
    reduce_scatter,
    reduce_scatter_inplace,
    alltoall,
    alltoall_inplace,
    alltoall_v,
    alltoall_v_inplace,
    barrier,
)
from . import bucket  # noqa: F401
from .parallel import distributed as _module_patch  # noqa: F401  (installs nn.Module.with_bagua)
from .parallel.distributed import BaguaModule  # noqa: F401
from .parallel import algorithms  # noqa: F401
from .parallel import data_parallel  # noqa: F401
from .parallel.data_parallel import DistributedDataParallel  # noqa: F401
from . import contrib  # noqa: F401
from . import ops  # noqa: F401
from . import checkpoint  # noqa: F401
from .parallel import moe  # noqa: F401
from . import amp  # noqa: F401


def version() -> str:
    """Package version string."""
    return __version__
