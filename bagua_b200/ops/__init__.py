"""Python faces of the sm_90a kernels in ``bagua_b200/csrc`` plus their torch oracles."""
from . import optim, quant  # noqa: F401
from .optim import FusedAdam, FusedLAMB, FusedLARS, FusedLion, FusedSGD  # noqa: F401
