"""Loader of the native core ``bagua_b200._C`` (C++ scheduler + sm_90a kernels).

On a box with a GPU the extension is mandatory — every hot op is a kernel in it and nothing silently falls back
to eager PyTorch.  It is built in-tree on first import if missing (``bagua_b200/_build.py``).
"""
from __future__ import annotations

import importlib
import os
import threading

import torch

from .define import TensorDtype

_lock = threading.Lock()
_C = None
_load_error: Exception | None = None


def _try_load():
    global _C, _load_error
    try:
        _C = importlib.import_module("bagua_b200._C")
        _load_error = None
    except Exception as e:  # noqa: BLE001
        _C = None
        _load_error = e


def native():
    """Return the native module, building it if necessary; raises with a clear message if unavailable."""
    global _C
    if _C is not None:
        return _C
    with _lock:
        if _C is not None:
            return _C
        _try_load()
        if _C is None and not os.environ.get("BAGUA_B200_NO_BUILD"):
            from . import _build

            _build.build()
            importlib.invalidate_caches()
            _try_load()
        if _C is None:
            raise RuntimeError(
                "bagua_b200 native core (_C.so) is not available: build it with `python -m bagua_b200._build` "
                f"(nvcc, sm_90a). Import error: {_load_error!r}"
            )
        return _C


def native_available() -> bool:
    try:
        native()
        return True
    except Exception:  # noqa: BLE001
        return False


# dtype codes — keep in sync with csrc/common.h
DTYPE_CODE = {
    torch.float32: 0,
    torch.float16: 1,
    torch.uint8: 2,
    torch.int64: 3,
    torch.bfloat16: 4,
}

_DTYPE_ENUM = {
    torch.float32: TensorDtype.F32,
    torch.float16: TensorDtype.F16,
    torch.bfloat16: TensorDtype.BF16,
    torch.uint8: TensorDtype.U8,
    torch.int64: TensorDtype.I64,
}


def dtype_code(dtype: torch.dtype) -> int:
    try:
        return DTYPE_CODE[dtype]
    except KeyError:
        raise ValueError(f"unsupported tensor dtype {dtype} (supported: {list(DTYPE_CODE)})") from None


def to_bagua_datatype(datatype: torch.dtype) -> TensorDtype:
    """torch dtype → :class:`TensorDtype` (reference: bagua/torch_api/utils.py:81-92, plus bf16)."""
    try:
        return _DTYPE_ENUM[datatype]
    except KeyError:
        raise ValueError(f"unsupported data type {datatype}.") from None


def stream_ptr(stream: "torch.cuda.Stream | None" = None) -> int:
    if not torch.cuda.is_available():
        return 0
    if stream is None:
        stream = torch.cuda.current_stream()
    return stream.cuda_stream
