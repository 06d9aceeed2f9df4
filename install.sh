#!/usr/bin/env bash
# Build the native core in-tree (sm_90a; nvcc cross-compiles without a GPU) and install the package in editable mode.
# No network access is needed: build isolation and dependency resolution are switched off (torch, numpy, pybind11 must be present).
set -euo pipefail
cd "$(dirname "$0")"
PY="${PYTHON:-python}"
"$PY" -c "import torch, pybind11" || { echo "install.sh: torch and pybind11 must be importable" >&2; exit 1; }
command -v nvcc >/dev/null || { echo "install.sh: nvcc not found (CUDA >= 12.0 toolkit needed for sm_90a)" >&2; exit 1; }
"$PY" -c "import __graft_entry__ as g; g.build()"
"$PY" -m pip install --no-index --no-build-isolation --no-deps -e . 2>/dev/null || \
  echo "install.sh: editable install skipped (pip could not run offline); use PYTHONPATH=$(pwd) instead"
"$PY" -c "from bagua_b200 import _C; print('bagua_b200 native core:', _C.show_version())"
