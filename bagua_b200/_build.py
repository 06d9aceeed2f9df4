"""In-tree build of the native core (``bagua_b200/_C.so``) for sm_90a (H100).

The reference builds its Rust/C++ core for every ``sm_XX`` nvcc knows
(rust/bagua-core/bagua-core-internal/build.rs:16-35).  This project targets exactly one
architecture: ``-gencode arch=compute_90a,code=sm_90a``.  Sources are compiled with plain
``nvcc``/``g++`` (no torch headers → seconds per file) and linked into one shared object that lives
next to the python package, so it travels with the source tree.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
OBJ_DIR = PKG_DIR / "csrc" / "build"
TARGET = PKG_DIR / "_C.so"

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.environ.get("NVCC", str(Path(CUDA_HOME) / "bin" / "nvcc"))
CXX = os.environ.get("CXX", "g++")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function"]


def _includes() -> list[str]:
    import pybind11

    incs = [str(CSRC), str(Path(CUDA_HOME) / "include"), pybind11.get_include(), sysconfig.get_paths()["include"]]
    cutlass = cutlass_include()
    if cutlass:
        incs.append(cutlass)
    return incs


def cutlass_include() -> str | None:
    """CUTLASS/CuTe header tree vendored in site-packages (used only as a header library)."""
    for sp in sys.path:
        cand = Path(sp) / "flashinfer" / "data" / "cutlass" / "include"
        if (cand / "cute").is_dir():
            return str(cand)
    return None


def _sources() -> list[Path]:
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def _deps_stamp() -> str:
    h = hashlib.sha1()
    for p in sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh"))):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(GENCODE + NVCC_FLAGS + CXX_FLAGS).encode())
    return h.hexdigest()


def _compile_one(src: Path, stamp: str, verbose: bool) -> tuple[Path, bool]:
    obj = OBJ_DIR / (src.name + ".o")
    meta = OBJ_DIR / (src.name + ".json")
    key = hashlib.sha1(src.read_bytes()).hexdigest() + stamp
    if obj.exists() and meta.exists():
        try:
            if json.loads(meta.read_text()).get("key") == key:
                return obj, False
        except Exception:
            pass
    incs = [f"-I{i}" for i in _includes()]
    if src.suffix == ".cu":
        cmd = [NVCC, *GENCODE, *NVCC_FLAGS, *incs, "-c", str(src), "-o", str(obj)]
        if os.environ.get("BAGUA_PTXAS_VERBOSE"):
            cmd[1:1] = ["-Xptxas", "-v"]
    else:
        cmd = [CXX, *CXX_FLAGS, *incs, "-c", str(src), "-o", str(obj)]
    if verbose:
        print("[bagua_b200 build]", " ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"compilation of {src.name} failed:\n{res.stdout}\n{res.stderr}")
    if verbose and res.stderr.strip():
        print(res.stderr, flush=True)
    meta.write_text(json.dumps({"key": key}))
    return obj, True


STAMP = PKG_DIR / "_C.so.stamp"


def _tree_stamp() -> str:
    """Hash of every source, header and flag that goes into ``_C.so``."""
    h = hashlib.sha1(_deps_stamp().encode())
    for src in _sources():
        h.update(src.name.encode())
        h.update(src.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every source under csrc/ for sm_90a and link ``bagua_b200/_C.so`` (incremental).

    The object cache (``csrc/build``) does not travel with a snapshot of the tree, the library and its stamp do: when the
    stamp matches the sources nothing is compiled, so a GPU box that received a current ``_C.so`` starts immediately."""
    stamp = _tree_stamp()
    if not force and TARGET.exists() and STAMP.exists() and STAMP.read_text().strip() == stamp:
        return TARGET
    if not Path(NVCC).exists():
        raise RuntimeError(f"nvcc not found at {NVCC}; set CUDA_HOME")
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    if force:
        shutil.rmtree(OBJ_DIR)
        OBJ_DIR.mkdir(parents=True)
    stamp = _deps_stamp()
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(s, stamp, verbose), srcs))
    objs = [str(o) for o, _ in results]
    changed = any(c for _, c in results)
    if changed or not TARGET.exists():
        cmd = [NVCC, *GENCODE, "-shared", "-o", str(TARGET), *objs, "-lcuda" if os.environ.get("BAGUA_LINK_LIBCUDA") else "", "-ldl", "-lpthread"]
        cmd = [c for c in cmd if c]
        if verbose:
            print("[bagua_b200 build]", " ".join(cmd), flush=True)
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    STAMP.write_text(_tree_stamp() + "\n")
    return TARGET


NET_DIR = CSRC / "net"
NET_TARGET = PKG_DIR / "libnccl-net-bagua.so"


def build_net_plugin(force: bool = False, verbose: bool = False) -> Path:
    """Build the NCCL network plugin (multi-stream TCP transport, host code only) as ``libnccl-net-bagua.so``."""
    srcs = sorted(NET_DIR.glob("*.cpp"))
    deps = srcs + sorted(NET_DIR.glob("*.h"))
    if not force and NET_TARGET.exists() and all(NET_TARGET.stat().st_mtime >= d.stat().st_mtime for d in deps):
        return NET_TARGET
    cmd = [CXX, "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-shared", f"-I{NET_DIR}", *map(str, srcs), "-o", str(NET_TARGET), "-lpthread"]
    if verbose:
        print("[bagua_b200 build]", " ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"net plugin build failed:\n{res.stdout}\n{res.stderr}")
    return NET_TARGET


HOOKS_DIR = CSRC / "torch_hooks"
HOOKS_TARGET = PKG_DIR / "_C_torch.so"


def build_torch_hooks(force: bool = False, verbose: bool = False) -> Path:
    """Build the optional torch extension with the native autograd hooks (``bagua_b200/_C_torch.so``): host code only, the one
    translation unit compiled against libtorch.  Uses the system ``g++`` (dynamic libstdc++, like torch itself)."""
    import torch
    from torch.utils import cpp_extension

    stamp_file = PKG_DIR / "_C_torch.so.stamp"
    srcs = sorted(HOOKS_DIR.glob("*.cpp"))
    stamp = hashlib.sha1(b"".join(p.read_bytes() for p in srcs) + torch.__version__.encode()).hexdigest()
    if not force and HOOKS_TARGET.exists() and stamp_file.exists() and stamp_file.read_text().strip() == stamp:
        return HOOKS_TARGET
    cxx = shutil.which("g++") or CXX
    lib_dir = str(Path(torch.__file__).parent / "lib")
    incs = [f"-I{i}" for i in cpp_extension.include_paths()] + [f"-I{sysconfig.get_paths()['include']}", f"-I{Path(CUDA_HOME) / 'include'}"]
    abi = int(getattr(torch._C, "_GLIBCXX_USE_CXX11_ABI", True))
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=_C_torch",
           "-DTORCH_API_INCLUDE_EXTENSION_H", *incs, *map(str, srcs), "-o", str(HOOKS_TARGET), f"-L{lib_dir}", "-ltorch", "-ltorch_cpu", "-lc10",
           "-lc10_cuda", "-ltorch_cuda", "-ltorch_python", f"-Wl,-rpath,{lib_dir}"]
    if verbose:
        print("[bagua_b200 build]", " ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"torch hooks extension build failed:\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}")
    stamp_file.write_text(stamp + "\n")
    return HOOKS_TARGET


def is_built() -> bool:
    return TARGET.exists()


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose=True)
    print(f"built {path}")
    print(f"built {build_net_plugin(force='--force' in sys.argv, verbose=True)}")
    print(f"built {build_torch_hooks(force='--force' in sys.argv, verbose=True)}")
