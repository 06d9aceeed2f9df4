"""Packaging for bagua_b200.

The native core is built IN-TREE by ``bagua_b200/_build.py`` (nvcc -gencode arch=compute_90a,code=sm_90a; no torch
headers), so ``pip install -e .`` / ``python setup.py build_ext --inplace`` only has to call it.  The reference
packages a Rust core through setuptools_rust and downloads NCCL at install time (setup.py:60-109 of the reference);
nothing here touches the network.
"""
from __future__ import annotations

import importlib.util
import os
from pathlib import Path

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py

ROOT = Path(__file__).resolve().parent


def _native_build(verbose: bool = True) -> None:
    spec = importlib.util.spec_from_file_location("_bagua_b200_build", ROOT / "bagua_b200" / "_build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build(verbose=verbose)


class BuildNative(Command):
    description = "compile bagua_b200/_C.so (and the optional NCCL net plugin) for sm_90a"
    user_options = [("inplace", "i", "kept for `build_ext --inplace` compatibility (the build is always in-tree)")]

    def initialize_options(self):
        self.inplace = True

    def finalize_options(self):
        pass

    def run(self):
        if os.environ.get("BAGUA_SKIP_NATIVE_BUILD") == "1":
            return
        _native_build()


class BuildPyWithNative(build_py):
    def run(self):
        self.run_command("build_ext")
        super().run()


setup(
    name="bagua-b200",
    version="0.1.0",
    description="Hopper-native distributed training engine with the capabilities of BaguaSys/bagua",
    packages=find_packages(include=["bagua_b200*", "bagua", "bagua.*", "bagua_core*"]),
    package_data={"bagua_b200": ["_C.so", "_C_torch.so", "libnccl-net-bagua.so", "*.stamp", "csrc/*", "csrc/net/*", "csrc/torch_hooks/*"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.6", "numpy", "pydantic>=2", "scikit-learn", "requests", "pybind11"],
    extras_require={"ssh": ["fabric", "paramiko"], "redis": ["redis"], "test": ["pytest", "pytest-timeout", "hypothesis"]},
    entry_points={
        "console_scripts": [
            "baguarun = bagua_b200.script.baguarun:main",
            "bagua_sys_perf = bagua_b200.script.bagua_sys_perf:main",
            "bagua_doctor = bagua_b200.script.bagua_doctor:main",
        ]
    },
    cmdclass={"build_ext": BuildNative, "build_py": BuildPyWithNative},
    zip_safe=False,
)
