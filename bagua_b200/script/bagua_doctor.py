"""``python -m bagua_b200.script.bagua_doctor [--json]`` — what a bug report needs, and a quick self-test.

Prints the build state of the three native libraries (and whether they are current with the sources), the toolchain and
library versions, the GPUs / NVLink peer access / symmetric-memory multicast support that the peer kernels depend on, the
``BAGUA_*`` environment that deviates from the defaults, and runs a small self-test: the C++ scheduler on the host backend
always, one fused optimizer kernel when a GPU is present, and — when started under a launcher with several ranks — an
all-reduce across the job (peer kernels on one NVSwitch node, NCCL / gloo otherwise).
Exit code 0 = everything that could be checked passed."""
from __future__ import annotations

import argparse
import json
import os
import platform
import shutil
import sys
from typing import Dict, List


def _lib_state() -> Dict[str, dict]:
    from bagua_b200 import _build

    out = {}
    stamp_ok = None
    try:
        stamp_ok = _build.STAMP.exists() and _build.STAMP.read_text().strip() == _build._tree_stamp()
    except Exception as e:  # noqa: BLE001
        stamp_ok = f"unknown ({e})"
    for name, path, current in (("_C.so (native core, sm_90a kernels)", _build.TARGET, stamp_ok),
                                ("libnccl-net-bagua.so (NCCL net plugin)", _build.NET_TARGET, None),
                                ("_C_torch.so (optional C++ autograd hooks)", _build.PKG_DIR / "_C_torch.so", None)):
        out[name] = {"path": str(path), "present": path.exists(), "bytes": path.stat().st_size if path.exists() else 0}
        if current is not None:
            out[name]["current_with_sources"] = current
    return out


def _versions() -> Dict[str, str]:
    import torch

    v = {"python": platform.python_version(), "torch": torch.__version__, "torch_cuda": str(torch.version.cuda), "platform": platform.platform()}
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    v["nvcc"] = nvcc if os.path.exists(nvcc) else "not found"
    try:
        v["nccl"] = ".".join(str(x) for x in torch.cuda.nccl.version())
    except Exception:  # noqa: BLE001
        v["nccl"] = "unavailable"
    try:
        from bagua_b200.core import native

        v["native_core"] = native().show_version()
    except Exception as e:  # noqa: BLE001
        v["native_core"] = f"NOT LOADABLE: {e}"
    return v


def _gpus() -> dict:
    import torch

    if not torch.cuda.is_available():
        return {"count": 0, "note": "no CUDA device visible: CPU/gloo backend only"}
    n = torch.cuda.device_count()
    devs = []
    for i in range(n):
        p = torch.cuda.get_device_properties(i)
        devs.append({"index": i, "name": p.name, "sm": f"{p.major}.{p.minor}", "sms": p.multi_processor_count, "memory_GiB": round(p.total_memory / 2 ** 30, 1)})
    peer = [[(i == j) or bool(torch.cuda.can_device_access_peer(i, j)) for j in range(n)] for i in range(n)]
    info = {"count": n, "devices": devs, "peer_access_all_pairs": all(all(r) for r in peer)}
    if any(d["sm"] != "9.0" for d in devs):
        info["warning"] = "the kernels are compiled for sm_90a only (H100); other architectures cannot load them"
    try:
        import torch.distributed._symmetric_memory as symm  # noqa: F401

        info["torch_symmetric_memory"] = True
    except Exception:  # noqa: BLE001
        info["torch_symmetric_memory"] = False
    return info


def _environment() -> Dict[str, str]:
    from bagua_b200 import env

    changed = {}
    for s in env.SETTINGS.values():
        if s.var in os.environ:
            changed[s.var] = os.environ[s.var]
    for k, v in os.environ.items():
        if (k.startswith("BAGUA_") or k.startswith("NCCL_")) and k not in changed:
            changed[k] = v
    return changed


def native_mod():
    from bagua_b200.core import native

    return native()


def _self_test(peer_kernels: bool = False) -> List[dict]:
    import numpy as np
    import torch

    results = []

    def check(name, fn):
        try:
            detail = fn()
            results.append({"test": name, "ok": True, "detail": detail})
        except Exception as e:  # noqa: BLE001
            results.append({"test": name, "ok": False, "detail": f"{type(e).__name__}: {e}"})

    def scheduler():
        from bagua_b200.core import native

        C = native()
        be = C.Backend(4, -1, 0, 10.0)
        src, dst = np.arange(16, dtype=np.float32), np.zeros(16, dtype=np.float32)
        t = C.Tensor("t", src.ctypes.data, 16, 0, -1)
        b = C.Bucket("b", [t])
        b.append_op(C.CopyOp(dst.ctypes.data, src.ctypes.data, 64))
        be.register_ordered_buckets([b])
        for inline in (False, True):
            dst[:] = 0
            be.set_inline(inline)
            be.mark_communication_ready(t, 0)
            assert be.wait_pending_comm_ops(0, True) == 1 and (dst == src).all()
        be.shutdown()
        return "ordered scheduling, worker and inline issue"

    check("C++ scheduler (host backend)", scheduler)

    def net_plugin():
        from bagua_b200 import net

        h = net.PluginHandle()
        return f"{len(h.devices())} usable interface(s)"

    check("NCCL net plugin loads", net_plugin)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:   # started under a launcher: exercise the communication path of this job
        def collective():
            import bagua_b200 as bagua

            on_gpu = torch.cuda.is_available() and os.environ.get("BAGUA_FORCE_CPU", "0") != "1"
            if on_gpu:
                torch.cuda.set_device(bagua.get_local_rank())
            if not bagua.is_initialized():
                bagua.init_process_group()
            n, r = bagua.get_world_size(), bagua.get_rank()
            detail = []
            for numel in (1024, 1 << 20):       # latency-bound (one-shot kernel) and bandwidth-bound message
                t = torch.full((numel,), float(r + 1), device="cuda" if on_gpu else "cpu")
                bagua.allreduce_inplace(t, op=bagua.ReduceOp.AVG)
                assert torch.allclose(t, torch.full_like(t, (n + 1) / 2)), f"all-reduce of {numel} elements is wrong on rank {r}"
            eng = bagua.communication._get_default_group().peer_engine() if on_gpu else None
            detail.append(f"{n} ranks, backend {'nccl + peer kernels' if eng is not None else ('nccl' if on_gpu else 'gloo')}")
            if eng is not None:
                detail.append(f"NVLS multicast {'available' if eng.has_multicast else 'not available'}")
            return ", ".join(detail)

        check("all-reduce across the job", collective)
    if torch.cuda.is_available():
        def fused_step():
            from bagua_b200.ops.optim import flat_sgd_

            p = torch.ones(4096, device="cuda")
            g = torch.full((4096,), 0.5, device="cuda")
            flat_sgd_(p, g, None, lr=0.1)
            torch.cuda.synchronize()
            assert torch.allclose(p, torch.full_like(p, 0.95))
            return "flat_sgd kernel"

        check("fused optimizer kernel (sm_90a)", fused_step)
        if peer_kernels:
            def virtual_world():
                """A 4-rank all-reduce, a fused allreduce+SGD step and a ByteGrad exchange among VIRTUAL ranks on this one GPU
                (parallel/virtual.py): the peer kernels' slice arithmetic, barriers and quantisation without a second GPU."""
                from bagua_b200.core import dtype_code
                from bagua_b200.parallel.virtual import VirtualPeerWorld

                C = native_mod()
                P, n = 4, 1 << 16
                w = VirtualPeerWorld(P, torch.device("cuda", torch.cuda.current_device()), timeout_s=10.0)
                buf = w.alloc(n * 4)
                for r in range(P):
                    buf.view(r, torch.float32, n).fill_(float(r + 1))
                w.run(lambda r: C.AllReduceOp(w.comms[r], buf.buf, buf.buf, 0, 0, n * 4, dtype_code(torch.float32), 1.0 / P, C.AR_TWO_SHOT, w.cfg(4)))
                assert all(torch.allclose(buf.view(r, torch.float32, n), torch.full((n,), (P + 1) / 2, device="cuda")) for r in range(P))
                numel = 32 * P * 64
                box = C.ByteGradOp.box_bytes(numel, P)
                inbox, outbox = w.alloc(box), w.alloc(box)
                datas = [torch.linspace(-1, 1, numel, device="cuda") * (r + 1) for r in range(P)]
                want = sum(datas) / P
                w.run(lambda r: C.ByteGradOp(w.comms[r], datas[r].data_ptr(), numel, dtype_code(torch.float32), inbox.buf, 0, outbox.buf, 0, True, w.cfg(2 * P, 256)))
                err = max((d - want).abs().max().item() for d in datas)
                assert err <= 2.5 * (2.0 * P) / 255, f"ByteGrad error {err}"
                return f"two-shot all-reduce and fused ByteGrad among {P} virtual ranks (max quantisation error {err:.4f})"

            check("peer kernels among virtual ranks (one GPU)", virtual_world)
    return results


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--json", action="store_true", help="machine-readable report")
    ap.add_argument("--no-self-test", action="store_true")
    ap.add_argument("--kernels", action="store_true", help="also run the NVSwitch peer kernels among virtual ranks on this GPU (no second GPU needed)")
    args = ap.parse_args(argv)
    report = {"libraries": _lib_state(), "versions": _versions(), "gpus": _gpus(), "environment": _environment()}
    report["self_test"] = [] if args.no_self_test else _self_test(peer_kernels=args.kernels)
    ok = all(r["ok"] for r in report["self_test"]) and report["libraries"]["_C.so (native core, sm_90a kernels)"]["present"]
    report["ok"] = bool(ok)
    if args.json:
        print(json.dumps(report, indent=1, default=str))
    else:
        for section in ("versions", "libraries", "gpus", "environment"):
            print(f"== {section}")
            for k, v in report[section].items():
                print(f"  {k}: {v}")
        print("== self test")
        for r in report["self_test"]:
            print(f"  [{'ok' if r['ok'] else 'FAIL'}] {r['test']}: {r['detail']}")
        print("RESULT:", "ok" if ok else "problems found")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
