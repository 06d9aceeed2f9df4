"""Public API surface parity (SURVEY Appendix A): names importable through ``bagua.torch_api`` / ``bagua_core`` exactly as
user code of the reference expects, tensor/bucket patch methods, multiple models in one process."""
import copy
import json
import os

import pytest
import torch

from tests.mp_utils import run_distributed


def test_reference_import_paths_resolve():
    import bagua.torch_api as bagua
    from bagua.bagua_define import BaguaHyperparameter, TensorDeclaration, TensorDtype, get_tensor_declaration_bytes  # noqa: F401
    from bagua.service import AutotuneClient, AutotuneService  # noqa: F401
    from bagua.service.autotune_task_manager import AutotuneTaskManager  # noqa: F401
    from bagua.service.bayesian_optimizer import BayesianOptimizer, BoolParam, FloatParam, IntParam  # noqa: F401
    from bagua.torch_api.algorithms import Algorithm, GlobalAlgorithmRegistry, async_model_average, bytegrad, decentralized, gradient_allreduce, q_adam  # noqa: F401
    from bagua.torch_api.bucket import BaguaBucket  # noqa: F401
    from bagua.torch_api.checkpoint import load_checkpoint, save_checkpoint  # noqa: F401
    from bagua.torch_api.communication import ReduceOp, _get_default_group, _rank_not_in_group, from_torch_group, init_process_group, is_initialized, new_group  # noqa: F401
    from bagua.torch_api.contrib import CachedDataset, CacheLoader, LoadBalancingDistributedBatchSampler, LoadBalancingDistributedSampler, fuse_optimizer  # noqa: F401
    from bagua.torch_api.contrib.sync_batchnorm import SyncBatchNorm  # noqa: F401
    from bagua.torch_api.contrib.utils.redis_store import RedisStore  # noqa: F401
    from bagua.torch_api.contrib.utils.store import ClusterStore, Store  # noqa: F401
    from bagua.torch_api.data_parallel import DistributedDataParallel  # noqa: F401
    from bagua.torch_api.data_parallel.functional import all_reduce  # noqa: F401
    from bagua.torch_api.model_parallel.moe import MoE  # noqa: F401
    from bagua.torch_api.moe import is_moe_param  # noqa: F401
    from bagua.torch_api.utils import StatisticalAverage  # noqa: F401

    for name in ["init_process_group", "get_rank", "get_world_size", "get_local_rank", "get_local_size", "send", "recv", "broadcast", "broadcast_coalesced",
                 "broadcast_object", "reduce", "reduce_inplace", "allreduce", "allreduce_inplace", "allreduce_coalesced_inplace", "allgather",
                 "allgather_inplace", "gather", "gather_inplace", "scatter", "scatter_inplace", "reduce_scatter", "reduce_scatter_inplace", "alltoall",
                 "alltoall_inplace", "alltoall_v", "alltoall_v_inplace", "barrier", "ReduceOp", "BaguaModule", "DistributedDataParallel"]:
        assert hasattr(bagua, name), name
    assert [int(ReduceOp.SUM), int(ReduceOp.PRODUCT), int(ReduceOp.MIN), int(ReduceOp.MAX), int(ReduceOp.BOR), int(ReduceOp.BAND), int(ReduceOp.BXOR),
            int(ReduceOp.AVG)] == [0, 1, 2, 3, 7, 8, 9, 10]
    assert set(GlobalAlgorithmRegistry.available_algorithms()) == {"gradient_allreduce", "bytegrad", "decentralized", "low_precision_decentralized", "qadam", "async"}
    assert isinstance(Algorithm.init("gradient_allreduce", hierarchical=True), gradient_allreduce.GradientAllReduceAlgorithm)
    for m in ("with_bagua", "bagua_module_name", "bagua_algorithm", "bagua_optimizers", "bagua_buckets"):
        assert hasattr(torch.nn.Module, m)
    for m in ("is_bagua_tensor", "ensure_bagua_tensor", "to_bagua_tensor", "bagua_getter_closure", "bagua_setter_closure", "bagua_backend_tensor",
              "bagua_ensure_grad", "bagua_mark_communication_ready", "bagua_mark_communication_ready_without_synchronization", "bagua_set_storage"):
        assert hasattr(torch.Tensor, m), m


def test_bagua_core_shim():
    import bagua_core as B

    assert "bagua_b200" in B.show_version()
    t = torch.arange(8, dtype=torch.float32)
    bt = B.BaguaTensorPy("t", t)
    assert bt.num_elements() == 8 and bt.dtype() == "f32" and bt.data_ptr() == t.data_ptr() and bt.device_id() == -1
    bucket = B.BaguaBucketPy("b", [bt])
    be = B.BaguaCommBackendPy(10, -1)
    hits = []
    bucket.append_python_op(lambda name: hits.append(name))
    be.register_ordered_buckets([bucket])
    be.mark_communication_ready(bt, 0)
    assert be.wait_pending_comm_ops() == 1 and hits == ["b"]
    c = bt.compress("MinMaxUInt8", 1)
    out = B.BaguaTensorPy("o", torch.zeros(8))
    out.decompress_from("MinMaxUInt8", 1, c)
    assert torch.allclose(out.torch_tensor, t, atol=7 / 255)
    assert list(c.to_numpy_u8()[32:40]) == [0, 36, 73, 109, 146, 182, 219, 255]


def _tensor_bucket_worker(rank, world):
    import bagua_b200 as bagua
    from bagua_b200.bucket import BaguaBucket

    bagua.init_process_group()
    p1, p2 = torch.nn.Parameter(torch.randn(3, 5)), torch.nn.Parameter(torch.randn(7))
    for p in (p1, p2):
        p.bagua_ensure_grad()
    t1 = p1.ensure_bagua_tensor("p1", "m", getter_closure=lambda p: p.grad, setter_closure=lambda p, t: setattr(p, "grad", t))
    t2 = p2.ensure_bagua_tensor("p2", "m", getter_closure=lambda p: p.grad, setter_closure=lambda p, t: setattr(p, "grad", t))
    assert t1.is_bagua_tensor() and t1.bagua_tensor_name == "p1" and t1.bagua_getter_closure() is p1.grad
    with pytest.raises(AssertionError):
        p1.ensure_bagua_tensor("other", "m")
    p1.grad.fill_(1.0)
    p2.grad.fill_(2.0)
    b = BaguaBucket([t1, t2], "b0", flatten=True, alignment=8)
    assert b.check_flatten() and b.padding_tensor is not None and b.padding_tensor.numel() == 2 and b.numel() == 24 and b.bytes() == 22 * 4
    assert torch.equal(b.backend_tensor[:15], torch.ones(15)) and torch.equal(b.backend_tensor[15:22], torch.full((7,), 2.0))
    assert p1.grad.data_ptr() == b.backend_tensor.data_ptr() and p1.bagua_backend_tensor().data_ptr() == p1.grad.data_ptr()
    p1.grad.add_(rank)  # writes go through the flat storage
    ran = []
    b.append_python_op(lambda name: ran.append(name)).append_centralized_synchronous_op(average=True)
    be = bagua.communication.get_backend("m")
    be.register_ordered_buckets([b.backend_bucket])
    t1.bagua_mark_communication_ready()
    t2.bagua_mark_communication_ready_without_synchronization()
    be.wait_pending_comm_ops(0, True)
    assert ran == ["b0"] and torch.allclose(p1.grad, torch.full((3, 5), 1.0 + (world - 1) / 2)) and torch.equal(p2.grad, torch.full((7,), 2.0))
    b.clear_ops()
    assert b.backend_bucket.num_ops() == 0
    return True


def test_tensor_and_bucket_api():
    assert all(run_distributed(_tensor_bucket_worker, world=2))


def _multi_models_worker(rank, world):
    """Two models with different algorithms in one process (reference: tests/torch_api/test_multi_models.py) —
    one native scheduler per module name."""
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms import bytegrad, gradient_allreduce

    bagua.init_process_group()
    torch.manual_seed(rank)
    nets = [torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 2)) for _ in range(2)]
    opts = [torch.optim.SGD(n.parameters(), lr=0.1) for n in nets]
    nets[0] = nets[0].with_bagua([opts[0]], gradient_allreduce.GradientAllReduceAlgorithm())
    nets[1] = nets[1].with_bagua([opts[1]], bytegrad.ByteGradAlgorithm())
    assert nets[0].bagua_module_name != nets[1].bagua_module_name
    for it in range(4):
        for n, o in zip(nets, opts):
            x = torch.randn(4, 8)
            o.zero_grad()
            F.mse_loss(n(x), torch.zeros(4, 2)).backward()
            o.step()
    return [torch.cat([p.detach().reshape(-1) for p in n.parameters()]) for n in nets]


def test_multiple_models_in_one_process():
    r0, r1 = run_distributed(_multi_models_worker, world=2)
    assert torch.equal(r0[0], r1[0])
    assert torch.allclose(r0[1], r1[1], atol=1e-2)


# names of the reference that are implementation details of ITS design (NCCL unique-id plumbing, Flask glue, the internals of
# its alias-based fused optimizer) and have no counterpart by construction
_NOT_APPLICABLE = {
    "bagua.torch_api.communication": {"run_flask_app"},
    "bagua.torch_api.contrib.fuse.optimizer": {"flatten_tensors_with_closure", "flatten_params_and_states", "group_tensors", "infer_state_tensors",
                                               "make_optimizer_instance", "fuse_step", "do_fuse", "check_optimizer", "sync_param_group_scalars",
                                               "sync_optimizer_state", "get_tensor_state", "get_optimizer_param_states"},
}


REFERENCE_API = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_api.json")


def _reference_api() -> dict:
    """Public names and parameter lists of every module of the reference's python package, stored as golden data
    (``scripts/reference_api_golden.py`` extracts them from a checkout of the reference)."""
    with open(REFERENCE_API) as f:
        return json.load(f)["modules"]


def test_every_public_name_of_the_reference_python_package_resolves():
    """Each public top-level class / function of the reference's python package exists under the same module path in the
    ``bagua`` alias package."""
    import importlib

    missing = []
    for mod, api in sorted(_reference_api().items()):
        if mod.startswith("bagua.script") or mod.startswith("bagua.distributed"):
            continue  # CLI entry points: covered by tests/test_launchers.py
        try:
            m = importlib.import_module(mod)
        except Exception as e:  # noqa: BLE001
            missing.append(f"{mod}: import failed: {e!r}")
            continue
        for n in api["names"]:
            if not hasattr(m, n) and n not in _NOT_APPLICABLE.get(mod, ()):
                missing.append(f"{mod}.{n}")
    assert not missing, missing


def test_compat_helpers_behave():
    import torch.distributed as dist

    from bagua.torch_api.communication import CommMember
    from bagua.torch_api.data_parallel.functional import torch_reduce_op_to_bagua
    from bagua.torch_api.utils import apply_flattened_call_all
    from bagua_b200 import ReduceOp

    assert torch_reduce_op_to_bagua(dist.ReduceOp.SUM) == ReduceOp.SUM and torch_reduce_op_to_bagua(dist.ReduceOp.MAX) == ReduceOp.MAX
    with pytest.raises(ValueError):
        torch_reduce_op_to_bagua("nonsense")
    ts = [torch.ones(3), torch.full((2, 2), 2.0), torch.ones(4, dtype=torch.float64)]
    apply_flattened_call_all(ts, lambda flat: flat.mul_(3))
    assert torch.equal(ts[0], torch.full((3,), 3.0)) and torch.equal(ts[1], torch.full((2, 2), 6.0)) and torch.equal(ts[2], torch.full((4,), 3.0, dtype=torch.float64))
    assert CommMember.NON_COMM_MEMBER is not None


def _core_shim_ops_worker(rank, world):
    """Low-level ``bagua_core`` usage as in the reference's rust-level tests: loose tensors → BaguaTensorPy → BaguaBucketPy with a
    centralized (plain and MinMaxUInt8) and a decentralized op → BaguaCommBackendPy."""
    import bagua_b200 as bagua
    import bagua_core as B

    bagua.init_process_group()
    a, b = torch.full((8,), float(rank + 1)), torch.full((4, 2), float(10 * (rank + 1)))
    ta, tb = B.BaguaTensorPy("a", a), B.BaguaTensorPy("b", b)
    bucket = B.BaguaBucketPy("bk", [ta, tb])
    bucket.append_centralized_synchronous_op(None, None, hierarchical=False, average=True)
    backend = B.BaguaCommBackendPy(10, -1)
    backend.register_ordered_buckets([bucket])
    backend.mark_communication_ready(ta, 0)
    backend.mark_communication_ready(tb, 0)
    assert backend.wait_pending_comm_ops() == 1
    plain = (a.clone(), b.clone())
    # compressed: values land within the 8-bit quantisation error of the mean
    c = torch.linspace(-1, 1, 16) * (rank + 1)
    tc = B.BaguaTensorPy("c", c)
    peer = torch.zeros(16)
    b2 = B.BaguaBucketPy("bk2", [tc])
    b2.append_centralized_synchronous_op(None, None, hierarchical=False, average=True, scattergather=True, compression="MinMaxUInt8")
    b2.append_decentralized_synchronous_op(None, None, hierarchical=False, peer_selection_mode="shift_one", peer_weight=B.BaguaTensorPy("pw", peer))
    backend2 = B.BaguaCommBackendPy(10, -1)
    backend2.register_ordered_buckets([b2])
    backend2.mark_communication_ready(tc, 0)
    backend2.wait_pending_comm_ops()
    # low-precision decentralized ring + asynchronous average on loose tensors (bagua-core-py/src/lib.rs:479-519)
    w0 = torch.linspace(0, 1, 32)
    x = w0 + 0.1 * (rank + 1)                         # "weights after the local step"
    tx = B.BaguaTensorPy("x", x)
    weight, left, right = w0.clone(), w0.clone(), w0.clone()
    b3 = B.BaguaBucketPy("bk3", [tx])
    b3.append_low_precision_decentralized_synchronous_op(None, None, hierarchical=False, peer_selection_mode="ring", compression="MinMaxUInt8",
                                                          weight=B.BaguaTensorPy("w", weight), left_peer_weight=B.BaguaTensorPy("l", left),
                                                          right_peer_weight=B.BaguaTensorPy("r", right))
    y = torch.full((6,), float(rank))
    ty = B.BaguaTensorPy("y", y)
    b4 = B.BaguaBucketPy("bk4", [ty])
    op = b4.append_decentralized_asynchronous_op(None, None, peer_selection_mode="all", torch_stream=0)
    backend3 = B.BaguaCommBackendPy(10, -1)
    backend3.register_ordered_buckets([b3, b4])
    assert op.get_status() is True
    op.lock_weight()
    y.add_(10.0)                                      # the trainer's update, made while it holds the weights
    op.unlock_weight()
    backend3.mark_communication_ready(tx, 0)
    backend3.mark_communication_ready(ty, 0)
    backend3.wait_pending_comm_ops()
    first = y.clone()
    ring = (x.clone(), weight.clone(), left.clone(), right.clone(), w0)
    op.abort()
    assert op.get_status() is False
    backend3.mark_communication_ready(tx, 0)
    backend3.mark_communication_ready(ty, 0)
    backend3.wait_pending_comm_ops()
    aborted = y.clone()
    op.reset()
    assert op.get_status() is True
    return plain, c.clone(), peer.clone(), ring, (first, aborted)


def test_bagua_core_shim_low_level_ops():
    res = run_distributed(_core_shim_ops_worker, world=2)
    for rank, ((a, b), c, peer, lp, (first, aborted)) in enumerate(res):
        assert torch.equal(a, torch.full((8,), 1.5)) and torch.equal(b, torch.full((4, 2), 15.0))
        torch.testing.assert_close(c, torch.linspace(-1, 1, 16) * 1.5, rtol=0, atol=0.03)
        torch.testing.assert_close(peer, c, rtol=0, atol=1e-6)      # both ranks hold the same compressed mean → pair average = itself
        # ring step: with all replicas equal to w0 the difference x + (l + r)/3 - 5w/3 = (x - w0) is what travels (8-bit); every rank's
        # own replica moves by its own difference, the neighbour replicas by the neighbour's (2 ranks: left = right = the other rank)
        x, weight, left, right, w0 = lp
        mine, other = 0.1 * (rank + 1), 0.1 * (2 - rank)
        torch.testing.assert_close(weight - w0, torch.full((32,), mine), rtol=0, atol=2e-3)
        torch.testing.assert_close(left - w0, torch.full((32,), other), rtol=0, atol=2e-3)
        torch.testing.assert_close(right - w0, torch.full((32,), other), rtol=0, atol=2e-3)
        assert torch.equal(x, weight)
        # asynchronous average: y = rank + 10 on both ranks → mean 10.5; an aborted op leaves the tensors alone
        assert torch.equal(first, torch.full((6,), 10.5)) and torch.equal(aborted, first)


REFERENCE_MODULES = [
    "bagua", "bagua.bagua_define", "bagua.distributed", "bagua.distributed.launch", "bagua.distributed.run", "bagua.script", "bagua.script.baguarun",
    "bagua.service", "bagua.service.autotune_service", "bagua.service.autotune_system", "bagua.service.autotune_task_manager",
    "bagua.service.bayesian_optimizer", "bagua.torch_api", "bagua.torch_api.algorithms", "bagua.torch_api.algorithms.async_model_average",
    "bagua.torch_api.algorithms.base", "bagua.torch_api.algorithms.bytegrad", "bagua.torch_api.algorithms.decentralized",
    "bagua.torch_api.algorithms.gradient_allreduce", "bagua.torch_api.algorithms.q_adam", "bagua.torch_api.bucket", "bagua.torch_api.checkpoint",
    "bagua.torch_api.checkpoint.checkpointing", "bagua.torch_api.communication", "bagua.torch_api.contrib", "bagua.torch_api.contrib.cache_loader",
    "bagua.torch_api.contrib.cached_dataset", "bagua.torch_api.contrib.fuse", "bagua.torch_api.contrib.fuse.optimizer",
    "bagua.torch_api.contrib.load_balancing_data_loader", "bagua.torch_api.contrib.sync_batchnorm", "bagua.torch_api.contrib.utils",
    "bagua.torch_api.contrib.utils.redis_store", "bagua.torch_api.contrib.utils.store", "bagua.torch_api.data_parallel",
    "bagua.torch_api.data_parallel.bagua_distributed", "bagua.torch_api.data_parallel.distributed", "bagua.torch_api.data_parallel.functional",
    "bagua.torch_api.distributed", "bagua.torch_api.env", "bagua.torch_api.model_parallel", "bagua.torch_api.model_parallel.moe",
    "bagua.torch_api.model_parallel.moe.experts", "bagua.torch_api.model_parallel.moe.layer", "bagua.torch_api.model_parallel.moe.sharded_moe",
    "bagua.torch_api.model_parallel.moe.utils", "bagua.torch_api.tensor", "bagua.torch_api.utils", "bagua.version",
]


def test_every_module_path_of_the_reference_package_imports():
    """All 49 python modules of the reference's ``bagua`` package (the modules of tests/golden/reference_api.json) exist under the same
    dotted path in the alias package, so ``import bagua.torch_api.contrib.cache_loader`` style imports in user code keep working."""
    import importlib

    assert sorted(REFERENCE_MODULES) == sorted(_reference_api())
    missing = []
    for name in REFERENCE_MODULES:
        try:
            importlib.import_module(name)
        except Exception as e:  # noqa: BLE001
            missing.append(f"{name}: {type(e).__name__}: {e}")
    assert not missing, missing


def _compat_symbols_worker(rank, world):
    """Helpers of the reference that user code may touch: comm.WORLD, the ProcessGroup patch class, NCCL-id broadcast through the
    store, the abstract DDP interface and what the concrete wrapper fills in."""
    import base64

    import torch
    import torch.distributed as dist

    import bagua.torch_api as bagua
    from bagua.torch_api import communication as C
    from bagua.torch_api.data_parallel.distributed import DistributedDataParallel_V1_9_0_Interface

    bagua.init_process_group()
    assert C.comm.WORLD is C.CommMember.WORLD
    t = torch.ones(3) * (rank + 1)
    bagua.allreduce_inplace(t, comm=C.comm.WORLD)
    assert t.tolist() == [3.0, 3.0, 3.0]
    pg = dist.group.WORLD
    assert pg.bagua_patch() is pg and isinstance(pg.bagua_pg, C.BaguaProcessGroup) and pg.bagua_get_global_communicator().nranks() == world
    assert dist.ProcessGroup.bagua_patch is C.BaguaProcessGroupPatch.bagua_patch
    ident = C.broadcast_nccl_unique_id("test_comm_key", root=1)
    assert len(base64.b64decode(ident)) == 128
    gathered = [None] * world
    dist.all_gather_object(gathered, ident)
    assert gathered[0] == gathered[1], "every rank must hold the id that rank 1 generated"

    iface = DistributedDataParallel_V1_9_0_Interface()
    for call in (lambda: iface.scatter((), {}, [0]), lambda: iface.gather([], 0), lambda: iface.register_comm_hook(None, None), iface.will_sync_module_buffers):
        try:
            call()
            raise AssertionError("the interface must stay abstract")
        except NotImplementedError:
            pass
    net = torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.BatchNorm1d(4))
    ddp = bagua.data_parallel.DistributedDataParallel(net, optimizers=[torch.optim.SGD(net.parameters(), lr=0.1)])
    assert ddp.will_sync_module_buffers() is True and ddp.train(False) is ddp and not ddp.training and ddp.train() is ddp
    assert all(callable(getattr(ddp, m)) for m in ("scatter", "to_kwargs", "gather"))   # device movers: exercised on GPUs only
    for call in (lambda: ddp.join(), lambda: ddp.register_comm_hook(None, None)):
        try:
            call()
            raise AssertionError("unsupported DDP features must say so")
        except NotImplementedError as e:
            assert str(e)
    return True


def test_compat_symbols_of_the_reference_modules():
    from tests.mp_utils import run_distributed

    assert all(run_distributed(_compat_symbols_worker, world=2))


def test_sampler_and_cache_compat_methods():
    import torch

    from bagua.torch_api.contrib.cache_loader import BatchFetcher
    from bagua.torch_api.contrib.load_balancing_data_loader import LoadBalancingDistributedBatchSampler, LoadBalancingDistributedSampler
    from bagua_b200.contrib.utils.store import MemoryStore

    data = [torch.zeros(n) for n in (5, 1, 9, 3, 7, 2, 8, 4)]
    s = LoadBalancingDistributedSampler(data, complexity_fn=len, num_replicas=2, rank=1, shuffle=True, seed=3)
    s.set_epoch(2)
    chunks, order = s.shuffle_chunks()
    assert sorted(i for c in chunks for i in c) == list(range(8)) and sorted(order) == list(range(4)) and all(len(c) == 2 for c in chunks)
    assert list(s) == [chunks[i][1] for i in order]                      # replica 1 reads column 1 of the chunks in this epoch's order
    assert all(abs(len(data[a]) - len(data[b])) <= 2 for a, b in chunks)   # neighbours in cost (jitter of at most 1 here)
    bs = LoadBalancingDistributedBatchSampler(LoadBalancingDistributedSampler(data, complexity_fn=len, num_replicas=2, rank=0), batch_fn=lambda idx: [idx[i:i + 3] for i in range(0, len(idx), 3)])
    before = list(bs)
    bs.generate_batches()
    assert list(bs) == before and len(bs) == 2

    store = MemoryStore()
    f = BatchFetcher(store, read_buffer_size=4, writer_buffer_size=2)
    assert f.read("a") is None
    f.write("a", {"x": 1})
    assert f.read("a") == {"x": 1} and store.get("a") is None and list(f.write_map) == ["a"]     # still buffered
    f.write("b", [2])
    assert store.get("a") is not None and not f.write_map                                        # the buffer reached its size
    f.write("c", 3)
    f.write_post_read()
    assert store.get("c") is None
    f.flush_write_map()
    assert f.read("c") == 3 and store.get("c") is not None


def test_public_signatures_accept_the_reference_parameter_names():
    """Every public function / method of the reference's python package can be called here with the reference's parameter
    NAMES in the reference's ORDER — keyword call sites in user code keep working."""
    import importlib
    import inspect

    allowed = {("bagua.torch_api.algorithms.gradient_allreduce", "GradientAllReduceAlgorithmImpl.init_operations")}   # the reference names it "_"
    problems, checked = [], 0
    for mod, api in sorted(_reference_api().items()):
        try:
            m = importlib.import_module(mod)
        except Exception:  # noqa: BLE001 - import gaps are the business of the tests above
            continue
        for name, ref in api["signatures"].items():
            obj = m
            for part in name.split("."):
                obj = getattr(obj, part, None)
                if obj is None:
                    break
            if obj is None or (mod, name) in allowed:
                continue
            try:
                params = list(inspect.signature(obj).parameters.values())
            except (TypeError, ValueError):
                continue
            ours = [p.name for p in params if p.name not in ("self", "cls")]
            takes_kwargs = any(p.kind == p.VAR_KEYWORD for p in params)
            missing = [a for a in ref if a not in ours and not takes_kwargs]
            positional = [p.name for p in params if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD) and p.name not in ("self", "cls")]
            if missing or [a for a in ref if a in positional] != [a for a in positional if a in ref]:
                problems.append(f"{mod}.{name}: reference {ref}, here {ours}")
            checked += 1
    assert not problems, problems
    assert checked > 150


def _mixed_bucket_worker(rank, world):
    import bagua_b200 as bagua
    from bagua_b200.bucket import BaguaBucket

    bagua.init_process_group()
    a = torch.zeros(4).ensure_bagua_tensor("a", "m")
    b = torch.zeros(4, dtype=torch.float16).ensure_bagua_tensor("b", "m")
    try:
        BaguaBucket([a, b], flatten=True, name="mixed")
    except ValueError as e:
        return "share one dtype" in str(e)
    return False


def test_a_bucket_rejects_mixed_dtypes_with_a_clear_message():
    """SURVEY appendix C: a bucket mixes tensors of one dtype only (the reference's backend rejects mixed dtype / device)."""
    assert all(run_distributed(_mixed_bucket_worker, world=1))
