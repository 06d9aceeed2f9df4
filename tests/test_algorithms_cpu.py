"""Algorithms end to end on CPU/gloo with world_size 2 (the BASELINE 'plumbing' config) against python oracles —
same strategy as the reference's tests (SURVEY §4): a torch re-implementation of each algorithm is the executable spec."""
import copy
import os

import pytest
import torch

from tests.mp_utils import run_distributed


def _net():
    import torch.nn as nn

    return nn.Sequential(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.Flatten(), nn.Linear(4 * 26 * 26, 10))


def _batch(rank, it):
    g = torch.Generator().manual_seed(1000 * rank + it)
    return torch.randn(4, 1, 28, 28, generator=g), torch.randint(0, 10, (4,), generator=g)


def _train(model, opt, rank, steps, post=None):
    import torch.nn.functional as F

    for it in range(steps):
        x, y = _batch(rank, it)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        if post is not None:
            post(it)
        opt.step()


def _flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()]).clone()


# ---- gradient allreduce ------------------------------------------------------------------------------------------------
def _grad_allreduce_worker(rank, world):
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms import gradient_allreduce

    bagua.init_process_group()
    torch.manual_seed(rank)  # different init per rank: broadcast from rank 0 must fix it
    model = _net()
    oracle = copy.deepcopy(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
    model = model.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    # oracle: rank-0 weights + manual gradient averaging with plain torch.distributed
    for p in oracle.parameters():
        dist.broadcast(p.data, 0)
    oopt = torch.optim.SGD(oracle.parameters(), lr=0.05, momentum=0.9)

    def avg(_it):
        for p in oracle.parameters():
            dist.all_reduce(p.grad)
            p.grad /= world

    model.bagua_ddp.comm_profile(True)
    _train(model, opt, rank, 6)
    _train(oracle, oopt, rank, 6, post=avg)
    assert len(model.bagua_buckets) >= 1 and all(b.check_flatten() for b in model.bagua_buckets)
    report = model.bagua_ddp.comm_report()
    assert len(report) == len(model.bagua_buckets) and all(r["launches"] == 6 and r["mean_ms"] > 0 and r["bytes"] > 0 for r in report), report
    return _flat(model), _flat(oracle)


def test_gradient_allreduce_matches_oracle():
    res = run_distributed(_grad_allreduce_worker, world=2)
    for mine, oracle in res:
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
    assert torch.equal(res[0][0], res[1][0])  # replicas bit-identical


# ---- every algorithm runs, stays finite, can be switched on the same module ---------------------------------------
def _all_algorithms_worker(rank, world):
    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms import Algorithm, q_adam

    bagua.init_process_group()
    torch.manual_seed(0)
    model = _net()
    out = {}
    for name in ["gradient_allreduce", "bytegrad", "decentralized", "low_precision_decentralized", "qadam", "async", "gradient_allreduce"]:
        if name == "qadam":
            opt = q_adam.QAdamOptimizer(model.parameters(), lr=1e-3, warmup_steps=2)
            algo = q_adam.QAdamAlgorithm(opt)
        else:
            opt = torch.optim.SGD(model.parameters(), lr=0.01)
            algo = Algorithm.init(name, **({"sync_interval_ms": 10} if name == "async" else {}))
        model = model.with_bagua([opt], algo)  # re-invoking with_bagua switches the algorithm
        # what is communicated must follow the algorithm: gradients (or QAdam's first moment) for the centralized families, the WEIGHTS
        # for decentralized / async — a re-registration replaces the getter closures, None meaning "the tensor itself"
        for p in model.parameters():
            eff = p.bagua_getter_closure()
            if name in ("decentralized", "low_precision_decentralized", "async"):
                assert eff.data_ptr() == p.data_ptr(), (name, "weight algorithms must communicate the weights, not stale gradient views")
            elif name != "qadam":
                assert p.grad is not None and eff.data_ptr() == p.grad.data_ptr(), name
        _train(model, opt, rank, 5)
        if name == "async":
            model.bagua_algorithm.abort(model)
        f = _flat(model)
        assert torch.isfinite(f).all(), name
        out[name] = f
    return out


def test_all_algorithms_and_switching():
    res = run_distributed(_all_algorithms_worker, world=2, timeout=400)
    assert torch.equal(res[0]["gradient_allreduce"], res[1]["gradient_allreduce"])
    # decentralized averaging must actually have mixed the replicas' weights (it would not if it exchanged gradient buffers): after the
    # average of the last step the replicas are one local SGD update apart
    assert (res[0]["decentralized"] - res[1]["decentralized"]).abs().max().item() < 0.05


# ---- decentralized: oracle as in the reference's tests/torch_api/test_decentralized.py ------------------------------
def _decentralized_worker(rank, world, mode, interval):
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.core import native
    from bagua_b200.parallel.algorithms import decentralized

    bagua.init_process_group()
    torch.manual_seed(42)
    model = _net()
    oracle = copy.deepcopy(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    oopt = torch.optim.SGD(oracle.parameters(), lr=0.05)
    model = model.with_bagua([opt], decentralized.DecentralizedAlgorithm(hierarchical=False, peer_selection_mode=mode, communication_interval=interval))
    import torch.nn.functional as F

    comm_step = 0
    for it in range(6):
        x, y = _batch(rank, it)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        opt.step()
        # oracle: average the weights as they were at the start of the iteration, then apply the local gradient step
        oopt.zero_grad()
        w0 = [p.detach().clone() for p in oracle.parameters()]
        F.cross_entropy(oracle(x), y).backward()
        if it % interval == 0:
            for p, w in zip(oracle.parameters(), w0):
                if mode == "all":
                    avg = w.clone()
                    dist.all_reduce(avg)
                    avg /= world
                else:
                    peer = native().PeerAverageOp.shift_one_peer(rank, world, comm_step)
                    other = torch.empty_like(w)
                    reqs = [dist.isend(w.clone(), peer), dist.irecv(other, peer)]
                    for r in reqs:
                        r.wait()
                    avg = (w + other) / 2
                p.data.copy_(avg)
            comm_step += 1
        oopt.step()
    return _flat(model), _flat(oracle)


@pytest.mark.parametrize("mode,interval", [("all", 1), ("shift_one", 1), ("all", 2)])
def test_decentralized_matches_oracle(mode, interval):
    for mine, oracle in run_distributed(_decentralized_worker, world=2, args=(mode, interval)):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)


# ---- low precision decentralized: oracle = reference python (tests/torch_api/test_low_precision_decentralized.py:218-240) ----
def _lpd_worker(rank, world):
    import torch.distributed as dist
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.ops import quant
    from bagua_b200.parallel.algorithms import decentralized

    bagua.init_process_group()
    torch.manual_seed(7)
    model = _net()
    oracle = copy.deepcopy(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    oopt = torch.optim.SGD(oracle.parameters(), lr=0.05)
    model = model.with_bagua([opt], decentralized.LowPrecisionDecentralizedAlgorithm(hierarchical=False))
    ow = _flat(oracle)
    W, L, R = ow.clone(), ow.clone(), ow.clone()
    n_pad = (-ow.numel()) % 32
    for it in range(4):
        x, y = _batch(rank, it)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        opt.step()
        oopt.zero_grad()
        F.cross_entropy(oracle(x), y).backward()
        oopt.step()
        xf = _flat(oracle)
        xf = xf + (1 / 3) * L
        xf = xf + (1 / 3) * R
        xf = xf - (5 / 3) * W
        pad = torch.cat([xf, torch.zeros(n_pad)])  # the bucket is padded to 32 elements with zeros
        mm, q = quant.torch_compress_chunk(pad)
        lp, rp = (rank + world - 1) % world, (rank + 1) % world
        ql, qr, ml, mr = torch.empty_like(q), torch.empty_like(q), torch.empty_like(mm), torch.empty_like(mm)
        reqs = [dist.isend(q, lp), dist.isend(q, rp), dist.irecv(ql, lp), dist.irecv(qr, rp)]
        for r in reqs:
            r.wait()
        reqs = [dist.isend(mm, lp), dist.isend(mm, rp), dist.irecv(ml, lp), dist.irecv(mr, rp)]
        for r in reqs:
            r.wait()
        n = xf.numel()
        L += quant.torch_decompress_chunk(ml, ql, torch.float32)[:n]
        R += quant.torch_decompress_chunk(mr, qr, torch.float32)[:n]
        new = W + quant.torch_decompress_chunk(mm, q, torch.float32)[:n]
        W = new.clone()
        off = 0
        for p in oracle.parameters():
            p.data.copy_(new[off : off + p.numel()].view_as(p))
            off += p.numel()
    return _flat(model), _flat(oracle)


def test_low_precision_decentralized_matches_oracle():
    for mine, oracle in run_distributed(_lpd_worker, world=2):
        # single bucket in both: identical quantisation chunks → agreement up to rare one-level flips caused by
        # fused-multiply-add vs two-rounding evaluation of x + L/3 (one level = range/255 of the *difference* tensor)
        assert ((mine - oracle).abs() > 1e-5).float().mean().item() < 1e-3
        torch.testing.assert_close(mine, oracle, rtol=0, atol=2e-3)


# ---- bytegrad fallback pipeline: bounded quantisation error w.r.t. the exact average ---------------------------------
def _bytegrad_worker(rank, world):
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.ops import quant

    bagua.init_process_group()
    pg = bagua.communication._get_default_group()

    class FakeBucket:
        def __init__(self, t):
            self.t = t

        def _flat_or_gather(self):
            return self.t, None

    torch.manual_seed(rank)
    x = torch.randn(2 * 64)
    exact = x.clone()
    dist.all_reduce(exact)
    exact /= world
    y = x.clone()
    quant.bytegrad_allreduce_fallback(FakeBucket(y), pg, True)
    gathered = [torch.empty_like(y) for _ in range(world)]
    dist.all_gather(gathered, y)
    assert all(torch.equal(gathered[0], g) for g in gathered)  # every rank decodes the same bytes
    return (y - exact).abs().max().item(), (x.max() - x.min()).item()


def test_bytegrad_pipeline_error_bound():
    for err, rng in run_distributed(_bytegrad_worker, world=2):
        assert err <= 2.0 * rng / 255


# ---- no_sync / DDP wrapper / broadcast of optimizer state ---------------------------------------------------------
def _ddp_wrapper_worker(rank, world):
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.parallel.data_parallel import DistributedDataParallel

    bagua.init_process_group()
    torch.manual_seed(rank)
    model = _net()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    # give rank 0 some optimizer state that must be broadcast
    if rank == 0:
        x, y = _batch(0, 99)
        F.cross_entropy(model(x), y).backward()
        opt.step()
        opt.zero_grad()
    else:
        for p in model.parameters():
            p.grad = torch.zeros_like(p)
        opt.step()
        opt.zero_grad()
    ddp = DistributedDataParallel(model, optimizers=[opt])
    state = torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in model.parameters()]).clone()
    with ddp.no_sync():
        x, y = _batch(rank, 0)
        F.cross_entropy(ddp(x), y).backward()
    local_grad = torch.cat([p.grad.reshape(-1) for p in model.parameters()]).clone()
    x, y = _batch(rank, 1)
    F.cross_entropy(ddp(x), y).backward()  # accumulates on top and synchronises
    synced = torch.cat([p.grad.reshape(-1) for p in model.parameters()]).clone()
    return _flat(model), state, local_grad, synced


def test_ddp_wrapper_no_sync_and_state_broadcast():
    r0, r1 = run_distributed(_ddp_wrapper_worker, world=2)
    assert torch.equal(r0[0], r1[0]) and torch.equal(r0[1], r1[1])  # params and Adam state broadcast from rank 0
    assert not torch.equal(r0[2], r1[2])                             # no_sync kept gradients local
    torch.testing.assert_close(r0[3], r1[3])                          # after the sync step both hold the average


# ---- fused allreduce+SGD algorithm: CPU/gloo fallback (plain allreduce + FusedSGD torch path) -------------------------
def _fused_fallback_worker(rank, world, kind="sgd"):
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_sgd

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)
    if kind == "sgd":
        opt = make_sharded_fused_sgd(model.parameters(), lr=0.05, momentum=0.9)
        oopt = torch.optim.SGD(oracle.parameters(), lr=0.05, momentum=0.9)
    else:
        opt = make_sharded_fused_adam(model.parameters(), lr=1e-2, weight_decay=0.01, adamw=True)
        oopt = torch.optim.AdamW(oracle.parameters(), lr=1e-2, weight_decay=0.01)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))

    def avg(_it):
        for p in oracle.parameters():
            dist.all_reduce(p.grad)
            p.grad /= world

    _train(model, opt, rank, 4)
    _train(oracle, oopt, rank, 4, post=avg)
    return _flat(model), _flat(oracle)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_fused_allreduce_sgd_cpu_fallback(kind):
    for mine, oracle in run_distributed(_fused_fallback_worker, world=2, args=(kind,)):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)


# ---- the same scenarios with the C++ autograd hooks (csrc/torch_hooks, BAGUA_NATIVE_HOOKS=1) ----------------------------------
def _native_hooks_worker(rank, world):
    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms import bytegrad, gradient_allreduce

    assert os.environ.get("BAGUA_NATIVE_HOOKS") == "1"
    mine, oracle = _grad_allreduce_worker(rank, world)               # oracle equality + comm_report with native hooks
    torch.manual_seed(rank)
    model = _net()
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    model = model.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    n_native = len(model.bagua_ddp._native_hooked)
    _train(model, opt, rank, 2)
    model = model.with_bagua([opt], bytegrad.ByteGradAlgorithm())    # switching algorithms re-installs the hooks on new buckets
    _train(model, opt, rank, 2)
    model.bagua_ddp._reset_buckets()                                  # what the autotuner does: new buckets, same algorithm
    _train(model, opt, rank, 2)
    return mine, oracle, n_native, len(model.bagua_ddp._native_hooked), _flat(model)


def test_native_autograd_hooks_match_python_hooks():
    from bagua_b200 import _build

    try:
        _build.build_torch_hooks()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"torch hooks extension cannot be built here: {e}")
    res = run_distributed(_native_hooks_worker, world=2, extra_env={"BAGUA_NATIVE_HOOKS": "1"}, timeout=300)
    for mine, oracle, n0, n1, _ in res:
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        assert n0 == 4 and n1 == 4                                    # every parameter of the net got a native hook, also after re-bucketing
    assert torch.equal(res[0][4], res[1][4])
    r0, r1 = run_distributed(_ddp_wrapper_worker, world=2, extra_env={"BAGUA_NATIVE_HOOKS": "1"})
    assert torch.equal(r0[0], r1[0]) and not torch.equal(r0[2], r1[2])   # no_sync() disables the native hooks too
    torch.testing.assert_close(r0[3], r1[3])


def test_in_bucket_optimizers_also_update_parameters_outside_the_buckets():
    """MoE experts and ignored parameters are not part of any bucket, so no bucket kernel updates them: the sharded optimizers'
    ``step()`` applies the ordinary update to exactly those parameters (and clears their gradients), and leaves the
    bucketed ones to the kernels."""
    import torch

    from bagua_b200.parallel.algorithms.gradient_allreduce import make_sharded_fused_adam, make_sharded_fused_sgd

    class Op:
        def set_hyper(self, *a):
            self.hyper = a

        def steps(self):
            return 0

    for make, ref_cls, kw in ((make_sharded_fused_sgd, torch.optim.SGD, dict(lr=0.1, momentum=0.9)),
                              (lambda ps, **k: make_sharded_fused_adam(ps, adamw=True, **k), torch.optim.AdamW, dict(lr=0.01, weight_decay=0.01))):
        torch.manual_seed(0)
        bucketed, expert = torch.nn.Parameter(torch.randn(5)), torch.nn.Parameter(torch.randn(3, 4))
        ref = torch.nn.Parameter(expert.detach().clone())
        opt = make([bucketed, expert], **kw)
        ropt = ref_cls([ref], **kw)
        opt._bucketing.hyper_ops, opt._bucketing.covered = [(Op(), 0)], {id(bucketed)}     # what FusedGradientAllReduceAlgorithm sets up on a GPU box
        before = bucketed.detach().clone()
        for _ in range(3):
            g = torch.randn(3, 4)
            bucketed.grad, expert.grad, ref.grad = torch.ones(5), g.clone(), g.clone()
            opt.step()
            ropt.step()
            assert float(expert.grad.abs().sum()) == 0.0          # cleared like the bucketed gradients
            assert torch.equal(bucketed.grad, torch.ones(5))      # the kernel's business, not step()'s
        torch.testing.assert_close(expert.detach(), ref.detach(), rtol=1e-5, atol=1e-6)
        assert torch.equal(bucketed.detach(), before)
        # the expert's optimizer state is part of the (otherwise shard-derived) checkpoint
        opt._bucketing.shards = [{"state": (), "group": None, "numel": 0, "layout": [], "lo": 0, "hi": 0, "step_ops": (Op(),), "weights": None}]
        sd = opt.state_dict()
        assert sd["sharded_fused"] and len(sd["uncovered"]["state"]) == 1
        opt2 = make([torch.nn.Parameter(bucketed.detach().clone()), torch.nn.Parameter(expert.detach().clone())], **kw)
        opt2.load_state_dict(sd)
        loaded = list(opt2.state.values())
        assert len(loaded) == 1 and all(torch.equal(v, list(opt.state.values())[0][k]) for k, v in loaded[0].items() if isinstance(v, torch.Tensor))


def _fused_two_groups_worker(rank, world):
    """Weight decay on the matrices, none on the biases — two parameter groups: the fused algorithm cuts every bucket into
    single-group pieces (one bucket kernel applies one set of hyper-parameters) and training equals torch AdamW with the same
    groups on averaged gradients."""
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)

    def groups(m):
        decay = [p for p in m.parameters() if p.dim() > 1]
        rest = [p for p in m.parameters() if p.dim() <= 1]
        return [{"params": decay, "weight_decay": 0.05}, {"params": rest, "weight_decay": 0.0, "lr": 5e-3}]

    opt = make_sharded_fused_adam(groups(model), lr=1e-2, adamw=True)
    oopt = torch.optim.AdamW(groups(oracle), lr=1e-2)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    group_of = {id(p): gi for gi, g in enumerate(opt.param_groups) for p in g["params"]}
    names = []
    for b in model.bagua_buckets:
        kinds = {group_of[id(t)] for t in b.tensors if not t.bagua_tensor_name.startswith("bagua_padding_tensor")}
        assert len(kinds) == 1 and b.name.endswith(f".g{kinds.pop()}")
        names.append(b.name)

    def avg(_it):
        for p in oracle.parameters():
            dist.all_reduce(p.grad)
            p.grad /= world

    _train(model, opt, rank, 4)
    _train(oracle, oopt, rank, 4, post=avg)
    return _flat(model), _flat(oracle), names


def test_fused_algorithm_splits_buckets_by_parameter_group():
    for mine, oracle, names in run_distributed(_fused_two_groups_worker, world=2):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        assert len(names) >= 2 and any(n.endswith(".g0") for n in names) and any(n.endswith(".g1") for n in names)


def _fused_init_operations_worker(rank, world):
    """``FusedGradientAllReduceAlgorithmImpl.init_operations`` — the code that builds the in-bucket optimizer on a GPU box
    (weights re-pointed into a symmetric slice, fp32 master shard, op construction, shard bookkeeping) — run on the host with
    doubles of the peer engine and of the two native op classes: parameters keep their values, the recorded layout addresses
    the right elements (consolidated ``master`` == the weights), ``state_dict`` / ``load_state_dict`` round-trip."""
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_sgd

    class Slice:
        has_multicast = False
        buf, offset = object(), 0

        def __init__(self, nbytes):
            self.tensor = torch.zeros(nbytes, dtype=torch.uint8)

        def view(self, dtype, numel):
            return self.tensor.view(dtype)[:numel]

        def free(self):
            pass

    class Engine:
        has_multicast, comm = False, object()

        def alloc(self, nbytes):
            return Slice(nbytes)

        def launch_cfg(self, variant, nbytes, blocks=0):
            return ("cfg", variant, blocks)

    class Op:
        def __init__(self, *args):
            self.args, self.hyper, self.s = args, None, 0

        def set_hyper(self, *a):
            self.hyper = a

        def steps(self):
            return self.s

        def set_steps(self, s):
            self.s = s

    class SgdOp(Op):
        pass

    class AdamOp(Op):
        pass

    class BackendBucket:
        def __init__(self):
            self.ops = []

        def append_op(self, op):
            self.ops.append(op)

        def clear_ops(self):
            self.ops = []

    real_native = core.native()

    class FakeC:
        AllReduceSgdOp, AllReduceAdamOp = SgdOp, AdamOp

        def __getattr__(self, name):
            return getattr(real_native, name)

    bagua.init_process_group()
    for make, op_cls, keys in ((lambda ps: make_sharded_fused_sgd(ps, lr=0.1, momentum=0.9), SgdOp, ("master", "momentum_buffer")),
                               (lambda ps: make_sharded_fused_adam([{"params": [p for p in ps if p.dim() > 1], "weight_decay": 0.1},
                                                                    {"params": [p for p in ps if p.dim() <= 1], "weight_decay": 0.0}], lr=0.01, adamw=True),
                                AdamOp, ("master", "exp_avg", "exp_avg_sq"))):
        torch.manual_seed(5)
        model = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.Flatten(), torch.nn.Linear(8 * 36, 5)).to(memory_format=torch.channels_last)
        want = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = make(list(model.parameters()))
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        core_native = core.native
        core.native = lambda: FakeC()
        try:
            for bucket in model.bagua_buckets:
                nbytes = bucket.backend_tensor.numel() * bucket.backend_tensor.element_size()
                bucket._engine = lambda group=None: Engine()
                bucket._slice = Slice(nbytes)
                bucket.backend_bucket = BackendBucket()
                impl.init_operations(ddp, bucket)
                assert isinstance(bucket.backend_bucket.ops[0], op_cls) and bucket.allreduce_variant.endswith("two_shot")
        finally:
            core.native = core_native
        bk = opt._bucketing
        assert len(bk.hyper_ops) == len(model.bagua_buckets) == len(bk.shards) and opt.collective_state_dict
        assert all(op.hyper is not None for op, _ in bk.hyper_ops)
        if op_cls is AdamOp:   # every bucket op follows the weight decay of ITS parameter group
            decays = {group_index: op.hyper[4] for op, group_index in bk.hyper_ops}
            assert decays == {0: 0.1, 1: 0.0}, decays
        for n, p in model.named_parameters():   # weights now live in the "symmetric" slices, values and memory format unchanged
            assert torch.equal(p.detach(), want[n]) and p.stride() == want[n].stride()
        opt._gather = lambda t, group: [t]      # world size 1: the all-gather is the identity
        sd = opt.state_dict()
        assert set(sd["state"]) == set(want)
        for n in want:
            torch.testing.assert_close(sd["state"][n]["master"], want[n].contiguous())
            assert all(sd["state"][n][k].shape == want[n].shape for k in keys)
        for rec in bk.shards:                  # perturb, restore, compare
            for t in rec["state"]:
                t.add_(1.0)
        opt.load_state_dict(sd)
        again = opt.state_dict()
        for n in want:
            for k in keys:
                assert torch.equal(again["state"][n][k], sd["state"][n][k])
    return True


def test_fused_init_operations_with_host_doubles():
    assert all(run_distributed(_fused_init_operations_worker, world=1))


def _hier_branch_worker(rank, world):
    """The multi-node branch of ``append_centralized_synchronous_op`` (NVLink reduce-scatter kernel → rail all-reduce of this
    rank's slice → NVLink all-gather kernel) with doubles of the intra-node engine and the two native ops that EXECUTE their
    contract through gloo: 4 ranks posing as 2 nodes × 2 GPUs must end with the global average in every bucket."""
    import torch.distributed as dist

    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.bucket import BaguaBucket

    bagua.init_process_group()
    pg = bagua.communication._get_default_group()
    L, nodes = 2, world // 2
    node, local = rank // L, rank % L
    intra = [dist.new_group([n * L + i for i in range(L)]) for n in range(nodes)][node]
    rail = [dist.new_group([n * L + i for n in range(nodes)]) for i in range(L)][local]
    ran = []

    class Slice:
        has_multicast, buf, offset = False, object(), 0

    class IntraEngine:
        has_multicast, comm, rank = False, object(), local

        def launch_cfg(self, variant, nbytes, blocks=0):
            return None

    flat_holder = {}

    class RS:   # contract of reduce_scatter_kernel: my 1/L slice of the buffer becomes scale × sum over the node
        def __init__(self, comm, buf, off, nbytes, dtype, scale, use_mc, cfg):
            self.nbytes, self.scale = nbytes, scale

        def run(self):
            flat = flat_holder["flat"]
            tmp = flat.clone()
            dist.all_reduce(tmp, group=intra)
            es = flat.element_size()
            vpr = (self.nbytes // 16 + L - 1) // L
            lo, hi = local * vpr * 16 // es, min((local + 1) * vpr * 16, self.nbytes) // es
            flat[lo:hi] = tmp[lo:hi] * self.scale
            ran.append("rs")

    class AG:   # contract of all_gather_kernel: every rank of the node receives every slice
        def __init__(self, comm, buf, off, nbytes, dtype, use_mc, cfg):
            self.nbytes = nbytes

        def run(self):
            flat = flat_holder["flat"]
            es = flat.element_size()
            vpr = (self.nbytes // 16 + L - 1) // L
            for src in range(L):
                lo, hi = src * vpr * 16 // es, min((src + 1) * vpr * 16, self.nbytes) // es
                if hi > lo:
                    piece = flat[lo:hi].clone()
                    dist.broadcast(piece, node * L + src, group=intra)
                    flat[lo:hi] = piece
            ran.append("ag")

    class BackendBucket:
        def __init__(self):
            self.ops = []

        def append_op(self, op):
            self.ops.append(("native", op))

        def append_python_op(self, fn, label="python"):
            self.ops.append(("python", fn))

        def clear_ops(self):
            self.ops = []

    real_native = core.native()

    class FakeC:
        ReduceScatterOp, AllGatherOp = RS, AG

        def __getattr__(self, name):
            return getattr(real_native, name)

    torch.manual_seed(rank)
    ts = [torch.randn(37).ensure_bagua_tensor("a", "hier"), torch.randn(3, 9).ensure_bagua_tensor("b", "hier")]
    want = torch.cat([t.reshape(-1).clone() for t in ts])
    dist.all_reduce(want)
    want /= world
    bucket = BaguaBucket(ts, "h", flatten=True, alignment=4)
    flat_holder["flat"] = bucket.backend_tensor
    bucket._slice = Slice()
    bucket.backend_bucket = BackendBucket()
    pg.nnodes = nodes
    pg.hier_engine = lambda: (IntraEngine(), rail, L, nodes)
    bucket._engine = lambda group=None: None
    core_native, core.native = core.native, (lambda: FakeC())
    import bagua_b200.bucket as bucket_mod

    bucket_native, bucket_mod.native = bucket_mod.native, (lambda: FakeC())
    try:
        bucket.append_centralized_synchronous_op(hierarchical=True, average=True)
    finally:
        core.native, bucket_mod.native = core_native, bucket_native
    kinds = [k for k, _ in bucket.backend_bucket.ops]
    assert kinds == ["native", "python", "native"] and bucket.allreduce_variant.startswith("hier:"), (kinds, bucket.allreduce_variant)
    for kind, op in bucket.backend_bucket.ops:
        op.run() if kind == "native" else op("h")
    got = torch.cat([t.reshape(-1) for t in ts])
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)
    return ran


def test_hierarchical_bucket_program_with_executing_doubles():
    for ran in run_distributed(_hier_branch_worker, world=4):
        assert ran == ["rs", "ag"]


def _inline_switch_worker(rank, world):
    mine, oracle = _grad_allreduce_worker(rank, world)
    import bagua_b200 as bagua  # noqa: F401
    from bagua_b200 import communication as comm_mod

    backends = list(comm_mod._backends.values())
    # gloo bucket programs are python ops: the switch is on, yet everything still goes through the worker thread
    return mine, oracle, [b.inline_mode() for b in backends], sum(b.inline_total() for b in backends)


def test_inline_comm_switch_is_harmless_for_python_bucket_programs():
    for mine, oracle, modes, inlined in run_distributed(_inline_switch_worker, world=2, extra_env={"BAGUA_INLINE_COMM": "1"}):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        assert modes and all(modes) and inlined == 0
