"""Global-norm clipping of the sharded in-bucket optimizers (``max_grad_norm``) without a GPU: the fallback path (gloo all-reduce +
the flat optimizer) against torch, and the GPU-only driver (``init_operations`` / ``step()`` / ``clip_grad_norm_``) with host
doubles of the peer engine and of the native ops."""
import copy
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _flat, _net

BOUNDS = {"sgd": 6.5, "adamw": 8.0}   # between the smallest and the largest norm of the six steps


def _groups(m):
    return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 0.05},
            {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0, "lr": 5e-3}]


def _fallback_worker(rank, world, kind):
    BOUND = BOUNDS[kind]
    import torch.distributed as dist
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_sgd

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)
    if kind == "sgd":
        opt = make_sharded_fused_sgd(_groups(model), lr=0.1, momentum=0.9, max_grad_norm=BOUND)
        oopt = torch.optim.SGD(_groups(oracle), lr=0.1, momentum=0.9)
    else:
        opt = make_sharded_fused_adam(_groups(model), lr=1e-2, adamw=True, max_grad_norm=BOUND)
        oopt = torch.optim.AdamW(_groups(oracle), lr=1e-2)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    norms, want = [], []
    for it in range(6):
        x, y = _batch(rank, it)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        if it == 2:   # an explicit call replaces the clipping inside step() for this step
            norms.append(float(opt.clip_grad_norm_(BOUND)))
        opt.step()
        if it != 2:
            norms.append(float(opt.last_grad_norm))
        oopt.zero_grad()
        F.cross_entropy(oracle(x), y).backward()
        for p in oracle.parameters():
            dist.all_reduce(p.grad)
            p.grad /= world
        want.append(float(torch.nn.utils.clip_grad_norm_(oracle.parameters(), BOUND)))
        oopt.step()
    return _flat(model), _flat(oracle), norms, want


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_fallback_path_clips_like_torch(kind):
    BOUND = BOUNDS[kind]
    for mine, oracle, norms, want in run_distributed(_fallback_worker, world=2, args=(kind,)):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(torch.tensor(norms), torch.tensor(want), rtol=1e-5, atol=0)
        assert any(n > BOUND for n in want) and any(n <= BOUND for n in want), want   # some steps clip, some do not


def _host_double_worker(rank, world):
    """``init_operations`` and ``step()`` of the clipping path with doubles of the engine and of the four native ops."""
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_sgd
    from bagua_b200.utils.graph import GraphedTrainStep

    events = []

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

    class GradDouble:
        def __init__(self, *args):
            self.args = args

    class NormDouble:
        COEF = 0.25

        def __init__(self, comm, box, box_off, partials, nslots, extra, out):
            self.out_ptr, self.extra_ptr, self.max_norm = out, extra, None

        def set_max_norm(self, m):
            self.max_norm = m

        def run(self, opt):
            clip = opt._bucketing.clip
            assert clip["out"].data_ptr() == self.out_ptr and clip["extra"].data_ptr() == self.extra_ptr
            events.append(("norm", self.max_norm, float(clip["extra"])))
            clip["out"].copy_(torch.tensor([7.0, self.COEF]))

    class UpdateOp:
        def __init__(self, *args):
            self.args, self.hyper, self.s = args, None, 0

        def set_hyper(self, *a):
            self.hyper = a

        def steps(self):
            return self.s

        def set_steps(self, s):
            self.s = s

        def run(self, opt):
            events.append(("update", opt._bucketing.update_ops.index(self)))
            self.s += 1

    class BackendBucket:
        def __init__(self):
            self.ops = []

        def append_op(self, op):
            self.ops.append(op)

        def clear_ops(self):
            self.ops = []

    real_native = core.native()
    current = {}

    class FakeC:
        ShardGradOp, GradNormOp, ShardSgdOp, ShardAdamOp, AllReduceSgdOp = GradDouble, NormDouble, UpdateOp, UpdateOp, UpdateOp
        MAX_COMM_BLOCKS, MAX_PEERS = real_native.MAX_COMM_BLOCKS, real_native.MAX_PEERS

        def run_op(self, op, stream, device):
            op.run(current["opt"])

        def __getattr__(self, name):
            return getattr(real_native, name)

    def build(make, extra_param):
        torch.manual_seed(5)
        model = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.Flatten(), torch.nn.Linear(8 * 36, 5)).to(memory_format=torch.channels_last)
        want = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = make(list(model.parameters()), extra_param)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        impl._carry_state_over()
        for bucket in model.bagua_buckets:
            nbytes = bucket.backend_tensor.numel() * bucket.backend_tensor.element_size()
            bucket._engine = lambda group=None: Engine()
            bucket._slice = Slice(nbytes)
            bucket.backend_bucket = BackendBucket()
            impl.init_operations(ddp, bucket)
        current["opt"] = opt
        return model, opt, want

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        extra = torch.nn.Parameter(torch.randn(6))   # outside every bucket, like an MoE expert
        for make, keys in ((lambda ps, e: make_sharded_fused_sgd(ps + [e], lr=0.1, momentum=0.9, max_grad_norm=1.5), ("master", "momentum_buffer")),
                           (lambda ps, e: make_sharded_fused_adam([{"params": [p for p in ps if p.dim() > 1] + [e], "weight_decay": 0.1},
                                                                   {"params": [p for p in ps if p.dim() <= 1], "weight_decay": 0.0}],
                                                                  lr=0.01, adamw=True, max_grad_norm=1.5), ("master", "exp_avg", "exp_avg_sq"))):
            model, opt, want = build(make, extra)
            buckets = model.bagua_buckets
            # phase A is the whole bucket program; the update ops are the optimizer's, one per bucket in bucket order
            assert all(len(b.backend_bucket.ops) == 1 and isinstance(b.backend_bucket.ops[0], GradDouble) for b in buckets)
            assert all("_clip_" in b.allreduce_variant for b in buckets)
            bk = opt._bucketing
            assert len(bk.update_ops) == len(buckets) and all(isinstance(op, UpdateOp) and op.hyper is not None for op in bk.update_ops)
            partials = bk.clip["partials"]
            assert partials.shape == (len(buckets), FakeC.MAX_COMM_BLOCKS) and partials.dtype == torch.float64
            for i, b in enumerate(buckets):
                assert b.backend_bucket.ops[0].args[6] == partials[i].data_ptr()        # its own row of partial sums
                assert b.backend_bucket.ops[0].args[5] == bk.shards[i]["shard"].data_ptr()     # the shard phase B reads
                assert bk.update_ops[i].args[5] == bk.shards[i]["shard"].data_ptr()
                assert bk.update_ops[i].args[6] == bk.clip["out"][1:].data_ptr()     # coef
            for n, p in model.named_parameters():
                assert torch.equal(p.detach(), want[n])

            # step(): norm, then every phase B in bucket order, then the uncovered parameter with its gradient scaled by coef
            g = torch.randn(6)
            extra.grad = g.clone()
            before = extra.detach().clone()
            ref = torch.nn.Parameter(before.clone())
            ref.grad = g * NormDouble.COEF
            oref = (torch.optim.SGD([ref], lr=0.1, momentum=0.9) if keys[1] == "momentum_buffer" else
                    torch.optim.AdamW([ref], lr=0.01, weight_decay=0.1))
            oref.step()
            events.clear()
            launches = opt.kernel_launches
            opt.step()
            assert events[0] == ("norm", 1.5, pytest.approx(float(g.double().square().sum()), rel=1e-12))
            assert events[1:] == [("update", i) for i in range(len(buckets))]
            assert opt.kernel_launches == launches + 1 + len(buckets)
            torch.testing.assert_close(extra.detach(), ref.detach(), rtol=1e-6, atol=1e-7)
            assert float(opt.last_grad_norm) == 7.0

            # clip_grad_norm_ then step(): the norm is computed once, with the bound given to clip_grad_norm_
            extra.grad = g.clone()
            events.clear()
            total = opt.clip_grad_norm_(0.5)
            assert float(total) == 7.0
            opt.step()
            assert [e[0] for e in events] == ["norm"] + ["update"] * len(buckets) and events[0][1] == 0.5
            # a step without uncovered gradients resets their term
            extra.grad = None
            events.clear()
            opt.step()
            assert events[0] == ("norm", 1.5, 0.0)
            with pytest.raises(ValueError):
                opt.clip_grad_norm_(1.0, norm_type=float("inf"))
            with pytest.raises(NotImplementedError):
                GraphedTrainStep(model, lambda x: x.sum(), (torch.zeros(1),), optimizers=[opt])

            # checkpoints: the phase-B ops carry the step count; consolidated state round-trips
            opt._gather = lambda t, group: [t]
            sd = opt.state_dict()
            assert sd["steps"] == 3 and set(want) <= set(sd["state"])
            for n in want:
                assert all(sd["state"][n][k].shape == want[n].shape for k in keys)
            for rec in bk.shards:
                for t in rec["state"]:
                    t.add_(1.0)
                rec["step_ops"][0].set_steps(0)
            opt.load_state_dict(sd)
            again = opt.state_dict()
            assert again["steps"] == 3
            for n in want:
                for k in keys:
                    assert torch.equal(again["state"][n][k], sd["state"][n][k])

        # no bound configured, bucket ops live: clip_grad_norm_ would read consumed gradients -> refuse
        model, opt, _ = build(lambda ps, e: make_sharded_fused_sgd(ps, lr=0.1), extra)
        assert opt._bucketing.clip is None and all(not isinstance(b.backend_bucket.ops[0], GradDouble) for b in model.bagua_buckets)
        with pytest.raises(RuntimeError, match="max_grad_norm"):
            opt.clip_grad_norm_(1.0)
        with pytest.raises(ValueError):
            make_sharded_fused_adam(list(model.parameters()), max_grad_norm=0.0)
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_clipping_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))
