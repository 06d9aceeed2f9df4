"""Loss scaling of the sharded in-bucket optimizers without a GPU: on the fallback path (gloo all-reduce + the flat optimizer)
``ShardedGradScaler`` is ``torch.amp.GradScaler``; and the GPU-only driver (``init_operations`` / ``step()`` / the scaler's live
path) with host doubles of the peer engine and the native ops: program, variants, launch count, the hand-over of the scale, the
vote recorded for ``update()``, the error cases, and the step count ``t`` through checkpoints and re-bucketing."""
import copy
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _flat, _net


def _fallback_worker(rank, world):
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.ops.optim import FusedAdam
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)
    opt = make_sharded_fused_adam(model.parameters(), lr=1e-2, adamw=True, max_grad_norm=2.0, loss_scaling=True)
    oopt = FusedAdam(oracle.parameters(), lr=1e-2, adamw=True)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    assert not opt._bucketing.hyper_ops and opt.last_step_skipped is None     # no peer engine: the flat path
    scaler = ShardedGradScaler(init_scale=2.0 ** 8, growth_interval=2, device="cpu")
    oscaler = torch.amp.GradScaler("cpu", init_scale=2.0 ** 8, growth_interval=2)
    scales = []
    for it in range(6):
        x, y = _batch(rank, it)
        opt.zero_grad()
        scaler.scale(F.cross_entropy(model(x), y)).backward()
        if it in (1, 4):                   # an overflow in the all-reduced gradient, which every rank holds
            next(model.parameters()).grad.view(-1)[0] = float("inf")
        scaler.step(opt)                   # torch's unscale → check → step; step() clips the unscaled gradients (max_grad_norm)
        scaler.update()
        xs, ys = zip(*[_batch(r, it) for r in range(world)])
        oopt.zero_grad()
        oscaler.scale(F.cross_entropy(oracle(torch.cat(xs)), torch.cat(ys))).backward()
        if it in (1, 4):
            next(oracle.parameters()).grad.view(-1)[0] = float("inf")
        oscaler.unscale_(oopt)
        torch.nn.utils.clip_grad_norm_(oracle.parameters(), 2.0)
        oscaler.step(oopt)
        oscaler.update()
        scales.append((scaler.get_scale(), oscaler.get_scale()))
    assert scaler.state_dict() == oscaler.state_dict()
    return _flat(model), _flat(oracle), scales


def test_fallback_path_is_torch_grad_scaler():
    for mine, oracle, scales in run_distributed(_fallback_worker, world=2):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        assert all(a == b for a, b in scales) and [a for a, _ in scales] == [256.0, 128.0, 128.0, 256.0, 128.0, 128.0], scales


def _host_double_worker(rank, world):
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.parallel.algorithms.gradient_allreduce import (FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_lamb,
                                                                  make_sharded_fused_sgd)
    from bagua_b200.utils.graph import GraphedTrainStep

    events, current = [], {}

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
        name = "op"

        def __init__(self, *args):
            self.args, self.hyper, self.s, self.dev = args, None, 0, None

        def set_hyper(self, *a):
            self.hyper = a

        def steps(self):
            return self.s

        def set_steps(self, s):
            self.s = s

        def set_max_norm(self, m):
            self.max_norm = m

        def set_scale_ptr(self, p):
            self.scale_ptr = p

        def set_device_step(self, vote, step):
            self.dev = (vote, step)

        def run(self, opt):
            events.append(self.name)
            self.s += 1

    class Ratio(Op):
        name = "ratio"

        @staticmethod
        def box_bytes(n):
            return 2 * 8 * n * 16

    class ScaledNorm(Op):
        name = "scaled_norm"

        def run(self, opt):    # the double of loss_scale_norm_kernel: the test plants the vote in current["overflow"]
            events.append(self.name)
            clip = opt._bucketing.clip
            assert self.scale_ptr == (clip["unit"] if opt._loss_scale is None else opt._loss_scale).data_ptr()
            found = bool(current.get("overflow"))
            clip["out"].copy_(torch.tensor([float("inf") if found else 3.0, 0.25, float(found)]))
            clip["t"] += 0 if found else 1

    def kinds(name):
        return type(name.capitalize(), (Op,), {"name": name})

    class BackendBucket:
        def __init__(self):
            self.ops = []

        def append_op(self, op):
            self.ops.append(op)

        def clear_ops(self):
            self.ops = []

    real_native = core.native()

    class FakeC:
        ShardGradOp, GradNormOp, LossScaleNormOp, LambRatioOp = kinds("phase_a"), kinds("norm"), ScaledNorm, Ratio
        LambMomentsOp, ShardLambOp, ShardAdamOp, ShardSgdOp = kinds("moments"), kinds("apply"), kinds("adam"), kinds("sgd")
        AllReduceAdamOp, AllReduceSgdOp = kinds("fused_adam"), kinds("fused_sgd")
        MAX_COMM_BLOCKS, MAX_PEERS = real_native.MAX_COMM_BLOCKS, real_native.MAX_PEERS

        def run_op(self, op, stream, device):
            op.run(current["opt"])

        def __getattr__(self, name):
            return getattr(real_native, name)

    class Group:
        def size(self):
            return 1

        def rank(self):
            return 0

    def build(make, state=None):
        torch.manual_seed(5)
        model = torch.nn.Sequential(torch.nn.Linear(12, 8), torch.nn.Tanh(), torch.nn.Linear(8, 5))
        opt = make(list(model.parameters()))
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        impl.process_group = Group()
        impl._carry_state_over()
        if state is not None:
            opt.load_state_dict(state)
        rebucket(model, opt)
        return model, opt

    def rebucket(model, opt):
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        impl._carry_state_over()
        for bucket in model.bagua_buckets:
            bucket._engine = lambda group=None: Engine()
            bucket._slice = Slice(bucket.backend_tensor.numel() * bucket.backend_tensor.element_size())
            bucket.backend_bucket = BackendBucket()
            impl.init_operations(ddp, bucket)
        opt._pending_state = None
        opt._gather = lambda t, group: [t]
        current["opt"] = opt

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        makes = {"sgd": lambda ps, **kw: make_sharded_fused_sgd(ps, lr=0.1, momentum=0.9, **kw),
                 "adam": lambda ps, **kw: make_sharded_fused_adam(ps, lr=0.01, adamw=True, **kw),
                 "lamb": lambda ps, **kw: make_sharded_fused_lamb(ps, lr=0.01, **kw)}
        for kind, make in makes.items():
            for bound in (None, 1.5):
                # without the argument: the programs and variants of today
                model, opt = build(lambda ps: make(ps, max_grad_norm=bound))
                two_phase = bound is not None or kind == "lamb"
                want = f"fused_{kind}_" + ("clip_" if bound else "")
                assert all(b.allreduce_variant == want + "two_shot" for b in model.bagua_buckets)
                assert all(b.backend_bucket.ops[0].name == ("phase_a" if two_phase else f"fused_{kind}") for b in model.bagua_buckets)
                assert not opt.native_ops_in_step == (not two_phase) and opt.last_step_skipped is None
                assert all(op.dev is None for rec in opt._bucketing.shards for op in rec["step_ops"])
                if bound:
                    assert opt._bucketing.clip["out"].numel() == 2 and "t" not in opt._bucketing.clip
                with pytest.raises(RuntimeError, match="loss_scaling=True"):
                    scaler = ShardedGradScaler(device="cpu")
                    scaler.scale(torch.zeros(1))
                    scaler.step(opt)
                with pytest.raises(RuntimeError, match="without loss_scaling"):
                    opt.set_loss_scale(torch.ones(1))

                # with it: phase A in the bucket program, one exchange, every stepped op reads the vote and t from device memory
                model, opt = build(lambda ps: make(ps, max_grad_norm=bound, loss_scaling=True))
                buckets, bk = model.bagua_buckets, opt._bucketing
                nb = len(buckets)
                assert all(b.allreduce_variant == f"fused_{kind}_scaled_" + ("clip_" if bound else "") + "two_shot" for b in buckets)
                assert all([o.name for o in b.backend_bucket.ops] == ["phase_a"] for b in buckets)
                vote, tptr = bk.clip["out"][1:].data_ptr(), bk.clip["t"].data_ptr()
                assert all(op.dev == (vote, tptr) for rec in bk.shards for op in rec["step_ops"]) and opt.native_ops_in_step
                with pytest.raises(NotImplementedError):
                    GraphedTrainStep(model, lambda x: x.sum(), (torch.zeros(1),), optimizers=[opt])
                program = ["scaled_norm"] + (["moments"] * nb + ["ratio"] + ["apply"] * nb if kind == "lamb" else [kind] * nb)

                # step() without a scaler: scale 1 (checked by the double), the bound or none
                events.clear()
                k0 = opt.kernel_launches
                opt.step()
                assert events == program and opt.kernel_launches - k0 == len(program)
                assert bk.clip["norm_op"].max_norm == (bound if bound else float("inf"))
                assert float(opt.last_step_skipped) == 0.0 and float(opt.last_grad_norm) == 3.0

                # the scaler: hands over its scale tensor, records the vote for update(); torch's update() backs off and grows
                scaler = ShardedGradScaler(init_scale=64.0, growth_interval=2, device="cpu")
                seen = []
                for overflow in (True, False, False, True):
                    current["overflow"] = overflow
                    scaler.scale(torch.zeros(1))
                    events.clear()
                    scaler.step(opt)
                    assert events == program and opt._loss_scale is scaler._scale
                    with pytest.raises(RuntimeError, match="already been called"):
                        scaler.step(opt)
                    assert float(opt.last_step_skipped) == float(overflow)
                    scaler.update()
                    seen.append(scaler.get_scale())
                assert seen == [32.0, 32.0, 64.0, 32.0]
                current["overflow"] = False
                with pytest.raises(RuntimeError, match="max_grad_norm"):
                    scaler.unscale_(opt)
                # clip_grad_norm_ bounds the unscaled norm: once per step, and with the scale that step() will use
                scaler.scale(torch.zeros(1))
                scaler.attach(opt)
                opt.clip_grad_norm_(0.5)
                assert bk.clip["norm_op"].max_norm == 0.5
                with pytest.raises(RuntimeError, match="once per step"):
                    opt.clip_grad_norm_(0.5)
                events.clear()
                scaler.step(opt)
                assert events == program[1:]
                scaler.update()
                opt.clip_grad_norm_(0.5)
                with pytest.raises(RuntimeError, match="another loss scale"):
                    opt.set_loss_scale(torch.ones(1))
                opt.step()

                # t (taken steps: 1 + 2 + 1 + 1 of 7 launches) goes through checkpoints and re-bucketing, with or without loss scaling
                assert int(bk.clip["t"]) == 5
                sd = opt.state_dict()
                assert sd["steps"] == 5
                rebucket(model, opt)
                assert opt._bucketing is not bk and int(opt._bucketing.clip["t"]) == 5 and opt.state_dict()["steps"] == 5
                _, plain = build(lambda ps: make(ps, max_grad_norm=bound), state=sd)
                assert all(op.steps() == 5 for rec in plain._bucketing.shards for op in rec["step_ops"])
                _, back = build(lambda ps: make(ps, max_grad_norm=bound, loss_scaling=True), state=plain.state_dict())
                assert int(back._bucketing.clip["t"]) == 5
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_loss_scaling_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))
