"""Gradient accumulation in the fp32 shard of the in-bucket sharded optimizers (``accumulate_grads=True``) without a GPU: the
GPU-only driver (``init_operations`` / ``step()`` / ``zero_grad()`` / re-bucketing) with host doubles of the peer engine and of the
native ops, the fallback path on 2 gloo ranks against ``no_sync()`` accumulation, the error cases, and the SQuAD example with
``--accumulate-in-shard``."""
import copy
import os
import sys
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _flat, _net

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULES = ("sgd", "adam", "lamb", "lars")


def _groups(m):
    return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 0.01},
            {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]


def _make(rule, params, **kw):
    from bagua_b200.parallel.algorithms import gradient_allreduce as ga

    if rule == "sgd":
        return ga.make_sharded_fused_sgd(params, lr=0.1, momentum=0.9, **kw)
    if rule == "adam":
        return ga.make_sharded_fused_adam(params, lr=1e-2, adamw=True, **kw)
    if rule == "lamb":
        return ga.make_sharded_fused_lamb(params, lr=1e-2, **kw)
    return ga.make_sharded_fused_lars(params, lr=0.5, trust_coefficient=0.02, **kw)


def _host_double_worker(rank, world):
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm
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

    class Op:
        def __init__(self, *args):
            self.args, self.hyper, self.s, self.dev = args, None, 0, None

        def set_hyper(self, *a):
            self.hyper = a

        def steps(self):
            return self.s

        def set_steps(self, s):
            self.s = s

        def set_max_norm(self, m):
            pass

        def set_scale_ptr(self, p):
            pass

        def set_device_step(self, vote, step):
            self.dev = (vote, step)

        def run(self, opt):
            events.append(type(self).__name__)
            self.s += 1

    class Grad(Op):
        """ShardGradOp's contract: the first run after construction or restart() overwrites, later ones add (accumulate=True)."""

        def __init__(self, *args):
            super().__init__(*args)
            self.accum = len(args) == 12 and args[11] is True
            self.fresh, self.modes, self.restarts = True, [], 0

        def restart(self):
            self.restarts += 1
            self.fresh = True

        def resume(self):
            self.fresh = False

        def pending(self):
            return self.accum and not self.fresh

        def backward(self, g):
            """One phase A with the reduced gradient g (the whole bucket: one rank)."""
            shard = self.args[5]
            t = next(rec["shard"] for rec in current["opt"]._bucketing.shards if rec["shard"].data_ptr() == shard)
            add = self.accum and not self.fresh
            self.fresh = False
            self.modes.append("add" if add else "overwrite")
            t[: g.numel()] = (t[: g.numel()] + g) if add else g

    class Ratio(Op):
        @staticmethod
        def box_bytes(n):
            return 2 * 8 * n * 16

    class BackendBucket:
        def __init__(self):
            self.ops = []

        def append_op(self, op):
            self.ops.append(op)

        def clear_ops(self):
            self.ops = []

    real_native = core.native()
    current = {}

    class Sgd(Op):
        pass

    class Adam(Op):
        pass

    class FakeC:
        ShardGradOp, LambRatioOp = Grad, Ratio
        ShardSgdOp = AllReduceSgdOp = Sgd
        ShardAdamOp = AllReduceAdamOp = Adam
        GradNormOp = LossScaleNormOp = LarsNormsOp = LambMomentsOp = ShardLambOp = ShardLarsOp = Op
        MAX_COMM_BLOCKS, MAX_PEERS = real_native.MAX_COMM_BLOCKS, real_native.MAX_PEERS

        def run_op(self, op, stream, device):
            op.run(current["opt"])

        def __getattr__(self, name):
            return getattr(real_native, name)

    def init_buckets(model):
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        for bucket in model.bagua_buckets:
            nbytes = bucket.backend_tensor.numel() * bucket.backend_tensor.element_size()
            bucket._engine = lambda group=None: Engine()
            bucket._slice = Slice(nbytes)
            bucket.backend_bucket = BackendBucket()
            impl.init_operations(ddp, bucket)
        model.bagua_ddp._fwd_pre_hook = impl.init_forward_pre_hook(ddp)

    def build(rule, **kw):
        torch.manual_seed(5)
        model = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.Flatten(), torch.nn.Linear(8 * 36, 5)).to(memory_format=torch.channels_last)
        opt = _make(rule, _groups(model), **kw)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        model.bagua_ddp.bagua_algorithm._carry_state_over()
        current["opt"] = opt
        init_buckets(model)
        return model, opt

    def grad_ops(model):
        return [b.backend_bucket.ops[0] for b in model.bagua_buckets]

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        for rule in RULES:
            per_param = rule in ("lamb", "lars")
            for kw in ({}, {"max_grad_norm": 1.5}, {"loss_scaling": True}):
                exchange = bool(kw)
                # without the flag: the parent's programs, op arguments and counts
                model, opt = build(rule, **kw)
                bk, buckets = opt._bucketing, model.bagua_buckets
                if exchange or per_param:
                    assert all(isinstance(o, Grad) and len(o.args) == 11 and not o.accum for o in grad_ops(model))
                    assert bk.unit is None and not any("accum_" in b.allreduce_variant for b in buckets)
                else:
                    assert all(isinstance(o, Sgd if rule == "sgd" else Adam) for o in grad_ops(model)) and not bk.update_ops
                base_launches, base_updates = bk.launches, len(bk.update_ops)
                assert not opt.native_ops_in_step or exchange or per_param

                # with the flag: phase A is the whole bucket program, the update runs in step()
                model, opt = build(rule, accumulate_grads=True, **kw)
                bk, buckets = opt._bucketing, model.bagua_buckets
                assert all(len(b.backend_bucket.ops) == 1 and isinstance(b.backend_bucket.ops[0], Grad) and b.backend_bucket.ops[0].accum
                           for b in buckets), rule
                assert all("_accum_" in b.allreduce_variant for b in buckets), [b.allreduce_variant for b in buckets]
                assert [rec["grad_op"] for rec in bk.shards] == grad_ops(model)
                assert len(bk.update_ops) == len(buckets) and opt.native_ops_in_step
                if exchange or per_param:
                    assert bk.launches == base_launches and len(bk.update_ops) == base_updates
                else:   # SGD / Adam: the bucket kernel's update moves to step() with a coefficient of exactly 1.0 on the device
                    assert bk.launches == len(buckets) and bk.unit is not None and float(bk.unit) == 1.0
                    cls = Sgd if rule == "sgd" else Adam
                    assert all(isinstance(o, cls) and o.args[6] == bk.unit.data_ptr() for o in bk.update_ops)
                    for rec, o in zip(bk.shards, bk.update_ops):
                        assert o.args[5] == rec["shard"].data_ptr() and rec["grad_op"].args[6] == rec["partials"].data_ptr()

                # transitions: construction, micro-batches, step(), zero_grad() after step(), a discarding zero_grad()
                ops = grad_ops(model)
                gs = []
                for rec in bk.shards:   # a reduced gradient is zero on the bucket's alignment padding
                    g = torch.zeros(rec["hi"] - rec["lo"])
                    for _, off, n, _, _ in rec["layout"]:
                        g[max(off - rec["lo"], 0): max(min(off + n, rec["hi"]) - rec["lo"], 0)].normal_()
                    gs.append(g)

                def micro():
                    for o, g in zip(ops, gs):
                        o.backward(g)

                for _ in range(3):
                    micro()
                assert all(o.modes == ["overwrite", "add", "add"] for o in ops)
                for rec, g in zip(bk.shards, gs):
                    torch.testing.assert_close(rec["shard"][: g.numel()], 3 * g)
                events.clear()
                launches = opt.kernel_launches
                opt.step()
                assert opt.kernel_launches - launches == bk.launches + (1 if exchange else 0)
                assert all(o.restarts == 1 and not o.pending() for o in ops)
                opt.zero_grad()                      # right after step(): free, no restart
                assert all(o.restarts == 1 for o in ops)
                micro()
                micro()
                opt.zero_grad()                      # mid-accumulation: discards the sum
                assert all(o.restarts == 2 for o in ops)
                micro()
                assert all(o.modes[3:] == ["overwrite", "add", "overwrite"] for o in ops)

                # re-bucketing mid-accumulation carries the sum over; the new phase-A ops continue it
                micro()
                opt._gather = lambda t, group: [t]
                sums = {rec["bucket"]: rec["shard"][: rec["hi"] - rec["lo"]].clone() for rec in bk.shards}
                assert all(o.pending() for o in ops)
                model.bagua_ddp.bagua_algorithm._carry_state_over()
                init_buckets(model)
                new = opt._bucketing
                assert all(rec["grad_op"].pending() for rec in new.shards)
                for rec in new.shards:
                    torch.testing.assert_close(rec["shard"][: rec["hi"] - rec["lo"]], sums[rec["bucket"]])
                # state_dict() mid-accumulation leaves the sum alone and does not save it
                before = [rec["shard"].clone() for rec in new.shards]
                sd = opt.state_dict()
                assert "grad_sum" not in sd and all(torch.equal(b, rec["shard"]) for b, rec in zip(before, new.shards))
                assert all(rec["grad_op"].pending() for rec in new.shards)
                # after step() nothing is pending: a re-bucketing then carries no sum
                opt.step()
                model.bagua_ddp.bagua_algorithm._carry_state_over()
                assert opt._pending_state["grad_sum"] is None
                init_buckets(model)
                assert not any(rec["grad_op"].pending() for rec in opt._bucketing.shards)

                with pytest.raises(NotImplementedError, match="accumulated gradient"):
                    GraphedTrainStep(model, lambda x: x.sum(), (torch.zeros(1),), optimizers=[opt])
                if not exchange:
                    with pytest.raises(RuntimeError, match="max_grad_norm"):
                        opt.clip_grad_norm_(1.0)
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_accumulating_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))


def _fallback_worker(rank, world, rule, bound):
    """K = 3 micro-batches per step for 4 steps: every micro-step communicating into the accumulating optimizer, against the same
    run with the first two micro-steps under ``no_sync()``."""
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    torch.manual_seed(3)
    base = _net()
    out = []
    for accum in (True, False):
        model = copy.deepcopy(base)
        opt = _make(rule, _groups(model), max_grad_norm=bound, accumulate_grads=accum)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        for it in range(4):
            opt.zero_grad()
            for k in range(3):
                x, y = _batch(rank, 3 * it + k)
                last = k == 2
                model.bagua_ddp.require_backward_grad_sync = accum or last
                (F.cross_entropy(model(x), y) / 3).backward()
            opt.step()
        model.bagua_ddp.require_backward_grad_sync = True
        out.append(_flat(model))
    return out


@pytest.mark.parametrize("bound", [None, 2.0])
@pytest.mark.parametrize("rule", RULES)
def test_fallback_accumulation_matches_no_sync(rule, bound):
    for accumulated, no_sync in run_distributed(_fallback_worker, world=2, args=(rule, bound)):
        torch.testing.assert_close(accumulated, no_sync, rtol=1e-5, atol=1e-6)
        assert not torch.equal(accumulated, _flat(_net())), "the weights must have moved"


def _average_false_worker(rank, world):
    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    model = _net()
    opt = _make("adam", model.parameters(), accumulate_grads=True)
    with pytest.raises(ValueError, match="average=True"):
        model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt, average=False))
    plain = _make("adam", _net().parameters())
    FusedGradientAllReduceAlgorithm(plain, average=False).reify(None)   # unchanged without the flag
    return True


def test_accumulation_needs_averaging():
    assert all(run_distributed(_average_false_worker, world=1))


def test_squad_example_accumulates_in_shard(tmp_path):
    from tests.mp_utils import free_port, run_in_session
    from tests.test_examples_cpu import ENV

    argv = [os.path.join(REPO, "examples", "squad", "main.py"), "--cpu", "--tiny", "--epochs", "1", "--num-synthetic", "24", "--batch-size", "4",
            "--max-seq-length", "64", "--doc_stride", "32", "--output_dir", str(tmp_path / "out"), "--do_lower_case", "--do_train",
            "--gradient_accumulation_steps", "2", "--fused-shard", "--accumulate-in-shard", "--logging_steps", "1"]
    cmd = [sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={free_port()}", *argv]
    r = run_in_session(cmd, 240, env=ENV, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
