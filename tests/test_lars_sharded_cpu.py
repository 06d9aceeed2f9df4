"""The sharded in-bucket LARS without a GPU: the fallback path (gloo all-reduce + ``FusedLARS``) against one process on the
concatenated batch, the GPU-only driver (``init_operations`` / ``step()``) with host doubles of the peer engine and the native ops
(segment tables, op order, launch counts, checkpoints across world sizes, the error cases), and the ImageNet example with
``--optimizer lars``."""
import copy
import os
import sys
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _flat, _net

BOUND = 9.0   # between the smallest and the largest norm of the six steps
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _groups(m):
    return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 5e-3},
            {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]


def _fallback_worker(rank, world, bound):
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.ops.optim import FusedLARS
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lars

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)
    opt = make_sharded_fused_lars(_groups(model), lr=0.5, trust_coefficient=0.02, max_grad_norm=bound)
    oopt = FusedLARS(_groups(oracle), lr=0.5, trust_coefficient=0.02)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    norms = []
    for it in range(6):
        lr = 0.5 if it < 3 else 0.2
        for o in (opt, oopt):
            for g in o.param_groups:
                g["lr"] = lr
        x, y = _batch(rank, it)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        opt.step()
        xs, ys = zip(*[_batch(r, it) for r in range(world)])
        oopt.zero_grad()
        F.cross_entropy(oracle(torch.cat(xs)), torch.cat(ys)).backward()
        if bound is not None:
            norms.append(float(torch.nn.utils.clip_grad_norm_(oracle.parameters(), bound)))
        oopt.step()
    return _flat(model), _flat(oracle), norms


@pytest.mark.parametrize("bound", [None, BOUND])
def test_fallback_path_matches_fused_lars_on_the_whole_batch(bound):
    for mine, oracle, norms in run_distributed(_fallback_worker, world=2, args=(bound,)):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        if bound is not None:
            assert any(n > bound for n in norms) and any(n <= bound for n in norms), norms


def _host_double_worker(rank, world):
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lamb, make_sharded_fused_lars
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
            self.max_norm = m

        def set_scale_ptr(self, p):
            self.scale_ptr = p

        def set_device_step(self, vote, step):
            self.dev = (vote, step)

    class Norms(Op):
        def run(self, opt):
            events.append(("norms", opt._bucketing.pre_ops.index(self)))
            self.s += 1

    class Ratio(Op):
        @staticmethod
        def box_bytes(n):
            return 2 * 8 * n * 16

        def run(self, opt):
            events.append(("exchange",))

    class Apply(Op):
        def run(self, opt):
            events.append(("apply", opt._bucketing.update_ops.index(self)))
            self.s += 1

    class Norm(Op):
        def run(self, opt):
            events.append(("norm",))

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
        ShardGradOp, LarsNormsOp, LambRatioOp, ShardLarsOp = Op, Norms, Ratio, Apply
        GradNormOp = LossScaleNormOp = Norm
        LambMomentsOp = ShardLambOp = Op
        MAX_COMM_BLOCKS, MAX_PEERS = real_native.MAX_COMM_BLOCKS, real_native.MAX_PEERS

        def run_op(self, op, stream, device):
            op.run(current["opt"])

        def __getattr__(self, name):
            return getattr(real_native, name)

    class Group:
        def __init__(self, n, r):
            self.n, self.r = n, r

        def size(self):
            return self.n

        def rank(self):
            return self.r

    def build(make, P=1, r=0, model=None, state=None):
        torch.manual_seed(5)
        model = model or torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.BatchNorm2d(8), torch.nn.Flatten(),
                                             torch.nn.Linear(8 * 36, 5)).to(memory_format=torch.channels_last)
        want = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = make(model)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        impl.process_group = Group(P, r)
        impl._carry_state_over()
        if state is not None:
            opt.load_state_dict(state)
        for bucket in model.bagua_buckets:
            nbytes = bucket.backend_tensor.numel() * bucket.backend_tensor.element_size()
            bucket._engine = lambda group=None: Engine()
            bucket._slice = Slice(nbytes)
            bucket.backend_bucket = BackendBucket()
            impl.init_operations(ddp, bucket)
        current["opt"] = opt
        return model, opt, want

    def lars(bound=None, scaled=False):
        return lambda m: make_sharded_fused_lars(_groups(m), lr=0.1, weight_decay=5e-3, max_grad_norm=bound, loss_scaling=scaled)

    class Odd(torch.nn.Module):   # 53 fp32 elements: vectors shared by several parameters, one straddling slices, a padding tail
        def __init__(self):
            super().__init__()
            for name, n in zip("abcdef", (1, 1, 1, 40, 3, 7)):
                setattr(self, name, torch.nn.Parameter(torch.randn(n)))

        def forward(self, x):
            return x

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        # segment tables: every element of every parameter in exactly one segment across the ranks; the LARS ops take the
        # [master, shard] lists, the gradient shard, the momentum and the exchange's sums
        for P in (3, 8):
            seen = {}
            for r in range(P):
                model, opt, _ = build(lambda m: make_sharded_fused_lars([{"params": list(m.parameters()), "weight_decay": 0.01}], lr=0.1), P=P, r=r,
                                      model=Odd())
                rec = opt._bucketing.shards[0]
                plan, partials, table, segs = rec["lamb_tables"]
                lam = opt._bucketing.lamb
                layout = {name: (off, n) for name, off, n, _, _ in rec["layout"]}
                for a, b, t in segs:
                    seen.setdefault(t, []).append((rec["lo"] + a, rec["lo"] + b))
                if segs:
                    assert len(plan.keep) == 2, "LARS stage 1 reads [master, gradient shard] only"
                    assert plan.keep[1][0].data_ptr() == rec["shard"].data_ptr() + 4 * segs[0][0]
                apply = opt._bucketing.update_ops[0]
                master, momentum = rec["state"]
                assert apply.args[5:12] == (rec["shard"].data_ptr(), 0, master.data_ptr(), momentum.data_ptr(), table.data_ptr(), len(segs),
                                            lam["sums"].data_ptr())
                assert isinstance(opt._bucketing.pre_ops[0], Norms) and lam["ratio_op"] is not None and len(lam["index"]) == 6
            for t, spans in seen.items():
                name = next(k for k, v in lam["index"].items() if v == t)
                assert sorted(spans)[0][0] == layout[name][0] and sum(b - a for a, b in spans) == layout[name][1]
            assert any(len(s) >= 3 for s in seen.values()), seen   # a parameter cut by two slice boundaries

        for bound, scaled in ((None, False), (1.5, False), (None, True)):
            events.clear()
            model, opt, want = build(lars(bound, scaled))
            buckets = model.bagua_buckets
            assert len(buckets) >= 2 and all(len(b.backend_bucket.ops) == 1 for b in buckets), "phase A is the whole bucket program"
            variant = "fused_lars_" + ("scaled_" if scaled else "") + ("clip_" if bound else "")
            assert all(b.allreduce_variant.startswith(variant) for b in buckets), [b.allreduce_variant for b in buckets]
            bk = opt._bucketing
            assert len(bk.update_ops) == len(bk.pre_ops) == len(buckets)
            exchange = bound is not None or scaled
            coef_ptr = bk.clip["out"][1:].data_ptr() if exchange else 0
            assert all(m.args[7] == coef_ptr for m in bk.pre_ops) and all(a.args[6] == coef_ptr for a in bk.update_ops)
            if scaled:
                assert all(o.dev == (coef_ptr, bk.clip["t"].data_ptr()) for rec in bk.shards for o in rec["step_ops"])
            # hyper-parameters per group: (lr, momentum, weight_decay, trust_coefficient)
            assert {o.hyper for o in bk.pre_ops + bk.update_ops} == {(0.1, 0.9, 5e-3, 1e-3), (0.1, 0.9, 0.0, 1e-3)}
            for n, p in model.named_parameters():
                assert torch.equal(p.detach(), want[n])
            launches = opt.kernel_launches
            opt.step()
            nb = len(buckets)
            assert [e[0] for e in events] == (["norm"] if exchange else []) + ["norms"] * nb + ["exchange"] + ["apply"] * nb
            assert opt.kernel_launches == launches + 2 * nb + 1 + (1 if exchange else 0)
            assert opt.native_ops_in_step
            with pytest.raises(NotImplementedError):
                GraphedTrainStep(model, lambda x: x.sum(), (torch.zeros(1),), optimizers=[opt])

        # consolidated checkpoints: written by 2 ranks, read back by 3, the same per-parameter state
        def positions(rec, k):   # a value per bucket position of the parameters (the alignment padding holds no state)
            covered = torch.zeros(rec["numel"], dtype=torch.bool)
            for _, off, n, _, _ in rec["layout"]:
                covered[off:off + n] = True
            n = rec["hi"] - rec["lo"]
            out = torch.zeros_like(rec["state"][k])
            vals = torch.arange(rec["lo"], rec["hi"], dtype=torch.float32) * (1.0 if k == 0 else -0.5)
            out[:n] = torch.where(covered[rec["lo"]:rec["hi"]], vals, torch.zeros(()))
            return out

        recs2 = []
        for r in range(2):
            _, o, want = build(lars(), P=2, r=r)
            for rec in o._bucketing.shards:
                for k, t in enumerate(rec["state"]):
                    t.copy_(positions(rec, k))
                for op in rec["step_ops"]:
                    op.set_steps(4)
            recs2.append(o)
        by_bucket = {rec["bucket"]: [o._bucketing.shards[i]["state"] for o in recs2] for i, rec in enumerate(recs2[0]._bucketing.shards)}
        opt2 = recs2[0]

        def gather(t, group):
            for states in by_bucket.values():
                for k in range(2):
                    if states[0][k] is t:
                        return [s[k] for s in states]
            raise AssertionError("unknown state tensor")

        opt2._gather = gather
        sd = opt2.state_dict()
        assert sd["sharded_fused"] == "lars" and sd["steps"] == 4 and set(want) <= set(sd["state"])
        assert all(set(st) == {"master", "momentum_buffer"} for st in sd["state"].values())
        for r in range(3):
            _, o3, _ = build(lars(), P=3, r=r, state=sd)
            for rec in o3._bucketing.shards:
                for k, t in enumerate(rec["state"]):
                    assert torch.equal(t, positions(rec, k)), (r, rec["bucket"], k)
                assert all(op.steps() == 4 for op in rec["step_ops"])
        # a LAMB checkpoint is refused, and LARS's is refused by LAMB
        lamb = build(lambda m: make_sharded_fused_lamb(_groups(m), lr=0.01))[1]
        lamb._gather = lambda t, group: [t]
        with pytest.raises(ValueError, match="lamb"):
            opt2.load_state_dict(lamb.state_dict())
        with pytest.raises(ValueError, match="lars"):
            lamb.load_state_dict(sd)
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_lars_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))


def test_graph_safe_optimizer_names_fused_lars():
    from bagua_b200.ops.optim import FusedLARS
    from bagua_b200.utils.graph import graph_safe_optimizer

    reason = graph_safe_optimizer(FusedLARS([torch.nn.Parameter(torch.zeros(3))]))
    assert reason is not None and "FusedLARS" in reason and "capturable" not in reason


def test_imagenet_example_with_lars(tmp_path):
    from tests.mp_utils import free_port, run_in_session

    env = dict(os.environ, PYTHONPATH=REPO + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="", BAGUA_FORCE_CPU="1")
    cmd = [sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={free_port()}",
           os.path.join(REPO, "examples/imagenet/main.py"), "--cpu", "--synthetic", "--epochs", "1", "--steps-per-epoch", "2", "--batch-size", "2",
           "--num-classes", "10", "--image-size", "32", "--print-freq", "1", "--optimizer", "lars", "--trust-coefficient", "0.002"]
    r = run_in_session(cmd, 240, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
