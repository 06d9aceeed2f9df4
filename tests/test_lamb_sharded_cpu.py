"""The sharded in-bucket LAMB without a GPU: the fallback path (gloo all-reduce + ``FusedLAMB``) against one process on the
concatenated batch, and the GPU-only driver (``init_operations`` / ``step()``) with host doubles of the peer engine and the native
ops: segment tables, op order, launch count, checkpoints and the error cases."""
import copy
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _flat, _net

BOUND = 9.0   # between the smallest and the largest norm of the six steps


def _groups(m):
    return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 0.05},
            {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]


def _fallback_worker(rank, world, bound):
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.ops.optim import FusedLAMB
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lamb

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)
    opt = make_sharded_fused_lamb(_groups(model), lr=1e-2, max_grad_norm=bound)
    oopt = FusedLAMB(_groups(oracle), lr=1e-2)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    norms = []
    for it in range(6):
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
def test_fallback_path_matches_fused_lamb_on_the_whole_batch(bound):
    for mine, oracle, norms in run_distributed(_fallback_worker, world=2, args=(bound,)):
        torch.testing.assert_close(mine, oracle, rtol=1e-5, atol=1e-6)
        if bound is not None:
            assert any(n > bound for n in norms) and any(n <= bound for n in norms), norms


def _host_double_worker(rank, world):
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_lamb
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
            events.append(("alloc", nbytes))
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

        def set_max_norm(self, m):
            self.max_norm = m

    class Moments(Op):
        def run(self, opt):
            events.append(("moments", opt._bucketing.pre_ops.index(self)))
            self.s += 1

    class Ratio(Op):
        @staticmethod
        def box_bytes(n):
            return 2 * 8 * n * 16

        def run(self, opt):
            events.append(("ratio",))

    class Apply(Op):
        def run(self, opt):
            events.append(("apply", opt._bucketing.update_ops.index(self)))
            self.s += 1

    class Norm(Op):
        def run(self, opt):
            events.append(("norm",))
            opt._bucketing.clip["out"].copy_(torch.tensor([7.0, 0.5]))

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
        ShardGradOp, GradNormOp, LambMomentsOp, LambRatioOp, ShardLambOp = Op, Norm, Moments, Ratio, Apply
        AllReduceAdamOp = ShardAdamOp = Op
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
        model = model or torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.Flatten(), torch.nn.Linear(8 * 36, 5)).to(memory_format=torch.channels_last)
        want = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = make(model)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        impl.process_group = Group(P, r)
        impl._carry_state_over()
        if state is not None:   # loaded while no shard exists (as before with_bagua): applied bucket by bucket below
            opt.load_state_dict(state)
            assert opt._pending_state is state
        for bucket in model.bagua_buckets:
            nbytes = bucket.backend_tensor.numel() * bucket.backend_tensor.element_size()
            bucket._engine = lambda group=None: Engine()
            bucket._slice = Slice(nbytes)
            bucket.backend_bucket = BackendBucket()
            impl.init_operations(ddp, bucket)
        current["opt"] = opt
        return model, opt, want

    def lamb(bound=None):
        return lambda m: make_sharded_fused_lamb(_groups(m), lr=0.01, max_grad_norm=bound)

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        # segment tables: parameters of 1, 3 and 7 elements, 16-byte vectors shared by 3+ parameters, a parameter straddling 3
        # slices, the padding tail, and an empty slice at P = 8 (53 fp32 elements = 14 vectors: 7 slices of 2 vectors)
        class Odd(torch.nn.Module):
            def __init__(self):
                super().__init__()
                for name, n in zip("abcdef", (1, 1, 1, 40, 3, 7)):
                    setattr(self, name, torch.nn.Parameter(torch.randn(n)))

            def forward(self, x):
                return x

        for P in (3, 8):
            seen, empty = {}, 0
            for r in range(P):
                model, opt, _ = build(lambda m: make_sharded_fused_lamb([{"params": list(m.parameters()), "weight_decay": 0.01}], lr=0.01),
                                      P=P, r=r, model=Odd())
                (bucket,) = model.bagua_buckets
                rec = opt._bucketing.shards[0]
                plan, partials, table, segs = rec["lamb_tables"]
                lam = opt._bucketing.lamb
                layout = {name: (off, n) for name, off, n, _, _ in rec["layout"]}
                for a, b, t in segs:
                    seen.setdefault(t, []).append((rec["lo"] + a, rec["lo"] + b))
                    name = next(k for k, v in lam["index"].items() if v == t)
                    off, n = layout[name]
                    assert off <= rec["lo"] + a < rec["lo"] + b <= off + n     # the segment lies inside its parameter
                assert torch.equal(table, torch.tensor([v for s in segs for v in s] or [0, 0, 0], dtype=torch.int32))
                if not segs:
                    empty += 1
                    assert plan is None     # an empty slice still builds its ops (and takes part in every exchange)
                assert lam["ratio_op"] is not None and len(lam["index"]) == 6   # the padding tensor has no ratio slot
                assert opt._bucketing.update_ops[0].args[9] == len(segs)
            assert empty == (1 if P == 8 else 0)
            for t, spans in seen.items():   # every element of every parameter in exactly one segment, across the ranks
                name = next(k for k, v in lam["index"].items() if v == t)
                assert sorted(spans)[0][0] == layout[name][0] and sum(b - a for a, b in spans) == layout[name][1]
            assert any(len(s) >= 3 for s in seen.values()), seen   # a parameter straddling 3 slices
            assert any(sum(1 for off, n in layout.values() if off < v + 4 and off + n > v) >= 3 for v in range(0, 56, 4))
            assert sum(n for _, n in layout.values()) == 53 and bucket.backend_tensor.numel() == 56   # a padding tail

        # a parameter longer than two 65536-element chunks: its segment gets consecutive stage-1 blocks, all summed for its ratio
        model, opt, _ = build(lambda m: make_sharded_fused_lamb(list(m.parameters()), lr=0.01), model=torch.nn.Linear(300, 500))
        lam = opt._bucketing.lamb
        (bucket,) = model.bagua_buckets
        plan, partials, table, segs = opt._bucketing.shards[0]["lamb_tables"]
        t_w = next(v for k, v in lam["index"].items() if k.endswith("weight"))
        t_b = next(v for k, v in lam["index"].items() if k.endswith("bias"))
        assert lam["seg_nblk"][t_w] == 3 and lam["seg_nblk"][t_b] == 1 and plan.n_blocks == 4
        first = {t: i for i, t in enumerate(s[2] for s in segs)}
        order = sorted((t_w, t_b), key=first.get)
        assert lam["seg_ptr"][order[0]] == partials.data_ptr() and lam["seg_ptr"][order[1]] == partials.data_ptr() + 16 * lam["seg_nblk"][order[0]]

        for bound in (None, 1.5):
            events.clear()
            model, opt, want = build(lamb(bound))
            buckets = model.bagua_buckets
            assert all(len(b.backend_bucket.ops) == 1 for b in buckets), "phase A is the whole bucket program"
            assert all(b.allreduce_variant.startswith("fused_lamb_" + ("clip_" if bound else "")) for b in buckets)
            bk = opt._bucketing
            assert len(bk.update_ops) == len(bk.pre_ops) == len(buckets)
            coef_ptr = bk.clip["out"][1:].data_ptr() if bound else 0
            assert all(m.args[7] == coef_ptr for m in bk.pre_ops)
            for n, p in model.named_parameters():
                assert torch.equal(p.detach(), want[n])
            events.clear()
            launches = opt.kernel_launches
            opt.step()
            nb = len(buckets)
            assert [e[0] for e in events] == (["norm"] if bound else []) + ["moments"] * nb + ["ratio"] + ["apply"] * nb
            assert opt.kernel_launches == launches + 2 * nb + 1 + (1 if bound else 0)
            # checkpoints: both step-carrying ops of a bucket restored; consolidated state round-trips
            opt._gather = lambda t, group: [t]
            sd = opt.state_dict()
            assert sd["sharded_fused"] == "lamb" and sd["steps"] == 1 and set(want) <= set(sd["state"])
            for rec in bk.shards:
                for t in rec["state"]:
                    t.add_(1.0)
                for op in rec["step_ops"]:
                    op.set_steps(0)
            opt.load_state_dict(sd)
            assert all(op.steps() == 1 for rec in bk.shards for op in rec["step_ops"])
            again = opt.state_dict()
            for n in want:
                for k in ("master", "exp_avg", "exp_avg_sq"):
                    assert torch.equal(again["state"][n][k], sd["state"][n][k])
            with pytest.raises(NotImplementedError):
                GraphedTrainStep(model, lambda x: x.sum(), (torch.zeros(1),), optimizers=[opt])
            if bound is None:
                with pytest.raises(RuntimeError, match="max_grad_norm"):
                    opt.clip_grad_norm_(1.0)

            # load_state_dict before with_bagua: applied to the shards when the ops are built
            model2, opt2, _ = build(lamb(bound), state=sd)
            assert all(op.steps() == 1 for rec in opt2._bucketing.shards for op in rec["step_ops"])
            opt2._gather = lambda t, group: [t]
            for n in want:
                assert torch.equal(opt2.state_dict()["state"][n]["exp_avg"], sd["state"][n]["exp_avg"])
            # an Adam checkpoint is refused
            adam = build(lambda m: make_sharded_fused_adam(_groups(m), lr=0.01, adamw=True))[1]
            adam._gather = lambda t, group: [t]
            with pytest.raises(ValueError, match="adam"):
                opt.load_state_dict(adam.state_dict())
            current["opt"] = opt
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_lamb_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))
