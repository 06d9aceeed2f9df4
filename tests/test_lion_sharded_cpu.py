"""The sharded in-bucket Lion without a GPU: the GPU-only driver (``init_operations`` / ``step()``) with host doubles of the peer
engine and the native ops (programs, op kinds and arguments, launch counts, ``allreduce_variant``, checkpoints across world sizes),
``FusedLion`` on the CPU against the fp32 replay, the fallback path (gloo all-reduce + ``FusedLion``) against one process on the
whole batch, the graph refusal, and the SQuAD example with ``--optimizer lion --fused-shard``."""
import copy
import os
import sys
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _flat, _net

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BETAS = (0.9, 0.99)


def _groups(m, wd=0.1):
    return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": wd},
            {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]


def test_fused_lion_on_the_cpu_is_the_replay_bit_for_bit():
    """fp32 and bf16 (fp32 master) parameters in two groups, an lr change, zero and NaN gradient elements."""
    from bagua_b200.ops.optim import FusedLion, lion_reference_step_

    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(7, 5)), torch.nn.Parameter(torch.randn(33).to(torch.bfloat16)), torch.nn.Parameter(torch.randn(4))]
    opt = FusedLion([{"params": ps[:2], "weight_decay": 0.2}, {"params": ps[2:]}], lr=1e-2, betas=BETAS)
    ref = {id(p): (p.detach().float().clone(), torch.zeros(p.shape)) for p in ps}
    for step, lr in enumerate([1e-2, 1e-2, 3e-3]):
        for g in opt.param_groups:
            g["lr"] = lr
        grads = [torch.randn(p.shape).to(p.dtype) for p in ps]
        grads[0][0] = 0
        if step == 1:
            grads[2][1] = float("nan")
        for p, g in zip(ps, grads):
            p.grad = g.clone()
        opt.step()
        for p, g, wd in zip(ps, grads, (0.2, 0.2, 0.0)):
            w, m = ref[id(p)]
            lion_reference_step_(w, m, g, lr, BETAS, wd)
            got = opt.state[p]["master"] if p.dtype == torch.bfloat16 else p.detach()
            assert torch.equal(torch.nan_to_num(got, 9.0), torch.nan_to_num(w, 9.0)) and torch.equal(torch.isnan(got), torch.isnan(w))
            assert torch.equal(torch.nan_to_num(opt.state[p]["exp_avg"], 9.0), torch.nan_to_num(m, 9.0))
            assert torch.equal(p.detach(), w.to(p.dtype)) or bool(torch.isnan(w).any())
            assert torch.count_nonzero(p.grad).item() == 0
    assert torch.isnan(ps[2][1]) and int(torch.isnan(ps[2]).sum()) == 1


def _fallback_worker(rank, world, bound):
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.ops.optim import FusedLion
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lion

    bagua.init_process_group()
    torch.manual_seed(3)
    model = _net()
    oracle = copy.deepcopy(model)
    opt = make_sharded_fused_lion(_groups(model), lr=1e-2, betas=BETAS, max_grad_norm=bound)
    oopt = FusedLion(_groups(oracle), lr=1e-2, betas=BETAS)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    for it in range(6):
        lr = 1e-2 if it < 3 else 4e-3
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
            torch.nn.utils.clip_grad_norm_(oracle.parameters(), bound)
        oopt.step()
    return _flat(model), _flat(oracle)


@pytest.mark.parametrize("bound", [None, 0.5])
def test_fallback_path_matches_fused_lion_on_the_whole_batch(bound):
    for mine, oracle in run_distributed(_fallback_worker, world=2, args=(bound,)):
        # an all-reduced mean and a whole-batch gradient differ in the last bits, which may flip a sign(u) near 0: ±2·lr there
        diff = (mine - oracle).abs()
        assert float(diff.max()) <= 2 * (3 * 1e-2 + 3 * 4e-3) + 1e-6 and float((diff > 1e-5).double().mean()) < 0.02


def _host_double_worker(rank, world):
    import bagua_b200 as bagua
    import bagua_b200.core as core
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_lion
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

        def set_weight(self, w):
            self.weight = w

        def run(self, opt):
            events.append(self.name)
            self.s += 1

    class Fused(Op):
        name = "allreduce_lion"

    class Apply(Op):
        name = "shard_lion"

    class Norm(Op):
        name = "norm"

    class Ema(Op):
        name = "ema"

    class Grad(Op):
        name = "shard_grad"

        def restart(self):
            events.append("restart")

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
        ShardGradOp, AllReduceLionOp, ShardLionOp, EmaOp = Grad, Fused, Apply, Ema
        GradNormOp = LossScaleNormOp = Norm
        AllReduceAdamOp = ShardAdamOp = ShardPublishOp = Op
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

    def build(make, P=1, r=0, state=None):
        torch.manual_seed(5)
        model = torch.nn.Sequential(torch.nn.Linear(6, 16), torch.nn.LayerNorm(16), torch.nn.Linear(16, 5))
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

    def lion(**kw):
        return lambda m: make_sharded_fused_lion(_groups(m), lr=1e-3, betas=BETAS, **kw)

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        configs = {"plain": {}, "clip": {"max_grad_norm": 1.5}, "scaled": {"loss_scaling": True}, "accumulate": {"accumulate_grads": True},
                   "ema": {"ema_decay": 0.9}}
        for name, kw in configs.items():
            events.clear()
            model, opt, want = build(lion(**kw), P=2, r=1)
            buckets, bk = model.bagua_buckets, opt._bucketing
            nb = len(buckets)
            assert nb >= 2
            two_phase = name in ("clip", "scaled", "accumulate")
            prefix = "fused_lion_" + {"scaled": "scaled_", "clip": "clip_", "accumulate": "accum_"}.get(name, "")
            assert all(b.allreduce_variant == prefix + "two_shot" for b in buckets), [b.allreduce_variant for b in buckets]
            for b, rec in zip(buckets, bk.shards):
                master, exp_avg = rec["state"][:2]
                assert len(rec["state"]) == (3 if name == "ema" else 2), "Lion keeps the master and one moment (+ the EMA)"
                assert [type(o) for o in b.backend_bucket.ops] == [Grad if two_phase else Fused]
                if two_phase:
                    a = b.backend_bucket.ops[0]
                    assert a.args[7:9] == (0.5, True) and (len(a.args) == 12) == (name == "accumulate"), "phase A averages, clears, accumulates"
                else:
                    op = b.backend_bucket.ops[0]
                    assert op.args[7:11] == (master.data_ptr(), exp_avg.data_ptr(), 0.5, True), "the fused op: master, exp_avg, 1/N, clear"
            if two_phase:
                coef = bk.clip["out"][1:].data_ptr() if name != "accumulate" else bk.unit.data_ptr()
                assert len(bk.update_ops) == nb and not bk.pre_ops
                for op, rec in zip(bk.update_ops, bk.shards):
                    assert isinstance(op, Apply)
                    assert op.args[5:9] == (rec["shard"].data_ptr(), coef, rec["state"][0].data_ptr(), rec["state"][1].data_ptr())
                if name == "scaled":
                    assert all(o.dev == (coef, bk.clip["t"].data_ptr()) for o in bk.update_ops)
            else:
                assert not bk.update_ops and bk.clip is None
            # hyper-parameters per group: (lr, beta1, beta2, weight_decay), as doubles
            assert {o.hyper for o, _ in bk.hyper_ops} == {(1e-3, 0.9, 0.99, 0.1), (1e-3, 0.9, 0.99, 0.0)}
            for n, p in model.named_parameters():
                assert torch.equal(p.detach(), want[n])
            launches = opt.kernel_launches
            opt.step()
            exchange = name in ("clip", "scaled")
            assert events == ((["norm"] if exchange else []) + (["shard_lion"] * nb if two_phase else []) + (["restart"] * nb if name == "accumulate" else [])
                              + (["ema"] if name == "ema" else []))
            assert opt.kernel_launches == launches + nb + (1 if exchange else 0) + (1 if name == "ema" else 0)
            assert opt.native_ops_in_step == (name != "plain")
            with pytest.raises((NotImplementedError, ValueError), match="FusedLion|native|graph"):
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

        opts2 = []
        for r in range(2):
            _, o, want = build(lion(), P=2, r=r)
            for rec in o._bucketing.shards:
                for k, t in enumerate(rec["state"]):
                    t.copy_(positions(rec, k))
                for op in rec["step_ops"]:
                    op.set_steps(4)
            opts2.append(o)
        by_bucket = {rec["bucket"]: [o._bucketing.shards[i]["state"] for o in opts2] for i, rec in enumerate(opts2[0]._bucketing.shards)}
        opt2 = opts2[0]

        def gather(t, group):
            for states in by_bucket.values():
                for k in range(2):
                    if states[0][k] is t:
                        return [s[k] for s in states]
            raise AssertionError("unknown state tensor")

        opt2._gather = gather
        sd = opt2.state_dict()
        assert sd["sharded_fused"] == "lion" and sd["steps"] == 4 and set(want) <= set(sd["state"])
        assert all(set(st) == {"master", "exp_avg"} for st in sd["state"].values())
        for r in range(3):
            _, o3, _ = build(lion(), P=3, r=r, state=sd)
            for rec in o3._bucketing.shards:
                for k, t in enumerate(rec["state"]):
                    assert torch.equal(t, positions(rec, k)), (r, rec["bucket"], k)
                assert all(op.steps() == 4 for op in rec["step_ops"])
        # an Adam checkpoint is refused, and Lion's is refused by Adam
        adam = build(lambda m: make_sharded_fused_adam(_groups(m), lr=1e-3, adamw=True))[1]
        adam._gather = lambda t, group: [t]
        with pytest.raises(ValueError, match="adam"):
            opt2.load_state_dict(adam.state_dict())
        with pytest.raises(ValueError, match="lion"):
            adam.load_state_dict(sd)
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_lion_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))


def test_graph_safe_optimizer_names_fused_lion():
    from bagua_b200.ops.optim import FusedLion
    from bagua_b200.parallel.algorithms.gradient_allreduce import make_sharded_fused_lion
    from bagua_b200.utils.graph import graph_safe_optimizer

    for opt in (FusedLion([torch.nn.Parameter(torch.zeros(3))]), make_sharded_fused_lion([torch.nn.Parameter(torch.zeros(3))])):
        reason = graph_safe_optimizer(opt)
        assert reason is not None and "FusedLion" in reason


def test_make_sharded_fused_lion_rejects_invalid_hyperparameters():
    from bagua_b200.parallel.algorithms.gradient_allreduce import make_sharded_fused_lion

    p = [torch.nn.Parameter(torch.zeros(3))]
    for kw in (dict(lr=-1.0), dict(weight_decay=-1.0), dict(betas=(0.9, 1.0)), dict(max_grad_norm=0.0), dict(ema_decay=1.0)):
        with pytest.raises(ValueError):
            make_sharded_fused_lion(p, **kw)


def test_squad_example_with_sharded_lion(tmp_path):
    from tests.mp_utils import free_port, run_in_session
    from tests.test_examples_cpu import ENV

    argv = [os.path.join(REPO, "examples", "squad", "main.py"), "--cpu", "--tiny", "--epochs", "1", "--num-synthetic", "24", "--batch-size", "4",
            "--max-seq-length", "64", "--doc_stride", "32", "--output_dir", str(tmp_path / "out"), "--do_lower_case", "--do_train",
            "--optimizer", "lion", "--learning_rate", "1e-5", "--weight_decay", "0.1", "--fused-shard", "--logging_steps", "1"]
    cmd = [sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={free_port()}", *argv]
    r = run_in_session(cmd, 240, env=ENV, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
