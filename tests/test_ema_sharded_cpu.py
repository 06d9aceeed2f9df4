"""The weight EMA of the in-bucket sharded optimizers (``ema_decay``) without a GPU: the GPU-only driver with host doubles of the peer
engine and of the native ops (op tables, launch counts, the vote, ``ema_weights()``, graph refusal, the checkpoint load matrix), the
fallback path on 2 gloo ranks against an fp32 replay and ``torch.optim.swa_utils.AveragedModel``, a checkpoint written by 2 ranks and
read by 3, and the ImageNet example with ``--ema-decay``."""
import copy
import os
import sys
import types

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_algorithms_cpu import _batch, _net

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


def _replay(e, m, decay):
    """The fp32 update the kernels make: three separately rounded operations."""
    w = torch.tensor(1.0 - float(decay), dtype=torch.float32)
    return e + torch.mul(torch.sub(m, e), w)


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
            self.args, self.hyper, self.s, self.dev, self.w = args, None, 0, None, None

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

        def set_weight(self, w):
            self.w = w

        def restart(self):
            pass

        def pending(self):
            return False

        def run(self, opt):
            events.append(type(self).__name__)
            self.s += 1

    class Ratio(Op):
        @staticmethod
        def box_bytes(n):
            return 2 * 8 * n * 16

    class Ema(Op):
        pass

    class Publish(Op):
        pass

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
        LambRatioOp = Ratio
        EmaOp, ShardPublishOp = Ema, Publish
        ShardGradOp = ShardSgdOp = AllReduceSgdOp = ShardAdamOp = AllReduceAdamOp = Op
        GradNormOp = LossScaleNormOp = LarsNormsOp = LambMomentsOp = ShardLambOp = ShardLarsOp = Op
        MAX_COMM_BLOCKS, MAX_PEERS = real_native.MAX_COMM_BLOCKS, real_native.MAX_PEERS

        def run_op(self, op, stream, device):
            op.run(current["opt"])

        def __getattr__(self, name):
            return getattr(real_native, name)

    def build(rule, state=None, **kw):
        torch.manual_seed(5)
        model = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.Flatten(), torch.nn.Linear(8 * 36, 5)).to(memory_format=torch.channels_last)
        opt = _make(rule, _groups(model), **kw)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        impl, ddp = model.bagua_ddp.bagua_algorithm, model.bagua_ddp
        impl._carry_state_over()
        if state is not None:
            opt.load_state_dict(state)
        current["opt"] = opt
        for bucket in model.bagua_buckets:
            nbytes = bucket.backend_tensor.numel() * bucket.backend_tensor.element_size()
            bucket._engine = lambda group=None: Engine()
            bucket._slice = Slice(nbytes)
            bucket.backend_bucket = BackendBucket()
            impl.init_operations(ddp, bucket)
        model.bagua_ddp._fwd_pre_hook = impl.init_forward_pre_hook(ddp)
        opt._gather = lambda t, group: [t]
        return model, opt

    bagua.init_process_group()
    core_native, cur_stream = core.native, torch.cuda.current_stream
    core.native = lambda: FakeC()
    torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
    try:
        for rule in RULES:
            for kw in ({}, {"loss_scaling": True}):
                # without ema_decay: no EMA state, no op, the parent's launch counts
                model, opt = build(rule, **kw)
                bk, nb = opt._bucketing, len(model.bagua_buckets)
                assert bk.ema is None and all("publish" not in rec for rec in bk.shards)
                assert all(len(rec["state"]) == (3 if rule in ("adam", "lamb") else 2) for rec in bk.shards)
                base_native = opt.native_ops_in_step
                launches = opt.kernel_launches
                opt.step()
                base = opt.kernel_launches - launches
                with pytest.raises(RuntimeError, match="ema_decay"):
                    with opt.ema_weights():
                        pass
                plain_sd = opt.state_dict()
                assert "ema_calls" not in plain_sd and all("ema" not in st for st in plain_sd["state"].values())

                # with it: an EMA shard per bucket next to the master, one table over all of them, two publish ops per bucket
                model, opt = build(rule, ema_decay=0.999, **kw)
                bk = opt._bucketing
                assert opt.native_ops_in_step and (base_native or rule in ("sgd", "adam"))
                for rec in bk.shards:
                    master, ema = rec["state"][0], rec["state"][-1]
                    assert ema.shape == master.shape and torch.equal(ema, master) and ema.data_ptr() != master.data_ptr()
                    to_ema, to_master = rec["publish"]
                    assert isinstance(to_ema, Publish) and to_ema.args[5] == ema.data_ptr() and to_master.args[5] == master.data_ptr()
                    assert to_ema.args[3] == rec["numel"] * rec["weights"].element_size()
                plan = bk.ema["plan"]
                assert [t.data_ptr() for t in plan.keep[0]] == [rec["state"][0].data_ptr() for rec in bk.shards]
                assert [t.data_ptr() for t in plan.keep[1]] == [rec["state"][-1].data_ptr() for rec in bk.shards]
                vote = bk.ema["op"].args[8]
                assert vote == (bk.clip["out"][2:].data_ptr() if kw else 0), "the vote is handed to the EMA only with loss scaling"
                assert bk.ema["op"].args[7] == pytest.approx(0.001)
                # +1 launch per EMA step
                events.clear()
                launches = opt.kernel_launches
                opt.step()
                assert opt.kernel_launches - launches == base + 1 and events[-1] == "Ema"
                assert bk.ema["op"].w == 1.0 - 0.999
                opt.ema_decay = 0.99                     # a user-side warm-up: the next update takes the new value
                opt.step()
                assert bk.ema["op"].w == 1.0 - 0.99
                # ema_weights(): one publish per bucket on entry and one on exit; step() inside raises
                events.clear()
                launches = opt.kernel_launches
                with opt.ema_weights():
                    assert events == ["Publish"] * nb
                    with pytest.raises(RuntimeError, match="ema_weights"):
                        opt.step()
                assert events == ["Publish"] * (2 * nb) and opt.kernel_launches - launches == 2 * nb
                ran = [rec["publish"][0].s + rec["publish"][1].s for rec in bk.shards]
                assert ran == [2] * nb
                with pytest.raises(NotImplementedError):
                    GraphedTrainStep(model, lambda x: x.sum(), (torch.zeros(1),), optimizers=[opt])

                # ema_every = 3: +1 on every third step() only
                model, opt = build(rule, ema_decay=0.9, ema_every=3, **kw)
                counts = []
                for _ in range(6):
                    launches = opt.kernel_launches
                    opt.step()
                    counts.append(opt.kernel_launches - launches - base)
                assert counts == [0, 0, 1, 0, 0, 1]

            # the load matrix: "ema" in the checkpoint or not, EMA in the optimizer or not
            model, opt = build(rule, ema_decay=0.9)
            for rec in opt._bucketing.shards:
                rec["state"][0].normal_()
                rec["state"][-1].normal_()
            sd = opt.state_dict()
            assert all(set(st) >= {"master", "ema"} for st in sd["state"].values())
            ema_sd = opt.ema_state_dict()
            assert list(ema_sd) == [n for n, _ in model.named_parameters()]
            for name, t in ema_sd.items():
                assert torch.equal(t, sd["state"][name]["ema"])
            # with EMA ← with "ema": the EMA continues
            _, o2 = build(rule, state=sd, ema_decay=0.9)
            assert all(torch.equal(t, ema_sd[n]) for n, t in o2.ema_state_dict().items())
            # without EMA ← with "ema": ignored
            _, o3 = build(rule, state=sd)
            assert all(len(rec["state"]) == len(o3._state_keys()) for rec in o3._bucketing.shards)
            assert all("ema" not in st for st in o3.state_dict()["state"].values())
            # with EMA ← without "ema": the EMA starts from the loaded master
            plain = {**sd, "state": {n: {k: v for k, v in st.items() if k != "ema"} for n, st in sd["state"].items()}}
            del plain["ema_calls"]
            _, o4 = build(rule, state=plain, ema_decay=0.9)
            assert all(torch.equal(rec["state"][-1], rec["state"][0]) for rec in o4._bucketing.shards)
            assert all(torch.equal(t, sd["state"][n]["master"]) for n, t in o4.ema_state_dict().items())
            # refresh_master_weights(): the EMA restarts from the refreshed master
            opt.refresh_master_weights()
            assert all(torch.equal(rec["state"][-1], rec["state"][0]) for rec in opt._bucketing.shards)
        with pytest.raises(ValueError, match="ema_decay"):
            _make("sgd", _net().parameters(), ema_decay=1.0)
        with pytest.raises(ValueError, match="ema_every"):
            _make("sgd", _net().parameters(), ema_decay=0.9, ema_every=0)
    finally:
        core.native, torch.cuda.current_stream = core_native, cur_stream
    return True


def test_ema_driver_with_host_doubles():
    assert all(run_distributed(_host_double_worker, world=1))


def _fallback_worker(rank, world, rule, decay, ckpt):
    """4 steps on the gloo fallback with an EMA, the masters saved after every step, the EMA compared with their fp32 replay and with
    ``AveragedModel`` on fp32 copies; ``ema_weights()`` swaps the EMA in and the live weights back; the state is saved for 3 ranks."""
    import torch.nn.functional as F
    from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    torch.manual_seed(3)
    base = _net()
    names = [n for n, _ in base.named_parameters()]
    averaged = AveragedModel(copy.deepcopy(base), multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=False)
    averaged.update_parameters(base)   # the EMA starts at the initial weights
    model = copy.deepcopy(base)
    opt = _make(rule, _groups(model), ema_decay=decay)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    replay = {n: p.detach().clone() for n, p in model.named_parameters()}
    for it in range(4):
        opt.zero_grad()
        x, y = _batch(rank, it)
        F.cross_entropy(model(x), y).backward()
        opt.step()
        replay = {n: _replay(replay[n], p.detach(), decay) for n, p in model.named_parameters()}
        averaged.update_parameters(model)
    got = opt.ema_state_dict()
    assert list(got) == names
    for n in names:
        assert torch.equal(got[n], replay[n]), n
        assert not torch.equal(got[n], dict(model.named_parameters())[n].detach()), "the EMA must lag the weights"
    avg = dict(averaged.module.named_parameters())
    gap = max(float((got[n] - avg[n].detach()).abs().max()) for n in names)
    assert gap <= 1e-6, gap   # torch's lerp may fuse its product and sum: a few ulp apart
    live = {n: p.detach().clone() for n, p in model.named_parameters()}
    with opt.ema_weights():
        for n, p in model.named_parameters():
            assert torch.equal(p.detach(), got[n])
        with pytest.raises(RuntimeError):
            opt.step()
    for n, p in model.named_parameters():
        assert torch.equal(p.detach(), live[n])
    sd = opt.state_dict()
    if rank == 0:
        torch.save({"model": model.state_dict(), "opt": sd, "ema": got}, ckpt)
    return True


def _resume_worker(rank, world, rule, decay, ckpt):
    """3 ranks read the 2-rank checkpoint: the EMA comes back bit for bit and continues as the fp32 replay over the new masters."""
    import torch.nn.functional as F

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    saved = torch.load(ckpt)
    model = _net()
    model.load_state_dict(saved["model"])
    opt = _make(rule, _groups(model), ema_decay=decay)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    opt.load_state_dict(saved["opt"])
    got = opt.ema_state_dict()
    for n, t in saved["ema"].items():
        assert torch.equal(got[n], t), n
    replay = dict(got)
    for it in range(3):
        opt.zero_grad()
        x, y = _batch(rank, 10 + it)
        F.cross_entropy(model(x), y).backward()
        opt.step()
        replay = {n: _replay(replay[n], p.detach(), decay) for n, p in model.named_parameters()}
    for n, t in opt.ema_state_dict().items():
        assert torch.equal(t, replay[n]), n
    return True


@pytest.mark.parametrize("rule", ["sgd", "adam"])
def test_fallback_ema_matches_fp32_replay_and_averaged_model(rule, tmp_path):
    ckpt = str(tmp_path / "ckpt.pt")
    assert all(run_distributed(_fallback_worker, world=2, args=(rule, 0.75, ckpt)))
    assert all(run_distributed(_resume_worker, world=3, args=(rule, 0.75, ckpt)))


def test_imagenet_example_with_ema(tmp_path):
    from tests.mp_utils import free_port, run_in_session

    env = dict(os.environ, PYTHONPATH=REPO + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="", BAGUA_FORCE_CPU="1")
    cmd = [sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={free_port()}",
           os.path.join(REPO, "examples/imagenet/main.py"), "--cpu", "--synthetic", "--epochs", "1", "--steps-per-epoch", "2", "--batch-size", "2",
           "--num-classes", "10", "--image-size", "32", "--print-freq", "1", "--fused-shard", "--ema-decay", "0.9", "--ema-every", "1",
           "--save-checkpoint", "--checkpoint-dir", str(tmp_path)]
    r = run_in_session(cmd, 240, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "EMA Acc@1" in r.stdout, r.stdout[-2000:]
    ck = torch.load(str(tmp_path / "checkpoint.pth.tar"), map_location="cpu", weights_only=False)
    assert ck["optimizer"]["ema_calls"] == 2 and all("ema" in st for st in ck["optimizer"]["state"].values())
