"""The weight EMA of the in-bucket sharded optimizers (``ema_decay``) on the GPU.

* ``multi_tensor_ema_kernel`` bit for bit against the host fp32 emulation, on aligned and misaligned views with sentinel margins,
  and with a set vote.
* ``shard_publish_kernel`` on virtual peer worlds of P = 1 … 8 ranks in fp32, bf16 and fp16: every rank's weights are the rounded
  consolidated shard, the margins untouched.
* ``make_sharded_fused_{sgd,adam,lamb,lars}(ema_decay=...)`` end to end in self-peer mode: the weights are those of the run without
  the EMA, the EMA is the fp32 replay over that run's masters, ``ema_weights()`` swaps it in and the live weights back, a resumed
  checkpoint and a re-bucketing continue bit-identically, a skipped loss-scaled step leaves it alone, and a parameter outside the
  buckets has one too.
"""
import copy

import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_virtual_peer_gpu import _code, _shard, _world

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


def _replay(e, m, decay):
    """e + w·(m − e) in three separately rounded fp32 operations on the CPU."""
    w = torch.tensor(1.0 - float(decay), dtype=torch.float32)
    return e + torch.mul(torch.sub(m, e), w)


SIZES = [0, 1, 65535, 65536, 65537, 2 * 65536 + 3]


@pytest.mark.parametrize("shift", [0, 1, 3])
def test_ema_kernel_matches_fp32_emulation(C, shift):
    from bagua_b200.ops.optim import multi_tensor_plan

    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(11 + shift)
    M = 8
    srcs, emas, bases = [], [], []
    for i, n in enumerate(SIZES):
        sb = torch.randn(n + 2 * M, generator=gen)
        eb = torch.randn(n + 2 * M, generator=gen)
        eb[:M + shift] = float("nan")                 # sentinels around the EMA view
        eb[M + shift + n:] = float("nan")
        # shift 0: 16-byte aligned views; 1, 3: misaligned EMA (and source when i is odd) take the scalar path
        so = M + (shift if i % 2 else 0)
        s, e = sb.to(dev), eb.to(dev)
        bases.append((s, e, eb.clone(), sb[so:so + n].clone()))
        srcs.append(s[so:so + n])
        emas.append(e[M + shift:M + shift + n])
    plan = multi_tensor_plan([srcs, emas])
    vote = torch.zeros(1, device=dev)
    decay = 0.9999
    op = C.EmaOp(*plan.args(), 1.0 - decay, vote.data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(2):
        C.run_op(op, stream, 0)
    torch.cuda.synchronize()
    for (s, e, eb, m), n in zip(bases, SIZES):
        want = eb.clone()
        view = want[M + shift:M + shift + n]
        for _ in range(2):
            view.copy_(_replay(view, m, decay))
        got = e.cpu()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), n
    before = [e.clone() for _, e, _, _ in bases]
    vote.fill_(1.0)                                     # an overflowed step: nothing is written
    C.run_op(op, stream, 0)
    torch.cuda.synchronize()
    assert all(torch.equal(a.view(torch.int32), e.view(torch.int32)) for a, (_, e, _, _) in zip(before, bases))


@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_shard_publish_rounds_the_consolidated_shard(C, P, dtype):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 15) + 16 // es * 3
    nbytes = numel * es
    off = 1024                                          # a leading margin; the allocation rounds up: a trailing one too
    weights = w.alloc(off + nbytes + 1024)
    for r in range(P):
        weights.view(r, torch.uint8).fill_(0xA5)
    gen = torch.Generator().manual_seed(P)
    full = torch.randn(numel, generator=gen) * 3
    srcs = []
    for r in range(P):
        lo, hi, length = _shard(numel, es, P, r)
        s = torch.full((length,), float("nan"))
        s[: hi - lo] = full[lo:hi]
        srcs.append(s.to(w.device))
    cfg = w.cfg(6)
    w.run(None, ops=[C.ShardPublishOp(w.comms[r], weights.buf, off, nbytes, _code(dtype), srcs[r].data_ptr(), False, cfg) for r in range(P)])
    want = full.to(dtype)
    for r in range(P):
        raw = weights.view(r, torch.uint8)
        assert torch.equal(raw[off:off + nbytes].view(dtype).cpu().view(torch.uint8), want.view(torch.uint8)), (P, dtype, r)
        assert bool((raw[:off] == 0xA5).all()) and bool((raw[off + nbytes:] == 0xA5).all()), "the margins must stay untouched"


# ---------------------------------------------------------------------------------------------------------------------
# end to end, self-peer (world 1) and real peers
# ---------------------------------------------------------------------------------------------------------------------
def _groups(ps):
    return [{"params": [p for p in ps if p.dim() > 1], "weight_decay": 0.01}, {"params": [p for p in ps if p.dim() <= 1], "weight_decay": 0.0}]


def _make(rule, ps, **kw):
    from bagua_b200.parallel.algorithms import gradient_allreduce as ga

    if rule == "sgd":
        return ga.make_sharded_fused_sgd(_groups(ps), lr=0.05, momentum=0.9, **kw)
    if rule == "adamw":
        return ga.make_sharded_fused_adam(_groups(ps), lr=1e-3, adamw=True, **kw)
    if rule == "lamb":
        return ga.make_sharded_fused_lamb(_groups(ps), lr=1e-3, **kw)
    return ga.make_sharded_fused_lars(_groups(ps), lr=0.5, trust_coefficient=0.02, **kw)


def _net(dev, dtype):
    import torch.nn as nn

    return nn.Sequential(nn.Conv2d(3, 16, 3), nn.ReLU(), nn.Flatten(), nn.Linear(16 * 100, 32)).to(dev).to(dtype).to(memory_format=torch.channels_last)


def _batch(dev, rank, it, k, dtype):
    g = torch.Generator(device=dev).manual_seed(1000 * it + 10 * k + rank)
    return torch.randn(8, 3, 12, 12, device=dev, generator=g).to(dtype).to(memory_format=torch.channels_last)


def _flat(m):
    return torch.cat([p.detach().reshape(-1).float() for p in m.parameters()])


def _train_worker(rank, world, rule, bound, K, every):
    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    dev, dtype, decay, steps = torch.device("cuda", rank), torch.bfloat16, 0.8, 6
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.manual_seed(9)
    base = _net(dev, dtype)

    def build(ema, state=None, model_sd=None):
        m = copy.deepcopy(base)
        if model_sd is not None:
            m.load_state_dict(model_sd)
        kw = {"ema_decay": decay, "ema_every": every} if ema else {}
        o = _make(rule, list(m.parameters()), max_grad_norm=bound, accumulate_grads=K > 1, **kw)
        if state is not None:
            o.load_state_dict(state)
        return m.with_bagua([o], FusedGradientAllReduceAlgorithm(o)), o

    def train(m, o, its, after=None):
        for it in its:
            o.zero_grad()
            for k in range(K):
                m(_batch(dev, rank, it, k, dtype)).float().pow(2).mean().div(K).backward()
            o.step()
            if after is not None:
                after(it)

    # the run without the EMA, its consolidated masters after every step
    m0, o0 = build(False)
    names = [n for n, _ in m0.named_parameters()]
    masters, weights = [], []
    train(m0, o0, range(steps), lambda it: (masters.append({n: t["master"] for n, t in o0.state_dict()["state"].items()}), weights.append(_flat(m0))))
    torch.cuda.synchronize()
    replay = [{n: p.detach().float().cpu() for n, p in base.named_parameters()}]
    for it in range(steps):
        replay.append({n: _replay(replay[-1][n], masters[it][n], decay) if (it + 1) % every == 0 else replay[-1][n] for n in names})

    # 1, 2: the same weights, and the EMA is the replay over the masters
    m1, o1 = build(True)
    seen = []
    train(m1, o1, range(3), lambda it: seen.append((_flat(m1), o1.ema_state_dict())))
    for it, (wts, ema) in enumerate(seen):
        assert torch.equal(wts, weights[it]), f"the EMA changed the weights at step {it}"
        assert list(ema) == names and all(torch.equal(ema[n], replay[it + 1][n]) for n in names), f"EMA ≠ fp32 replay at step {it}"
    # 3: inside ema_weights() the parameters are the EMA rounded once; after it the live weights are back, training continues unchanged
    live = [p.detach().clone() for p in m1.parameters()]
    with o1.ema_weights():
        for n, p in m1.named_parameters():
            assert torch.equal(p.detach().float().cpu(), replay[3][n].to(dtype).float()), n
        with pytest.raises(RuntimeError, match="ema_weights"):
            o1.step()
    assert all(torch.equal(a, p.detach()) for a, p in zip(live, m1.parameters()))
    sd, msd = copy.deepcopy(o1.state_dict()), {k: v.clone() for k, v in m1.state_dict().items()}
    train(m1, o1, range(3, steps))
    torch.cuda.synchronize()
    assert torch.equal(_flat(m1), weights[-1]) and all(torch.equal(t, replay[-1][n]) for n, t in o1.ema_state_dict().items())

    # 4: a resumed checkpoint and a re-bucketing continue bit-identically
    m2, o2 = build(True, state=sd, model_sd=msd)
    train(m2, o2, range(3, steps))
    m3, o3 = build(True)
    train(m3, o3, range(2))
    m3.bagua_ddp._reset_buckets()
    train(m3, o3, range(2, steps))
    torch.cuda.synchronize()
    for m, o in ((m2, o2), (m3, o3)):
        assert torch.equal(_flat(m), weights[-1])
        assert all(torch.equal(t, replay[-1][n]) for n, t in o.ema_state_dict().items())
    return _flat(m1).cpu()


@pytest.mark.parametrize("bound", [None, 0.05])
@pytest.mark.parametrize("rule", ["sgd", "adamw", "lamb", "lars"])
def test_self_peer_ema_is_the_fp32_replay(rule, bound):
    run_distributed(_train_worker, world=1, args=(rule, bound, 1, 1), use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


def test_self_peer_ema_with_accumulation():
    run_distributed(_train_worker, world=1, args=("adamw", None, 4, 2), use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


def _loss_scale_worker(rank, world):
    """fp16 with ShardedGradScaler: the step with an injected inf is skipped and leaves every EMA bit alone; the others move it."""
    import bagua_b200 as bagua
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.manual_seed(4)
    model = _net(dev, torch.float16)
    opt = _make("sgd", list(model.parameters()), loss_scaling=True, ema_decay=0.9)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    sc = ShardedGradScaler(init_scale=1024.0, growth_interval=100)
    moved = []
    for it in range(4):
        before = opt.ema_state_dict()
        opt.zero_grad()
        loss = model(_batch(dev, rank, it, 0, torch.float16)).float().pow(2).mean()
        if it == 1:
            loss = loss * float("inf")
        sc.scale(loss).backward()
        sc.step(opt)
        sc.update()
        after = opt.ema_state_dict()
        moved.append(any(not torch.equal(before[n], after[n]) for n in after))
    assert moved == [True, False, True, True]
    return True


def test_loss_scaled_skip_leaves_the_ema_alone():
    run_distributed(_loss_scale_worker, world=1, use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


def _uncovered_worker(rank, world):
    """A parameter the engine ignores (outside the buckets) keeps a local EMA of its fp32 master: the same replay, swapped in and out."""
    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    dev, dtype, decay = torch.device("cuda", rank), torch.bfloat16, 0.7
    torch.manual_seed(5)
    model = _net(dev, dtype)
    model._bagua_params_and_buffers_to_ignore = ["3.bias"]
    opt = _make("adamw", list(model.parameters()), ema_decay=decay)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    bias = dict(model.named_parameters())["3.bias"]
    assert id(bias) not in opt._bucketing.covered
    want = bias.detach().float().cpu()
    for it in range(3):
        opt.zero_grad()
        model(_batch(dev, rank, it, 0, dtype)).float().pow(2).mean().backward()
        opt.step()
        want = _replay(want, opt.state[bias]["master"].cpu(), decay)
    got = opt.ema_state_dict()["3.bias"]
    assert torch.equal(got, want)
    live = bias.detach().clone()
    with opt.ema_weights():
        assert torch.equal(bias.detach().float().cpu(), want.to(dtype).float())
    assert torch.equal(bias.detach(), live)
    return True


def test_parameter_outside_the_buckets_has_an_ema():
    run_distributed(_uncovered_worker, world=1, use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
@pytest.mark.parametrize("rule", ["adamw", "lars"])
def test_ema_on_real_peers(rule):
    n = min(torch.cuda.device_count(), 8)
    res = run_distributed(_train_worker, world=n, args=(rule, 0.05, 1, 1), use_cuda=True, timeout=300)
    for r in res[1:]:
        assert torch.equal(r, res[0]), "every rank must hold the same weights"
