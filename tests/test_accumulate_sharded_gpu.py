"""Gradient accumulation in the fp32 shard of the in-bucket sharded optimizers (``accumulate_grads=True``) on the GPU.

* ``shard_grad_kernel``'s ACCUM flavour on virtual peer worlds of P = 1 … 8 ranks against the bit-exact fp32 oracle
  ``s_k = fl32(s_{k−1} + red_k)``, with its partial sums, the cleared bucket and restart().
* ``make_sharded_fused_{sgd,adam,lamb,lars}(accumulate_grads=True)`` end to end in self-peer mode: K micro-batches against the
  reference optimizer on the fp32 sum of the micro-batch gradients, bit-identity with the program without the flag at K = 1,
  the precision that bf16 local accumulation loses, loss scaling with a skipped step, discards, re-bucketing and resuming.
"""
import copy

import numpy as np
import pytest
import torch

from tests.mp_utils import run_distributed
from tests.test_virtual_peer_gpu import _code, _f32, _owned_slice_sum, _shard, _world

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 3, 4, 8]


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("K", [1, 2, 5])
def test_accumulating_phase_a_matches_fp32_oracle(C, P, dtype, K):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 15) + 16 // es * 3          # not a multiple of P·vector: slices of unequal length, a padded tail
    nbytes = numel * es
    grads = w.alloc(nbytes)
    cfg = w.cfg(6)
    ranks = []
    for r in range(P):
        lo, hi, length = _shard(numel, es, P, r)
        shard = torch.full((length,), float("nan"), device=w.device)   # the first launch must overwrite whatever is there
        partials = torch.zeros(C.MAX_COMM_BLOCKS, dtype=torch.float64, device=w.device)
        op = C.ShardGradOp(w.comms[r], grads.buf, 0, nbytes, _code(dtype), shard.data_ptr(), partials.data_ptr(), _f32(1.0 / P).item(), True, False, cfg,
                           accumulate=True)
        ranks.append((lo, hi, shard, partials, op))
    gen = torch.Generator().manual_seed(7 + P + K)
    want = None
    for k in range(K + 1):
        if k == K:   # after restart() the next launch overwrites again
            for *_, op in ranks:
                op.restart()
            want = None
        gs = [(torch.randn(numel, generator=gen) * (k + 1)).to(dtype) for _ in range(P)]
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r].to(w.device))
        red = _owned_slice_sum(gs, _f32(1.0 / P))
        want = red if want is None else want + red          # fp32 adds on the CPU: correctly rounded, no FMA
        assert all(op.pending() == (k > 0 and k != K) for *_, op in ranks)
        w.run(None, ops=[op for *_, op in ranks])
        for r, (lo, hi, shard, partials, op) in enumerate(ranks):
            got = shard[: hi - lo].cpu()
            assert torch.equal(got.view(torch.int32), want[lo:hi].view(torch.int32)), (P, dtype, K, k, r)
            ss = float(got.double().square().sum())
            assert float(partials.sum()) == pytest.approx(ss, rel=1e-12, abs=1e-300), (P, dtype, k, r)
            assert torch.count_nonzero(grads.view(r, torch.uint8, nbytes)).item() == 0, "the bucket must be cleared after every launch"
            assert op.pending()
    if K == 1:   # one launch of an accumulating op is the non-accumulating kernel, bit for bit
        gs = [torch.randn(numel, generator=gen).to(dtype) for _ in range(P)]
        outs = []
        for accumulate in (True, False):
            shards = []
            ops = []
            for r in range(P):
                lo, hi, length = _shard(numel, es, P, r)
                s = torch.zeros(length, device=w.device)
                p = torch.zeros(C.MAX_COMM_BLOCKS, dtype=torch.float64, device=w.device)
                ops.append(C.ShardGradOp(w.comms[r], grads.buf, 0, nbytes, _code(dtype), s.data_ptr(), p.data_ptr(), 1.0 / P, True, False, cfg, accumulate))
                shards.append((s, p))
                grads.view(r, dtype, numel).copy_(gs[r].to(w.device))
            w.run(None, ops=ops)
            outs.append([(s.cpu(), p.cpu()) for s, p in shards])
        for (a, pa), (b, pb) in zip(*outs):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)) and torch.equal(pa, pb)


# ---------------------------------------------------------------------------------------------------------------------
# end to end, self-peer (world 1) and real peers
# ---------------------------------------------------------------------------------------------------------------------
def _groups(ps):
    return [{"params": [p for p in ps if p.dim() > 1], "weight_decay": 0.01}, {"params": [p for p in ps if p.dim() <= 1], "weight_decay": 0.0}]


def _make(rule, ps, **kw):
    from bagua_b200.parallel.algorithms import gradient_allreduce as ga

    if rule == "sgd":
        return ga.make_sharded_fused_sgd(_groups(ps), lr=0.05, momentum=0.9, nesterov=True, **kw)
    if rule == "adamw":
        return ga.make_sharded_fused_adam(_groups(ps), lr=1e-3, adamw=True, **kw)
    if rule == "lamb":
        return ga.make_sharded_fused_lamb(_groups(ps), lr=1e-3, **kw)
    return ga.make_sharded_fused_lars(_groups(ps), lr=0.5, trust_coefficient=0.02, **kw)


def _reference(rule, ps):
    """The optimizer the sharded rule is checked against on the summed gradient (torch for SGD / AdamW; the flat fused LAMB / LARS,
    themselves checked against the float64 oracles in tests/test_lamb_gpu.py and tests/test_lars_gpu.py)."""
    from bagua_b200.ops.optim import FusedLAMB, FusedLARS

    if rule == "sgd":
        return torch.optim.SGD(_groups(ps), lr=0.05, momentum=0.9, nesterov=True)
    if rule == "adamw":
        return torch.optim.AdamW(_groups(ps), lr=1e-3)
    if rule == "lamb":
        return FusedLAMB(_groups(ps), lr=1e-3)
    return FusedLARS(_groups(ps), lr=0.5, trust_coefficient=0.02)


def _net(dev):
    import torch.nn as nn

    return nn.Sequential(nn.Conv2d(3, 16, 3), nn.ReLU(), nn.Flatten(), nn.Linear(16 * 100, 32)).to(dev).to(memory_format=torch.channels_last)


def _batch(dev, rank, it, k):
    g = torch.Generator(device=dev).manual_seed(1000 * it + 10 * k + rank)
    return torch.randn(8, 3, 12, 12, device=dev, generator=g).to(memory_format=torch.channels_last)


def _flat(m):
    return torch.cat([p.detach().reshape(-1).float() for p in m.parameters()])


def _train(m, o, its, K, rank, reset_at=None, discard_at=None):
    dev = next(m.parameters()).device
    for it in its:
        o.zero_grad()
        if discard_at == it:     # a sum discarded by zero_grad() mid-accumulation
            m(_batch(dev, rank, it, 99)).float().pow(2).mean().backward()
            o.zero_grad()
        for k in range(K):
            if reset_at == (it, k):
                m.bagua_ddp._reset_buckets()
            m(_batch(dev, rank, it, k)).float().pow(2).mean().div(K).backward()
        o.step()


def _accum_train_worker(rank, world, rule, bound, K):
    """K micro-batches per step for 6 steps against the reference on the fp32 sum of the micro-batch gradients (averaged over the
    ranks); K = 1: bit-identical to the program without the flag; mid-run re-bucketing, a discarded sum and a resumed checkpoint."""
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.manual_seed(9)
    base = _net(dev)

    def build(accum, b=bound, state=None, model_sd=None):
        m = copy.deepcopy(base)
        if model_sd is not None:
            m.load_state_dict(model_sd)
        o = _make(rule, list(m.parameters()), max_grad_norm=b, accumulate_grads=accum)
        if state is not None:
            o.load_state_dict(state)
        m = m.with_bagua([o], FusedGradientAllReduceAlgorithm(o))
        assert all(("_accum_" in bk.allreduce_variant) == accum for bk in m.bagua_buckets), [bk.allreduce_variant for bk in m.bagua_buckets]
        return m, o

    # against the reference on the summed gradient
    model, opt = build(True)
    _train(model, opt, range(6), K, rank)
    torch.cuda.synchronize()
    got = _flat(model)
    oracle = copy.deepcopy(base)
    oopt = _reference(rule, list(oracle.parameters()))
    for it in range(6):
        oopt.zero_grad()
        for k in range(K):
            oracle(_batch(dev, rank, it, k)).pow(2).mean().div(K).backward()
        for p in oracle.parameters():
            if world > 1:
                dist.all_reduce(p.grad)
                p.grad /= world
        if bound is not None:
            torch.nn.utils.clip_grad_norm_(oracle.parameters(), bound)
        oopt.step()
    want = _flat(oracle)
    torch.testing.assert_close(got, want, rtol=2e-4, atol=2e-5)
    assert not torch.equal(got, _flat(base))

    # re-bucketing between micro-batches, and a discarded partial sum, leave the result unchanged
    m2, o2 = build(True)
    _train(m2, o2, range(6), K, rank, reset_at=(2, K // 2), discard_at=4)
    torch.cuda.synchronize()
    assert torch.equal(_flat(m2), got), "re-bucketing or a discarded sum changed the result"

    # a checkpoint at a step boundary resumes bit-identically
    m3, o3 = build(True)
    _train(m3, o3, range(3), K, rank)
    sd, msd = copy.deepcopy(o3.state_dict()), {k: v.clone() for k, v in m3.state_dict().items()}
    m4, o4 = build(True, state=sd, model_sd=msd)
    _train(m4, o4, range(3, 6), K, rank)
    torch.cuda.synchronize()
    assert torch.equal(_flat(m4), got), "a resumed checkpoint must continue bit-identically"

    if K == 1:   # one micro-batch per step: exactly the program without the flag (SGD / Adam: both multiply by 1.0 then)
        m5, o5 = build(False, b=1e30 if bound is None and rule in ("sgd", "adamw") else bound)
        _train(m5, o5, range(6), 1, rank)
        torch.cuda.synchronize()
        assert torch.equal(_flat(m5), got), "K = 1 must be bit-identical to the program without accumulate_grads"
    return got.cpu()


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("bound", [None, 0.05])
@pytest.mark.parametrize("rule", ["sgd", "adamw", "lamb", "lars"])
def test_self_peer_accumulation_matches_reference(rule, bound, K):
    run_distributed(_accum_train_worker, world=1, args=(rule, bound, K), use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


def _precision_worker(rank, world):
    """bf16 weights, K = 16 micro-batches: the first contributes 1.0 per element, the others 2⁻⁹, below half a bf16 ulp of 1.0.
    Local accumulation in the bucket (no_sync) loses all of them; the fp32 shard keeps them."""
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_sgd

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    K, n = 16, 256
    exact = 1.0 + (K - 1) * 2.0 ** -9
    out = {}
    class Scaled(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.zeros(n, device=dev, dtype=torch.bfloat16))

        def forward(self, c):
            return (self.w.float() * c).sum()

    for accum in (False, True):
        model = Scaled()
        opt = make_sharded_fused_sgd([model.w], lr=0.0, max_grad_norm=1e30, accumulate_grads=accum)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        opt.zero_grad()
        for k in range(K):
            c = 1.0 if k == 0 else 2.0 ** -9
            model.bagua_ddp.require_backward_grad_sync = accum or k == K - 1
            model(c).backward()
        torch.cuda.synchronize()
        rec = opt._bucketing.shards[0]
        got = rec["shard"][: rec["hi"] - rec["lo"]][:n].double().cpu()
        opt.step()
        torch.cuda.synchronize()
        out[accum] = (got, float(opt.last_grad_norm))
    bound = K * np.finfo(np.float32).eps * exact     # fp32 summation error of K terms
    assert (out[False][0] - exact).abs().max().item() > bound, "bf16 local accumulation was expected to drop the small terms"
    assert (out[True][0] - exact).abs().max().item() <= bound
    assert out[True][1] == pytest.approx(exact * n ** 0.5, rel=1e-6)
    return True


def test_fp32_shard_keeps_what_bf16_local_accumulation_drops():
    run_distributed(_precision_worker, world=1, use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


def _loss_scale_worker(rank, world):
    """fp16, K = 3, ShardedGradScaler: an inf in micro-batch 2 of step 1 skips that step on every rank and backs the scale off; the
    next step starts from an empty sum; the run otherwise matches stock GradScaler + SGD on the fp32 master copy."""
    import bagua_b200 as bagua
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.manual_seed(4)
    base = _net(dev)
    K, INIT = 3, 1024.0
    model = copy.deepcopy(base).half()
    opt = _make("sgd", list(model.parameters()), loss_scaling=True, accumulate_grads=True)
    model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
    sc = ShardedGradScaler(init_scale=INIT, growth_interval=100)
    oracle = copy.deepcopy(base)
    oopt = _reference("sgd", list(oracle.parameters()))
    osc = torch.amp.GradScaler("cuda", init_scale=INIT, growth_interval=100)
    skipped, scales = [], []
    for it in range(4):
        before = _flat(model)
        opt.zero_grad()
        oopt.zero_grad()
        for k in range(K):
            x = _batch(dev, rank, it, k)
            loss = model(x.half()).float().pow(2).mean() / K
            oloss = oracle(x).pow(2).mean() / K
            if it == 1 and k == 1:
                loss = loss * float("inf")
                oloss = oloss * float("inf")
            sc.scale(loss).backward()
            osc.scale(oloss).backward()
        sc.step(opt)
        sc.update()
        osc.step(oopt)
        osc.update()
        torch.cuda.synchronize()
        skipped.append(float(opt.last_step_skipped))
        scales.append((sc.get_scale(), osc.get_scale()))
        if it == 1:
            assert torch.equal(_flat(model), before), "a skipped step must not change any weight"
    assert skipped == [0.0, 1.0, 0.0, 0.0]
    assert all(a == b for a, b in scales) and scales[1][0] == INIT / 2
    sd = opt.state_dict()
    masters = torch.cat([sd["state"][n]["master"].reshape(-1).to(dev) for n, _ in model.named_parameters()])
    torch.testing.assert_close(masters, _flat(oracle), rtol=2e-3, atol=2e-3)
    return True


def test_loss_scaled_accumulation_skips_and_restarts():
    run_distributed(_loss_scale_worker, world=1, use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
@pytest.mark.parametrize("rule", ["adamw", "lamb"])
def test_accumulation_on_real_peers(rule):
    n = min(torch.cuda.device_count(), 8)
    res = run_distributed(_accum_train_worker, world=n, args=(rule, 0.05, 4), use_cuda=True, timeout=300)
    for r in res[1:]:
        assert torch.equal(r, res[0]), "every rank must hold the same weights"
