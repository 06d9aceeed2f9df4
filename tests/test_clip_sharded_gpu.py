"""Global-norm clipping of the in-bucket optimizers on the GPU.

* The three kernels (phase A ``shard_grad``, the norm exchange ``grad_norm``, phase B ``shard_sgd`` / ``shard_adam``) on virtual
  peer worlds of P = 1 … 8 ranks against fixed-order fp32 / float64 oracles.
* ``make_sharded_fused_{sgd,adam}(max_grad_norm=…)`` end to end in self-peer mode (and on 2+ real GPUs) against torch's
  ``clip_grad_norm_`` + SGD / AdamW, with a checkpoint resumed mid-run.
"""
import copy
import math

import numpy as np
import pytest
import torch

from tests import optim_oracle as oo
from tests.mp_utils import run_distributed
from tests.test_virtual_peer_gpu import _code, _f32, _owned_slice_sum, _shard, _world

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 3, 4, 8]


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


def _torch_coef(total: torch.Tensor, max_norm: float) -> torch.Tensor:
    return torch.clamp(max_norm / (total + 1e-6), max=1.0)   # torch.nn.utils.clip_grad_norm_'s formula, fp32


class _Rank:
    """One virtual rank's buffers of the clipped two-phase update of a single bucket."""

    def __init__(self, C, w, r, kind, dtype, numel, grads, weights, box, w0, cfg):
        es = torch.empty(0, dtype=dtype).element_size()
        P = w.world
        self.lo, self.hi, length = _shard(numel, es, P, r)
        dev = w.device
        self.shard = torch.zeros(length, device=dev)
        self.partials = torch.zeros(1, C.MAX_COMM_BLOCKS, dtype=torch.float64, device=dev)
        self.out = torch.zeros(2, device=dev)
        self.master = torch.zeros(length, device=dev)
        if self.hi > self.lo:
            self.master[: self.hi - self.lo].copy_(w0[self.lo:self.hi].float())
        self.m1, self.m2 = torch.zeros(length, device=dev), torch.zeros(length, device=dev)
        nbytes = numel * es
        self.a = C.ShardGradOp(w.comms[r], grads.buf, 0, nbytes, _code(dtype), self.shard.data_ptr(), self.partials.data_ptr(), 1.0 / P, True, False, cfg)
        self.norm = C.GradNormOp(w.comms[r], box.buf, 0, self.partials.data_ptr(), self.partials.numel(), 0, self.out.data_ptr())
        coef = self.out[1:].data_ptr()
        if kind == "sgd":
            self.b = C.ShardSgdOp(w.comms[r], weights.buf, 0, nbytes, _code(dtype), self.shard.data_ptr(), coef, self.master.data_ptr(), self.m1.data_ptr(),
                                  False, cfg)
        else:
            self.b = C.ShardAdamOp(w.comms[r], weights.buf, 0, nbytes, _code(dtype), self.shard.data_ptr(), coef, self.master.data_ptr(), self.m1.data_ptr(),
                                   self.m2.data_ptr(), False, cfg)


def _setup(C, P, kind, dtype, numel):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    nbytes = numel * es
    torch.manual_seed(11)
    w0 = torch.randn(numel, device=w.device).to(dtype)
    grads, weights, box = w.alloc(nbytes), w.alloc(nbytes), w.alloc(2 * C.MAX_PEERS * 8)
    ranks = []
    for r in range(P):
        weights.view(r, dtype, numel).copy_(w0)
        ranks.append(_Rank(C, w, r, kind, dtype, numel, grads, weights, box, w0, w.cfg(6)))
        if kind == "sgd":
            ranks[r].b.set_hyper(0.1, 0.9, 0.0, 1e-4, True)
        else:
            ranks[r].b.set_hyper(1e-2, 0.9, 0.999, 1e-8, 0.01, True)
    return w, grads, weights, ranks


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_clipped_phases_match_oracles(C, P, dtype, kind):
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 16) + 16 // es * 3       # slices of unequal length
    w, grads, weights, ranks = _setup(C, P, kind, dtype, numel)
    clipped = []
    for step, max_norm in enumerate([1e6, 50.0, 1e6, 3.0]):   # steps that do not clip and steps that do
        gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
        ref = _owned_slice_sum(gs, _f32(1.0 / P))
        w.run(None, ops=[rk.a for rk in ranks])
        for r, rk in enumerate(ranks):
            n = rk.hi - rk.lo
            assert torch.equal(rk.shard[:n].cpu(), ref[rk.lo:rk.hi]), (P, dtype, step, r)
            assert torch.count_nonzero(grads.view(r, torch.uint8, numel * es)).item() == 0, "gradient bucket must be cleared"
        for rk in ranks:
            rk.norm.set_max_norm(max_norm)
        w.run(None, ops=[rk.norm for rk in ranks])
        outs = [rk.out.cpu() for rk in ranks]
        for o in outs[1:]:
            assert torch.equal(o, outs[0]), "every rank must compute the same bits"
        want = np.float32(math.sqrt(float(ref.double().square().sum())))
        total = outs[0][0]
        assert abs(float(total) - float(want)) <= float(np.spacing(want)), (float(total), float(want))
        coef = _torch_coef(total, max_norm)
        assert torch.equal(outs[0][1], coef), (outs[0][1], coef)
        clipped.append(float(coef) < 1.0)
        # phase B against the float64 per-step oracle fed with shard·coef
        before = [(rk.master.clone(), rk.m1.clone(), rk.m2.clone()) for rk in ranks]
        w.run(None, ops=[rk.b for rk in ranks])
        for r, rk in enumerate(ranks):
            n = rk.hi - rk.lo
            if n == 0:
                continue
            m, a, b = (t[:n] for t in before[r])
            g = rk.shard[:n]
            if kind == "sgd":
                hp = oo.Sgd(lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True, first_step=step == 0, grad_scale=float(coef))
                w_new, m_new, tol_w, tol_m = oo.sgd(m, g, a, hp)
                oo.check(rk.m1[:n], m_new, tol_m, f"momentum P={P} step {step} rank {r}")
            else:
                hp = oo.Adam(lr=1e-2, step=step + 1, weight_decay=0.01, adamw=True, grad_scale=float(coef))
                w_new, m1_new, m2_new, tol_w, tol_1, tol_2 = oo.adam(m, g, a, b, hp)
                oo.check(rk.m1[:n], m1_new, tol_1, f"exp_avg P={P} step {step} rank {r}")
                oo.check(rk.m2[:n], m2_new, tol_2, f"exp_avg_sq P={P} step {step} rank {r}")
            oo.check(rk.master[:n], w_new, tol_w, f"master P={P} step {step} rank {r}")
        # the weights are the masters rounded once, identical on every rank
        model = torch.empty(numel, dtype=dtype, device=w.device)
        for rk in ranks:
            model[rk.lo:rk.hi] = rk.master[: rk.hi - rk.lo].to(dtype)
        for r in range(P):
            assert torch.equal(weights.view(r, dtype, numel), model), (P, dtype, step, r)
    assert clipped == [False, True, False, True]


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_nan_gradient_follows_torch(C, kind):
    """A NaN in one gradient element makes the norm and the coefficient NaN, as in torch: every weight becomes NaN."""
    P, dtype, numel = 2, torch.bfloat16, 4096 + 24
    w, grads, weights, ranks = _setup(C, P, kind, dtype, numel)
    gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
    gs[1][17] = float("nan")
    for r in range(P):
        grads.view(r, dtype, numel).copy_(gs[r])
    ref = torch.nn.Parameter(weights.view(0, dtype, numel).float().clone())
    ref.grad = sum(g.float() for g in gs) / P
    total = torch.nn.utils.clip_grad_norm_([ref], 1.0)
    (torch.optim.SGD([ref], lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-4) if kind == "sgd" else
     torch.optim.AdamW([ref], lr=1e-2, weight_decay=0.01)).step()
    for ops in ([rk.a for rk in ranks], [rk.norm for rk in ranks], [rk.b for rk in ranks]):
        w.run(None, ops=ops)
    assert torch.isnan(total) and all(torch.isnan(rk.out).all() for rk in ranks)
    for r in range(P):
        got = weights.view(r, dtype, numel).float()
        assert torch.equal(torch.isnan(got), torch.isnan(ref.detach())), "NaN pattern differs from torch"


# ---------------------------------------------------------------------------------------------------------------------
# end to end: self-peer (world 1) and real peers
# ---------------------------------------------------------------------------------------------------------------------
def _clip_train_worker(rank, world, kind):
    """channels_last conv + linear, two parameter groups (+ one parameter outside the buckets at world 1), 6 steps with the bound
    active on some of them, against torch clip_grad_norm_ + SGD / AdamW in fp32; a checkpoint taken after step 3 resumes
    bit-identically. Returns the final weights and the norms (``last_grad_norm``) for the cross-rank comparison."""
    import torch.distributed as dist
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_sgd

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False   # the resumed run must see the same gradients
    BOUND = 0.05
    bounds = [None, 1e3, None, 1e3, 0.02, None]    # None: step() clips with max_grad_norm; a number: clip_grad_norm_(number) first
    out = {}

    def groups(ps):
        return [{"params": [p for p in ps if p.dim() > 1], "weight_decay": 0.01}, {"params": [p for p in ps if p.dim() <= 1], "weight_decay": 0.0}]

    def make(ps, **kw):
        if kind == "sgd":
            return make_sharded_fused_sgd(groups(ps), lr=0.05, momentum=0.9, **kw)
        return make_sharded_fused_adam(groups(ps), lr=1e-3, adamw=True, **kw)

    def batch(it):
        g = torch.Generator(device=dev).manual_seed(100 * it + rank)
        return torch.randn(8, 3, 12, 12, device=dev, generator=g).to(memory_format=torch.channels_last)

    use_extra = world == 1
    for dtype in (torch.float32, torch.bfloat16):
        torch.manual_seed(9)
        base = nn.Sequential(nn.Conv2d(3, 16, 3), nn.ReLU(), nn.Flatten(), nn.Linear(16 * 100, 32)).to(dev).to(memory_format=torch.channels_last)
        extra0 = torch.randn(40, device=dev)
        oracle = copy.deepcopy(base)
        oextra = nn.Parameter(extra0.clone())
        oparams = list(oracle.parameters()) + ([oextra] if use_extra else [])
        oopt = (torch.optim.SGD(groups(oparams), lr=0.05, momentum=0.9) if kind == "sgd" else torch.optim.AdamW(groups(oparams), lr=1e-3))

        def build(state=None, model_sd=None, ex_val=None):
            m = copy.deepcopy(base).to(dtype)
            if model_sd is not None:
                m.load_state_dict(model_sd)
            ex = nn.Parameter((extra0 if ex_val is None else ex_val).clone().to(dtype))
            o = make(list(m.parameters()) + ([ex] if use_extra else []), max_grad_norm=BOUND)
            if state is not None:
                o.load_state_dict(state)
            m = m.with_bagua([o], FusedGradientAllReduceAlgorithm(o))
            assert all("_clip_" in b.allreduce_variant for b in m.bagua_buckets), [b.allreduce_variant for b in m.bagua_buckets]
            return m, o, ex

        def train(m, o, ex, its):
            norms = []
            for it in its:
                x = batch(it)
                o.zero_grad()
                m(x.to(dtype)).float().pow(2).mean().backward()
                if use_extra:
                    ex.grad = (torch.sin(torch.arange(40, device=dev, dtype=torch.float32) + it) * 0.03).to(dtype)
                if bounds[it] is not None:
                    o.clip_grad_norm_(bounds[it])
                o.step()
                norms.append(o.last_grad_norm.clone())
            return norms

        model, opt, ex = build()
        norms = train(model, opt, ex, range(3))
        torch.cuda.synchronize()
        # a snapshot as torch.save would write it: the uncovered parameter's state in state_dict() is a live reference
        sd, msd, ex3 = copy.deepcopy(opt.state_dict()), {k: v.clone() for k, v in model.state_dict().items()}, ex.detach().clone()
        norms += train(model, opt, ex, range(3, 6))
        torch.cuda.synchronize()
        final = torch.cat([p.detach().reshape(-1).float() for p in model.parameters()] + ([ex.detach().float()] if use_extra else []))

        model2, opt2, ex2 = build(sd, msd, ex3)          # resume from the checkpoint taken after step 3
        norms2 = train(model2, opt2, ex2, range(3, 6))
        torch.cuda.synchronize()
        final2 = torch.cat([p.detach().reshape(-1).float() for p in model2.parameters()] + ([ex2.detach().float()] if use_extra else []))

        onorms = []
        for it in range(6):
            oopt.zero_grad()
            oracle(batch(it)).pow(2).mean().backward()
            for p in oracle.parameters():
                if world > 1:
                    dist.all_reduce(p.grad)
                    p.grad /= world
            if use_extra:
                oextra.grad = torch.sin(torch.arange(40, device=dev, dtype=torch.float32) + it) * 0.03
                if dtype == torch.bfloat16:
                    oextra.grad = oextra.grad.to(dtype).float()
            onorms.append(torch.nn.utils.clip_grad_norm_(oparams, bounds[it] if bounds[it] is not None else BOUND))
            oopt.step()
        want = torch.cat([p.detach().reshape(-1) for p in oparams])
        got_norms, want_norms = torch.stack(norms).cpu(), torch.stack(onorms).cpu()
        assert (want_norms > BOUND).any() and (want_norms < 1e3).all()
        sdf = opt.state_dict()
        masters = torch.cat([sdf["state"][n]["master"].reshape(-1).to(dev) for n, _ in model.named_parameters()])
        if use_extra:
            st = opt.state[ex]
            masters = torch.cat([masters, (st["master"] if "master" in st else ex.detach()).float().reshape(-1)])
        if dtype == torch.float32:
            torch.testing.assert_close(got_norms, want_norms, rtol=1e-5, atol=0)
            torch.testing.assert_close(masters, want, rtol=1e-4, atol=1e-5)
        else:
            torch.testing.assert_close(got_norms, want_norms, rtol=5e-2, atol=0)
            assert (masters - want).abs().max().item() < 5e-2
        out[str(dtype)] = (final.cpu(), got_norms)
        assert torch.equal(final2, final), (f"{dtype}: a resumed checkpoint must continue bit-identically; max diff "
                                            f"{(final2 - final).abs().max().item()}, norms {torch.stack(norms2).tolist()} vs {got_norms[3:].tolist()}")
        assert torch.equal(torch.stack(norms2).cpu(), got_norms[3:])
    return out


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_self_peer_clipped_training_matches_torch(kind):
    run_distributed(_clip_train_worker, world=1, args=(kind,), use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
@pytest.mark.parametrize("multimem", ["0", "1"])
def test_clipped_training_on_real_peers(multimem):
    n = min(torch.cuda.device_count(), 8)
    res = run_distributed(_clip_train_worker, world=n, args=("adamw",), use_cuda=True, extra_env={"BAGUA_FUSED_MULTIMEM": multimem}, timeout=300)
    for r in res[1:]:
        for k in res[0]:
            assert torch.equal(r[k][1], res[0][k][1]), "last_grad_norm must be bitwise equal on every rank"
            assert torch.equal(r[k][0], res[0][k][0])
