"""Dynamic loss scaling of the in-bucket optimizers on the GPU.

* The kernels on virtual peer worlds of P = 1 … 8 ranks: phase A ``shard_grad`` → ``LossScaleNormOp`` → the phase-B ops told to
  take ``{coef, found_inf, t}`` from device memory, over steps that are taken (clipped or not) and steps that overflow (an ``inf``
  or a ``NaN`` planted in one rank's gradient — ordinary data —, on the very first step, and an fp16 sum that overflows only in the
  reduction), against ``tests/test_loss_scale_oracle.py`` and the per-step float64 optimizer oracle.
* With scale 1 and finite gradients the result is bit-identical to the clipped path without loss scaling (same kernels' update
  code, the same coefficient bits, bias corrections from the same double-precision formula — asserted with ``torch.equal``).
* ``make_sharded_fused_*(loss_scaling=True)`` + ``ShardedGradScaler`` end to end in self-peer mode (and on 2+ real GPUs) against an
  fp32 torch model stepped with stock ``GradScaler`` on the same gradients.
"""
import copy
import math

import numpy as np
import pytest
import torch

from tests import optim_oracle as oo
from tests.mp_utils import run_distributed
from tests.test_loss_scale_oracle import exchange
from tests.test_virtual_peer_gpu import _code, _f32, _owned_slice_sum, _shard, _world

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 3, 4, 8]
SGD_HP = (0.1, 0.9, 0.0, 1e-4, True)
ADAM_HP = (1e-2, 0.9, 0.999, 1e-8, 0.01, True)
LAMB_HP = (1e-2, 0.9, 0.999, 1e-6, 0.01)


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


class _Rank:
    """One virtual rank's buffers and ops of the two-phase update of a single bucket, with (``scaled``) or without loss scaling."""

    def __init__(self, C, w, r, kind, dtype, numel, grads, weights, box, ratio_box, w0, cfg, scaled):
        from bagua_b200.ops.optim import multi_tensor_plan

        es = torch.empty(0, dtype=dtype).element_size()
        self.lo, self.hi, length = _shard(numel, es, w.world, r)
        dev, comm, nbytes, code = w.device, w.comms[r], numel * es, _code(dtype)
        self.n = self.hi - self.lo
        self.symmetric = (grads, weights, box, ratio_box)   # the ops hold raw pointers: the buffers must outlive them
        self.shard = torch.zeros(length, device=dev)
        self.partials = torch.zeros(1, C.MAX_COMM_BLOCKS, dtype=torch.float64, device=dev)
        self.out = torch.zeros(3 if scaled else 2, device=dev)
        self.t = torch.zeros(1, dtype=torch.int32, device=dev)
        self.scale = torch.ones(1, device=dev)
        self.master = torch.zeros(length, device=dev)
        if self.n > 0:
            self.master[: self.n].copy_(w0[self.lo:self.hi].float())
        self.m1, self.m2 = torch.zeros(length, device=dev), torch.zeros(length, device=dev)
        self.a = C.ShardGradOp(comm, grads.buf, 0, nbytes, code, self.shard.data_ptr(), self.partials.data_ptr(), 1.0 / w.world, True, False, cfg)
        if scaled:
            self.norm = C.LossScaleNormOp(comm, box.buf, 0, self.partials.data_ptr(), self.partials.numel(), 0, self.out.data_ptr(), self.t.data_ptr())
            self.norm.set_scale_ptr(self.scale.data_ptr())
        else:
            self.norm = C.GradNormOp(comm, box.buf, 0, self.partials.data_ptr(), self.partials.numel(), 0, self.out.data_ptr())
        coef = self.out[1:].data_ptr()
        self.pre = self.ratio = None
        if kind == "sgd":
            self.b = C.ShardSgdOp(comm, weights.buf, 0, nbytes, code, self.shard.data_ptr(), coef, self.master.data_ptr(), self.m1.data_ptr(), False, cfg)
            self.b.set_hyper(*SGD_HP)
        elif kind == "adam":
            self.b = C.ShardAdamOp(comm, weights.buf, 0, nbytes, code, self.shard.data_ptr(), coef, self.master.data_ptr(), self.m1.data_ptr(),
                                   self.m2.data_ptr(), False, cfg)
            self.b.set_hyper(*ADAM_HP)
        else:   # the whole bucket is one parameter: one segment per rank, one ratio
            if self.n > 0:
                self.plan = multi_tensor_plan([[t[: self.n]] for t in (self.master, self.shard, self.m1, self.m2)])
                self.lpart = torch.zeros(self.plan.n_blocks, 2, dtype=torch.float64, device=dev)
                self.pre = C.LambMomentsOp(*self.plan.args(), coef, self.lpart.data_ptr())
                nblk = self.plan.n_blocks
            else:
                self.lpart = torch.zeros(1, 2, dtype=torch.float64, device=dev)
                self.pre = C.LambMomentsOp(0, 0, 0, 0, 0, 0, 65536, coef, self.lpart.data_ptr())
                nblk = 0
            self.tables = (torch.tensor([self.lpart.data_ptr()], dtype=torch.int64, device=dev), torch.tensor([nblk], dtype=torch.int32, device=dev),
                           torch.tensor([0, max(self.n, 0), 0], dtype=torch.int32, device=dev))
            self.ratio_out, self.sums = torch.ones(1, device=dev), torch.zeros(1, 2, dtype=torch.float64, device=dev)
            self.ratio = C.LambRatioOp(comm, ratio_box.buf, 0, self.tables[0].data_ptr(), self.tables[1].data_ptr(), 1, self.ratio_out.data_ptr(),
                                       self.sums.data_ptr())
            self.b = C.ShardLambOp(comm, weights.buf, 0, nbytes, code, self.master.data_ptr(), self.m1.data_ptr(), self.m2.data_ptr(),
                                   self.tables[2].data_ptr(), 1 if self.n > 0 else 0, self.ratio_out.data_ptr(), False, cfg)
            self.pre.set_hyper(*LAMB_HP)
            self.b.set_hyper(*LAMB_HP)
        if scaled:
            for op in (self.b, self.pre):
                if op is not None:
                    op.set_device_step(coef, self.t.data_ptr())

    def state(self):
        return self.master.clone(), self.m1.clone(), self.m2.clone()


def _setup(C, P, kind, dtype, numel, scaled=True):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    nbytes = numel * es
    torch.manual_seed(11)
    w0 = torch.randn(numel, device=w.device).to(dtype)
    grads, weights, box, rbox = w.alloc(nbytes), w.alloc(nbytes), w.alloc(2 * C.MAX_PEERS * 8), w.alloc(C.LambRatioOp.box_bytes(1))
    ranks = []
    for r in range(P):
        weights.view(r, dtype, numel).copy_(w0)
        ranks.append(_Rank(C, w, r, kind, dtype, numel, grads, weights, box, rbox, w0, w.cfg(6), scaled))
    return w, grads, weights, ranks


def _run_step(w, ranks, max_norm):
    """phase A → exchange → (LAMB: moments → ratio) → update, each as one collective over the virtual ranks."""
    w.run(None, ops=[rk.a for rk in ranks])
    for rk in ranks:
        rk.norm.set_max_norm(max_norm)
    w.run(None, ops=[rk.norm for rk in ranks])
    if ranks[0].pre is not None:
        _run_local(w, [rk.pre for rk in ranks])   # the moments kernels exchange nothing
        w.run(None, ops=[rk.ratio for rk in ranks])
    w.run(None, ops=[rk.b for rk in ranks])


def _run_local(w, ops):
    from bagua_b200.core import native

    s = torch.cuda.current_stream(w.device)
    for op in ops:
        native().run_op(op, s.cuda_stream, w.device.index)
    s.synchronize()


# what each step of the sequence does: (scale, bound, planted value or None, rank that gets it)
INF = float("inf")
STEPS = [(1024.0, INF, "inf", 0),         # an overflow on the very first step
         (512.0, INF, None, 0),           # the first step that counts: SGD's momentum initialisation, Adam's t = 1
         (512.0, 0.01, None, 0),          # clipped
         (512.0, INF, "nan", -1),         # a NaN on the last rank
         (256.0, 1e6, None, 0),           # bound far away
         (256.0, INF, "sum", 0),          # finite on every rank, the sum over the ranks is not (see the test)
         (128.0, 0.02, None, 0)]


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("kind", ["sgd", "adam", "lamb"])
def test_scaled_phases_match_oracles(C, P, dtype, kind):
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 15) + 16 // es * 3       # slices of unequal length
    w, grads, weights, ranks = _setup(C, P, kind, dtype, numel)
    t, taken = 0, []
    for step, (scale, bound, plant, who) in enumerate(STEPS):
        if plant == "sum" and P == 1:
            continue
        gen = torch.Generator(device=w.device).manual_seed(100 + step)
        gs = [(torch.randn(numel, device=w.device, generator=gen) * 1e-3 * scale).to(dtype) for _ in range(P)]
        if plant in ("inf", "nan"):
            gs[who][numel // 3] = float(plant)
        elif plant == "sum":
            # The reduction accumulates in fp32. fp16: 40000 + 40000 does not fit the bucket's dtype, but the fp32 sum and its
            # average do, so the step is taken. bf16 / fp32: 3e38 + 3e38 overflows the accumulator itself, so it is skipped.
            for g in gs:
                g[7] = 40000.0 if dtype == torch.float16 else 3e38
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
            ranks[r].scale.fill_(scale)
        before = [rk.state() for rk in ranks]
        wbefore = [weights.view(r, dtype, numel).clone() for r in range(P)]
        t_before = [int(rk.t.item()) for rk in ranks]
        _run_step(w, ranks, bound)

        ref = _owned_slice_sum(gs, _f32(1.0 / P))
        outs = [rk.out.cpu() for rk in ranks]
        for o in outs[1:]:
            assert torch.equal(o.view(torch.int32), outs[0].view(torch.int32)), "every rank must compute the same bits"
        sums = [float(ref[rk.lo:rk.hi].double().square().sum()) for rk in ranks]
        total, coef, found, t = exchange(sums, scale, bound, t)
        assert bool(outs[0][2]) == found == (plant in ("inf", "nan") or (plant == "sum" and dtype != torch.float16)), (step, outs[0])
        assert all(int(rk.t.item()) == t for rk in ranks), (step, t, [int(rk.t.item()) for rk in ranks])
        for r in range(P):
            assert torch.count_nonzero(grads.view(r, torch.uint8, numel * es)).item() == 0, "gradient bucket must be cleared either way"
        if found:
            assert not math.isfinite(float(outs[0][0]))
            assert [int(rk.t.item()) for rk in ranks] == t_before
            for r, rk in enumerate(ranks):
                for a, b in zip(before[r], rk.state()):
                    assert torch.equal(a, b), f"step {step}: a skipped step changed optimizer state on rank {r}"
                assert torch.equal(weights.view(r, dtype, numel), wbefore[r]), f"step {step}: a skipped step changed the weights of rank {r}"
            continue
        taken.append(step)
        got_total = np.float32(outs[0][0].item())
        assert abs(float(got_total) - float(total)) <= float(np.spacing(total)), (step, got_total, total)
        # coef exactly, given the kernel's own total
        inv = np.float32(1.0 / np.float64(np.float32(scale)))
        clip = np.float32(1.0)
        if math.isfinite(bound):
            clip = torch.clamp(np.float32(bound) / (outs[0][0] + 1e-6), max=1.0).numpy()
        assert np.float32(outs[0][1].item()) == np.float32(inv * clip), (step, outs[0], inv, clip)
        c = float(outs[0][1])
        for r, rk in enumerate(ranks):
            n = rk.n
            if n == 0 or kind == "lamb":   # LAMB's arithmetic is checked bit for bit against the unscaled path below
                continue
            m, a, b = (x[:n] for x in before[r])
            g = rk.shard[:n]
            assert torch.equal(g.cpu(), ref[rk.lo:rk.hi])
            if kind == "sgd":
                hp = oo.Sgd(lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True, first_step=t == 1, grad_scale=c)
                w_new, m_new, tol_w, tol_m = oo.sgd(m, g, a, hp)
                oo.check(rk.m1[:n], m_new, tol_m, f"momentum P={P} step {step} rank {r}")
            else:
                hp = oo.Adam(lr=1e-2, step=t, weight_decay=0.01, adamw=True, grad_scale=c)
                w_new, m1_new, m2_new, tol_w, tol_1, tol_2 = oo.adam(m, g, a, b, hp)
                oo.check(rk.m1[:n], m1_new, tol_1, f"exp_avg P={P} step {step} rank {r}")
                oo.check(rk.m2[:n], m2_new, tol_2, f"exp_avg_sq P={P} step {step} rank {r}")
            oo.check(rk.master[:n], w_new, tol_w, f"master P={P} step {step} rank {r}")
        model = torch.empty(numel, dtype=dtype, device=w.device)
        for rk in ranks:
            model[rk.lo:rk.hi] = rk.master[: rk.n].to(dtype)
        for r in range(P):
            assert torch.equal(weights.view(r, dtype, numel), model), (P, dtype, step, r)
    assert taken[:2] == [1, 2] and t == len(taken)


def _trajectory(C, P, kind, scaled):
    """Four steps (bounds that clip and bounds that do not) at scale 1; per step {total, coef}, every rank's state and weights."""
    dtype, numel = torch.bfloat16, (1 << 14) + 24
    w, grads, weights, ranks = _setup(C, P, kind, dtype, numel, scaled=scaled)
    out = []
    for step, bound in enumerate([1e6, 0.05, 1e6, 0.02]):
        gen = torch.Generator(device=w.device).manual_seed(step)
        for r in range(P):
            grads.view(r, dtype, numel).copy_(torch.randn(numel, device=w.device, generator=gen).mul(0.01).to(dtype))
        _run_step(w, ranks, bound)
        out.append(([rk.out[:2].cpu() for rk in ranks], [[t.cpu() for t in rk.state()] for rk in ranks],
                    [weights.view(r, dtype, numel).cpu() for r in range(P)]))
    count = int(ranks[0].t.item()) if scaled else ranks[0].b.steps()
    return out, count


@pytest.mark.parametrize("P", [1, 3, 8])
@pytest.mark.parametrize("kind", ["sgd", "adam", "lamb"])
def test_scale_one_is_bit_identical_to_the_clipped_path(C, P, kind):
    """loss_scaling with scale 1 and finite gradients against the same ops without it (host step count, GradNormOp): bit for bit —
    1/1 is exact, coef = 1·clip, and the device builds the bias corrections with the formula the host uses."""
    plain, n_plain = _trajectory(C, P, kind, scaled=False)
    scaled, n_scaled = _trajectory(C, P, kind, scaled=True)
    assert n_plain == n_scaled == 4
    for step, ((o1, s1, w1), (o2, s2, w2)) in enumerate(zip(plain, scaled)):
        for r in range(P):
            assert torch.equal(o1[r], o2[r]), (step, r, o1[r], o2[r])
            assert all(torch.equal(a, b) for a, b in zip(s1[r], s2[r])), (kind, P, step, r)
            assert torch.equal(w1[r], w2[r]), (kind, P, step, r)


# ---------------------------------------------------------------------------------------------------------------------
# end to end: self-peer (world 1) and real peers
# ---------------------------------------------------------------------------------------------------------------------
def _scaled_train_worker(rank, world, kind):
    """An fp16 model with two parameter groups (+ one parameter outside the buckets at world 1), 8 steps with ShardedGradScaler:
    init_scale so large that the first steps overflow and back off, growth_interval=2 so that it grows again; against an fp32
    model stepped with stock GradScaler logic on the same all-rank-averaged gradients. A checkpoint (optimizer + scaler) taken
    after step 4 resumes bit-identically."""
    import torch.distributed as dist
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.parallel.algorithms.gradient_allreduce import (FusedGradientAllReduceAlgorithm, make_sharded_fused_adam, make_sharded_fused_lamb,
                                                                  make_sharded_fused_sgd)

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    dtype, BOUND, STEPS_, INIT = torch.float16, 0.5, 8, 2.0 ** 24
    use_extra = world == 1
    variant_kind = {"sgd": "sgd", "adamw": "adam", "lamb": "lamb"}[kind]

    def groups(ps):
        return [{"params": [p for p in ps if p.dim() > 1], "weight_decay": 0.01}, {"params": [p for p in ps if p.dim() <= 1], "weight_decay": 0.0}]

    def make(ps, **kw):
        if kind == "sgd":
            return make_sharded_fused_sgd(groups(ps), lr=0.05, momentum=0.9, **kw)
        if kind == "lamb":
            return make_sharded_fused_lamb(groups(ps), lr=1e-3, **kw)
        return make_sharded_fused_adam(groups(ps), lr=1e-3, adamw=True, **kw)

    def batch(it):
        g = torch.Generator(device=dev).manual_seed(100 * it + rank)
        return torch.randn(16, 64, device=dev, generator=g)

    torch.manual_seed(9)
    base = nn.Sequential(nn.Linear(64, 128), nn.Tanh(), nn.Linear(128, 32)).to(dev)
    extra0 = torch.randn(40, device=dev)

    def extra_grad(it, scale):
        return (torch.sin(torch.arange(40, device=dev, dtype=torch.float32) + it) * 0.03 * scale).to(dtype)

    def build(state=None, model_sd=None, ex_val=None, scaler_sd=None, **kw):
        m = copy.deepcopy(base).to(dtype)
        if model_sd is not None:
            m.load_state_dict(model_sd)
        ex = nn.Parameter((extra0 if ex_val is None else ex_val).clone().to(dtype))
        o = make(list(m.parameters()) + ([ex] if use_extra else []), **kw)
        if state is not None:
            o.load_state_dict(state)
        m = m.with_bagua([o], FusedGradientAllReduceAlgorithm(o))
        sc = ShardedGradScaler(init_scale=INIT, growth_interval=2)
        if scaler_sd is not None:
            sc.load_state_dict(scaler_sd)
        return m, o, ex, sc

    def train(m, o, ex, sc, its):
        log = []
        for it in its:
            o.zero_grad()
            loss = m(batch(it).to(dtype)).float().pow(2).mean()
            sc.scale(loss).backward()
            scale = sc.get_scale()
            if use_extra:
                ex.grad = extra_grad(it, scale)
            sc.step(o)
            log.append((scale, o.last_step_skipped.clone(), o.last_grad_norm.clone()))
            sc.update()
        torch.cuda.synchronize()
        return [(s, bool(k.item()), float(n) if bool(torch.isfinite(n)) else None) for s, k, n in log]

    def flat(m, ex):
        return torch.cat([p.detach().reshape(-1).float() for p in m.parameters()] + ([ex.detach().float()] if use_extra else []))

    model, opt, ex, scaler = build(max_grad_norm=BOUND, loss_scaling=True)
    assert all("_scaled_clip_" in b.allreduce_variant for b in model.bagua_buckets), [b.allreduce_variant for b in model.bagua_buckets]
    with pytest.raises(RuntimeError, match="max_grad_norm"):
        scaler.unscale_(opt)
    log = train(model, opt, ex, scaler, range(4))
    sd, ssd = copy.deepcopy(opt.state_dict()), scaler.state_dict()
    msd, ex4 = {k: v.clone() for k, v in model.state_dict().items()}, ex.detach().clone()
    log += train(model, opt, ex, scaler, range(4, STEPS_))
    final = flat(model, ex)
    skipped = [k for _, k, _ in log]
    assert skipped[0] and not all(skipped) and sd["steps"] == 4 - sum(skipped[:4]), (log, sd["steps"])
    assert any(b > a for (a, _, _), (b, _, _) in zip(log, log[1:])), f"the scale never grew again: {log}"

    model2, opt2, ex2, scaler2 = build(sd, msd, ex4, ssd, max_grad_norm=BOUND, loss_scaling=True)
    log2 = train(model2, opt2, ex2, scaler2, range(4, STEPS_))
    assert log2 == log[4:], (log2, log[4:])
    assert torch.equal(flat(model2, ex2), final), "a resumed checkpoint (optimizer + scaler) must continue bit-identically"

    # the reference: fp32 weights, gradients of the fp16 model's loss are not available to it, so it runs its own fp32 forward on
    # the same batches; stock GradScaler logic (unscale → inf check → clip → step / skip → update) on the averaged gradients
    oracle = copy.deepcopy(base)
    oextra = nn.Parameter(extra0.clone())
    oparams = list(oracle.parameters()) + ([oextra] if use_extra else [])
    if kind == "sgd":
        oopt = torch.optim.SGD(groups(oparams), lr=0.05, momentum=0.9)
    elif kind == "lamb":
        from bagua_b200.ops.optim import FusedLAMB

        oopt = FusedLAMB(groups(oparams), lr=1e-3)
    else:
        oopt = torch.optim.AdamW(groups(oparams), lr=1e-3)
    oscaler = torch.amp.GradScaler("cuda", init_scale=INIT, growth_interval=2)
    olog = []
    for it in range(STEPS_):
        oopt.zero_grad()
        # the half-precision run overflows in fp16 where an fp32 backward would not: the reference takes the scaled fp16 gradients'
        # overflow pattern from a backward in fp16 arithmetic of its own weights
        half = copy.deepcopy(oracle).to(dtype)
        oscaler.scale(half(batch(it).to(dtype)).float().pow(2).mean()).backward()
        scale = oscaler.get_scale()
        for p, hp in zip(oracle.parameters(), half.parameters()):
            g = hp.grad.float()
            if world > 1:
                g = (g.to(dtype).float())
                dist.all_reduce(g)
                g /= world
            p.grad = g
        if use_extra:
            oextra.grad = extra_grad(it, scale).float()
        oscaler.unscale_(oopt)
        norm = torch.nn.utils.clip_grad_norm_(oparams, BOUND)
        before = oextra.detach().clone()
        oscaler.step(oopt)
        olog.append((scale, not math.isfinite(float(norm)), float(norm) if math.isfinite(float(norm)) else None))
        if olog[-1][1]:
            assert torch.equal(oextra.detach(), before)
        oscaler.update()
    assert [(s, k) for s, k, _ in log] == [(s, k) for s, k, _ in olog], f"skip pattern / scale trajectory differ:\n{log}\n{olog}"
    for (_, k, n), (_, _, on) in zip(log, olog):
        if not k:
            assert abs(n - on) <= 5e-2 * on, (log, olog)
    want = torch.cat([p.detach().reshape(-1) for p in oparams])
    sdf = opt.state_dict()
    masters = torch.cat([sdf["state"][n]["master"].reshape(-1).to(dev) for n, _ in model.named_parameters()])
    if use_extra:
        st = opt.state[ex]
        masters = torch.cat([masters, (st["master"] if "master" in st else ex.detach()).float().reshape(-1)])
    assert (masters - want).abs().max().item() < 5e-2, (masters - want).abs().max().item()
    if use_extra:   # the parameter outside the buckets is skipped with the others: after the first (skipped) step it is untouched
        m3, o3, ex3, sc3 = build(max_grad_norm=BOUND, loss_scaling=True)
        train(m3, o3, ex3, sc3, range(1))
        assert torch.equal(ex3.detach(), extra0.to(dtype)) and torch.equal(flat(m3, ex3)[:-40], flat(copy.deepcopy(base).to(dtype), ex3)[:-40])

    # unchanged without the new argument: variants and launches per step; and such an optimizer refuses the scaler
    m4, o4, _, sc4 = build(max_grad_norm=BOUND)
    assert all(b.allreduce_variant.startswith(f"fused_{variant_kind}_clip_") for b in m4.bagua_buckets)
    nb = len(m4.bagua_buckets)
    per_step = 1 + (2 * nb + 1 if kind == "lamb" else nb)
    o4.zero_grad()
    sc4.scale(m4(batch(0).to(dtype)).float().pow(2).mean()).backward()
    with pytest.raises(RuntimeError, match="loss_scaling=True"):
        sc4.step(o4)
    k0 = o4.kernel_launches
    o4.step()
    assert o4.kernel_launches - k0 == per_step, (o4.kernel_launches - k0, nb)
    m5, o5, ex5, sc5 = build(max_grad_norm=BOUND, loss_scaling=True)
    k0 = o5.kernel_launches
    train(m5, o5, ex5, sc5, range(1))
    assert o5.kernel_launches - k0 == per_step, "loss scaling must cost the launches clipping costs"
    return final.cpu(), log


@pytest.mark.parametrize("kind", ["sgd", "adamw", "lamb"])
def test_self_peer_scaled_training_matches_torch(kind):
    run_distributed(_scaled_train_worker, world=1, args=(kind,), use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
def test_scaled_training_on_real_peers():
    n = min(torch.cuda.device_count(), 8)
    res = run_distributed(_scaled_train_worker, world=n, args=("adamw",), use_cuda=True, timeout=300)
    for final, log in res[1:]:
        assert torch.equal(final, res[0][0]), "weights must be identical on every rank"
        assert [x[:2] for x in log] == [x[:2] for x in res[0][1]]
