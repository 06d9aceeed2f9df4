"""LARS on the GPU.

* ``FusedLARS`` (the two multi-tensor kernels) against the float64 oracle of ``tests/lars_oracle.py``, with an ``lr`` change.
* The in-bucket kernels (phase A ``shard_grad``, the LARS norms, the per-parameter exchange of ``LambRatioOp``, momentum + apply +
  all-gather) on virtual peer worlds of P = 1 … 8 ranks, with a bucket whose slices cut parameters anywhere: with and without
  weight decay, with clipping, and with loss scaling and an overflowed step.
* ``make_sharded_fused_lars`` end to end in self-peer mode (and on 2+ real GPUs) against ``FusedLARS`` without bagua.
"""
import copy
import math

import pytest
import torch

from tests import lars_oracle as lo
from tests.lamb_oracle import sum_bound
from tests.mp_utils import run_distributed
from tests.test_virtual_peer_gpu import _code, _f32, _owned_slice_sum, _world

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


def _check(actual, expected, tol, what):
    assert lo.excess(actual, expected, tol) <= 1.0, what


# ---------------------------------------------------------------------------------------------------------------------
# FusedLARS
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [0, 1, 65535, 65536, 65537, 2 * 65536 + 3]
PAD = 32
LRS = [0.5, 0.5, 0.2]   # an lr change between the second and the third step


def _padded(n, dtype, gen, scale=1.0):
    """A tensor of n elements inside a larger buffer whose margins hold sentinel values."""
    buf = torch.full((n + 2 * PAD,), 7.0, device="cuda", dtype=dtype)
    t = buf[PAD:PAD + n]
    t.copy_((torch.randn(n, device="cuda", generator=gen) * scale).to(dtype))
    return buf, t


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_fused_lars_matches_oracle(dtype):
    from bagua_b200.ops.optim import FusedLARS

    gen = torch.Generator(device="cuda").manual_seed(3)
    params, bufs = [], []
    for n in SIZES:
        wb, w = _padded(n, dtype, gen)
        gb, g = _padded(n, dtype, gen, 0.1)
        p = torch.nn.Parameter(torch.empty(0, device="cuda", dtype=dtype))
        p.data = w
        p.grad = g
        params.append(p)
        bufs += [wb, gb]
    cl = torch.nn.Parameter(torch.randn(4, 5, 3, 3, device="cuda").to(dtype).to(memory_format=torch.channels_last))
    params.append(cl)
    # the decay group holds every tensor of several 65536-element chunks and the channels_last one: their trust is a fixed-order
    # sum over several blocks (stage 2)
    groups = [{"params": params[2:], "weight_decay": 5e-4}, {"params": params[:2], "weight_decay": 0.0}]
    opt = FusedLARS(groups, lr=LRS[0], momentum=0.9, trust_coefficient=1e-3)
    mixed = dtype != torch.float32

    def flat(t):   # memory order, as the kernels walk it
        return torch.as_strided(t, (t.numel(),), (1,))

    for step, lr in enumerate(LRS):
        for g in opt.param_groups:
            g["lr"] = lr
        for p in params:
            if p is cl:
                p.grad = (torch.randn(p.shape, device="cuda", generator=gen) * 0.1).to(dtype)   # contiguous: a copy in the layout
            elif step > 0:
                p.grad.copy_((torch.randn(p.numel(), device="cuda", generator=gen) * 0.1).to(dtype))
        before = {}
        for p in params:
            st = opt.state[p]
            w = st["master"] if "master" in st else p.detach().float()
            g = p.grad.contiguous(memory_format=torch.channels_last) if p is cl else p.grad
            v = flat(st["momentum_buffer"]).clone() if "momentum_buffer" in st else torch.zeros(p.numel(), device="cuda")
            before[p] = (flat(w).clone(), flat(g).clone(), v)
        opt.step()
        torch.cuda.synchronize()
        for group in groups:
            hp = lo.Lars(lr=lr, momentum=0.9, weight_decay=group["weight_decay"], trust_coefficient=1e-3)
            for p in group["params"]:
                w_new, v_new, tr, tol_w, tol_v = lo.lars([before[p]], hp)[0]
                if group["weight_decay"] != 0 and p.numel() > 65536:
                    assert tr != 1.0, "a multi-chunk parameter must get a real trust"
                st = opt.state[p]
                _check(flat(st["momentum_buffer"]), v_new, tol_v, f"momentum {dtype} n={p.numel()} step {step}")
                if mixed:
                    _check(flat(st["master"]), w_new, tol_w, f"master {dtype} n={p.numel()} step {step}")
                    assert torch.equal(flat(p.detach()), flat(st["master"]).to(dtype)), "model copy = master rounded once"
                else:
                    _check(flat(p.detach()), w_new, tol_w, f"param {dtype} n={p.numel()} step {step}")
                assert torch.count_nonzero(p.grad).item() == 0, "zero_grad_in_step clears the gradient"
        for b in bufs:
            assert torch.all(b[:PAD] == 7.0) and torch.all(b[-PAD:] == 7.0), "write outside a tensor"


# ---------------------------------------------------------------------------------------------------------------------
# in-bucket kernels on a virtual peer world
# ---------------------------------------------------------------------------------------------------------------------
WORLDS = [1, 2, 3, 4, 8]
# parameters packed back to back: tiny ones share 16-byte vectors, an odd-sized one straddles the slices, one is zero
SIZES_BUCKET = [1, 3, 7, 1, 513, 2, 20000, 5, 1, 777, 4099, 3, 131077]
BIG_PARAM = 12
ZERO_PARAM = 9
HP = dict(momentum=0.9, trust_coefficient=1e-3)


class _Rank:
    def __init__(self, C, w, r, dtype, numel, grads, weights, box, rbox, w0, cfg, mode, wd):
        from bagua_b200.ops.optim import multi_tensor_plan

        es = torch.empty(0, dtype=dtype).element_size()
        P, dev, comm = w.world, w.device, w.comms[r]
        per = 16 // es
        vpr = (numel * es // 16 + P - 1) // P
        self.lo, self.hi, length = r * vpr * per, min((r + 1) * vpr * per, numel), vpr * per
        self.symmetric = (grads, weights, box, rbox)
        self.shard = torch.zeros(length, device=dev)
        self.master = torch.zeros(length, device=dev)
        if self.hi > self.lo:
            self.master[: self.hi - self.lo].copy_(w0[self.lo:self.hi].float())
        self.mom = torch.zeros(length, device=dev)
        self.gpart = torch.zeros(1, C.MAX_COMM_BLOCKS, dtype=torch.float64, device=dev)
        self.out = torch.zeros(3, device=dev)
        self.t = torch.zeros(1, dtype=torch.int32, device=dev)
        self.scale = torch.ones(1, device=dev)
        nbytes = numel * es
        self.a = C.ShardGradOp(comm, grads.buf, 0, nbytes, _code(dtype), self.shard.data_ptr(), self.gpart.data_ptr(), 1.0 / P, True, False, cfg)
        self.norm = None
        if mode == "clip":
            self.norm = C.GradNormOp(comm, box.buf, 0, self.gpart.data_ptr(), self.gpart.numel(), 0, self.out.data_ptr())
        elif mode == "scaled":
            self.norm = C.LossScaleNormOp(comm, box.buf, 0, self.gpart.data_ptr(), self.gpart.numel(), 0, self.out.data_ptr(), self.t.data_ptr())
            self.norm.set_scale_ptr(self.scale.data_ptr())
        coef = self.out[1:].data_ptr() if self.norm is not None else 0
        T = len(SIZES_BUCKET)
        self.segs, views, off = [], [[], []], 0
        for t, n in enumerate(SIZES_BUCKET):
            a, b = max(off, self.lo), min(off + n, self.hi)
            if a < b:
                self.segs.append((a - self.lo, b - self.lo, t))
                for lst, buf in zip(views, (self.master, self.shard)):
                    lst.append(buf[a - self.lo: b - self.lo])
            off += n
        self.seg_ptr, self.seg_nblk = [0] * T, [0] * T
        if self.segs:
            self.plan = multi_tensor_plan(views)
            self.partials = torch.zeros(max(1, self.plan.n_blocks), 2, dtype=torch.float64, device=dev)
            self.norms = C.LarsNormsOp(*self.plan.args(), coef, self.partials.data_ptr())
            blk = 0
            for a, b, t in self.segs:
                nb = (b - a + 65535) // 65536
                self.seg_ptr[t], self.seg_nblk[t] = (self.partials.data_ptr() + 16 * blk, nb)
                blk += nb
        else:
            self.partials = torch.zeros(1, 2, dtype=torch.float64, device=dev)
            self.norms = C.LarsNormsOp(0, 0, 0, 0, 0, 0, 65536, coef, self.partials.data_ptr())
        self.ptrs = torch.tensor(self.seg_ptr, dtype=torch.int64, device=dev)
        self.nblk = torch.tensor(self.seg_nblk, dtype=torch.int32, device=dev)
        self.ratio = torch.zeros(T, device=dev)
        self.sums = torch.zeros(T, 2, dtype=torch.float64, device=dev)
        self.rop = C.LambRatioOp(comm, rbox.buf, 0, self.ptrs.data_ptr(), self.nblk.data_ptr(), T, self.ratio.data_ptr(), self.sums.data_ptr())
        self.table = torch.tensor([v for s in self.segs for v in s] or [0, 0, 0], dtype=torch.int32, device=dev)
        self.b = C.ShardLarsOp(comm, weights.buf, 0, nbytes, _code(dtype), self.shard.data_ptr(), coef, self.master.data_ptr(), self.mom.data_ptr(),
                               self.table.data_ptr(), len(self.segs), self.sums.data_ptr(), False, cfg)
        for op in (self.norms, self.b):
            op.set_hyper(LRS[0], HP["momentum"], wd, HP["trust_coefficient"])
            if mode == "scaled":
                op.set_device_step(coef, self.t.data_ptr())


def _run(C, P, dtype, wd, mode, overflow_step=None, check_oracle=True):
    """Three steps of the in-bucket LARS program on a virtual world of P ranks (lr changes before the last); returns the published
    weights after each step."""
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    payload = sum(SIZES_BUCKET)
    numel = (payload * es + 15) // 16 * 16 // es     # the bucket total is padded to 16 bytes; the tail is not a parameter
    torch.manual_seed(5)
    w0 = torch.randn(numel, device=w.device)
    w0[payload:] = 0
    off = sum(SIZES_BUCKET[:ZERO_PARAM])
    w0[off:off + SIZES_BUCKET[ZERO_PARAM]] = 0
    w0 = w0.to(dtype)
    nbytes = numel * es
    grads, weights = w.alloc(nbytes), w.alloc(nbytes)
    box, rbox = w.alloc(2 * C.MAX_PEERS * 8), w.alloc(C.LambRatioOp.box_bytes(len(SIZES_BUCKET)))
    ranks = []
    for r in range(P):
        weights.view(r, dtype, numel).copy_(w0)
        ranks.append(_Rank(C, w, r, dtype, numel, grads, weights, box, rbox, w0, w.cfg(6), mode, wd))
    assert any(len([s for s in rk.segs if s[2] == BIG_PARAM]) for rk in ranks)
    if P > 1:
        assert sum(1 for rk in ranks for s in rk.segs if s[2] == BIG_PARAM) >= 2, "the odd-sized parameter is cut by a slice boundary"
    published, prev_lr = [], None
    for step, lr in enumerate(LRS):
        for rk in ranks:
            for op in (rk.norms, rk.b):
                op.set_hyper(lr, HP["momentum"], wd, HP["trust_coefficient"])
        gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        for g in gs:
            g[payload:] = 0
        if step == overflow_step:
            gs[P - 1][SIZES_BUCKET[0] + 1] = float("inf")
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
        ref = _owned_slice_sum(gs, _f32(1.0 / P))
        w.run(None, ops=[rk.a for rk in ranks])
        coef = 1.0
        if mode == "clip":
            for rk in ranks:
                rk.norm.set_max_norm(0.5 * math.sqrt(float(ref.double().square().sum())))   # clips
        if ranks[0].norm is not None:
            w.run(None, ops=[rk.norm for rk in ranks])
            coef = float(ranks[0].out[1])
            if mode == "clip":
                assert coef < 1.0
        before = [(rk.master.clone(), rk.mom.clone(), rk.shard.clone()) for rk in ranks]
        w.run(None, ops=[rk.norms for rk in ranks])
        w.run(None, ops=[rk.rop for rk in ranks])
        w.run(None, ops=[rk.b for rk in ranks])
        torch.cuda.synchronize()
        pub = weights.view(0, dtype, numel).clone()
        for r in range(P):
            assert torch.equal(weights.view(r, dtype, numel), pub), "every rank holds the same published weights"
        published.append(pub)
        if step == overflow_step:
            assert float(ranks[0].out[2]) == 1.0, "the overflow is voted"
            for rk, (m, v, _) in zip(ranks, before):
                assert torch.equal(rk.master, m) and torch.equal(rk.mom, v), "a skipped step leaves master and momentum alone"
            assert torch.equal(pub, published[-2] if step > 0 else w0), "a skipped step publishes nothing new"
            continue
        # the exchanged per-parameter sums: the fixed-order sum of the kernel's segment partials, identical bits on every rank
        local_sums = []
        for rk in ranks:
            part, blk, local = rk.partials.cpu(), 0, torch.zeros(len(SIZES_BUCKET), 2, dtype=torch.float64)
            for a, b, t in rk.segs:
                nb = (b - a + 65535) // 65536
                for k in range(nb):
                    local[t] += part[blk + k]
                blk += nb
            local_sums.append(local)
        want = torch.zeros(len(SIZES_BUCKET), 2, dtype=torch.float64)
        for local in local_sums:
            want += local
        for rk in ranks:
            assert torch.equal(rk.sums.cpu(), want), (P, dtype, step)
        if not check_oracle:
            prev_lr = lr
            continue
        full = {k: torch.zeros(numel, dtype=torch.float64) for k in ("w", "v", "g")}
        for rk, (m, v, g) in zip(ranks, before):
            n = rk.hi - rk.lo
            for k, t in zip(("w", "v", "g"), (m, v, g)):
                full[k][rk.lo:rk.hi] = t[:n].cpu().double()
        params, off = [], 0
        for n in SIZES_BUCKET:
            params.append(tuple(full[k][off:off + n] for k in ("w", "g", "v")))
            off += n
        hp = lo.Lars(lr=lr, weight_decay=wd, coef=coef, **HP)
        res = lo.lars(params, hp)
        for t, (pw, pg, _) in enumerate(params):
            sq = [x * x for x in pw.tolist()]
            assert abs(float(want[t, 0]) - math.fsum(sq)) <= sum_bound(sq), (P, dtype, step, t)
            gt = (pg * lo.f32(coef)).float().double()   # the fp32 g̃ the kernels square
            sg = [x * x for x in gt.tolist()]
            assert abs(float(want[t, 1]) - math.fsum(sg)) <= sum_bound(sg), (P, dtype, step, t)
            # the trust the apply kernel takes: the oracle's rule on the exchanged sums, bit for bit
            tr = lo.trust(float(want[t, 0]), float(want[t, 1]), hp)
            if wd != 0 and t == BIG_PARAM:
                assert tr != 1.0
            if t == ZERO_PARAM and step == 0:
                assert tr == 1.0, "an all-zero parameter gets trust 1"
        got = torch.zeros(numel, dtype=torch.float32)
        got_v = torch.zeros(numel, dtype=torch.float32)
        for rk in ranks:
            got[rk.lo:rk.hi] = rk.master[: rk.hi - rk.lo].cpu()
            got_v[rk.lo:rk.hi] = rk.mom[: rk.hi - rk.lo].cpu()
        off = 0
        for t, (n, out) in enumerate(zip(SIZES_BUCKET, res)):
            _check(got[off:off + n], out[0], out[3], f"master P={P} {dtype} wd={wd} {mode} step {step} param {t}")
            _check(got_v[off:off + n], out[1], out[4], f"momentum P={P} {dtype} wd={wd} {mode} step {step} param {t}")
            off += n
        assert torch.count_nonzero(got[payload:]).item() == 0, "the padding stays zero"
        assert torch.equal(pub, got.to(dtype).to(w.device)), "published weights = owner's master rounded once"
        prev_lr = lr
    w.check()
    return published


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("wd,mode", [(5e-4, "plain"), (0.0, "plain"), (5e-4, "clip")])
def test_in_bucket_lars_matches_oracle(C, P, dtype, wd, mode):
    _run(C, P, dtype, wd, mode)


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_in_bucket_lars_overflow_is_skipped_everywhere(C, P, dtype):
    _run(C, P, dtype, 5e-4, "scaled", overflow_step=1)


@pytest.mark.parametrize("P", [1, 3, 8])
def test_loss_scaling_at_scale_one_is_bit_identical(C, P):
    plain = _run(C, P, torch.bfloat16, 5e-4, "plain", check_oracle=False)
    scaled = _run(C, P, torch.bfloat16, 5e-4, "scaled", check_oracle=False)
    for a, b in zip(plain, scaled):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def _lars_train_worker(rank, world):
    """A small conv + BatchNorm model with a decay and a no-decay group: make_sharded_fused_lars against FusedLARS without bagua
    for 16 steps (lr changes at step 8), with and without clipping; a checkpoint after step 8 resumes bit-identically; re-bucketing
    mid-run keeps the state."""
    import torch.distributed as dist
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.ops.optim import FusedLARS
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lars

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False

    def groups(m):
        return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 5e-4},
                {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]

    def batch(it):
        g = torch.Generator(device=dev).manual_seed(100 * it + rank)
        return torch.randn(4, 3, 16, 16, device=dev, generator=g)

    def lr_at(it):
        return 0.5 if it < 8 else 0.2

    out = {}
    for bound in (None, 0.5):
        torch.manual_seed(9)
        # the head's weight (64·16·16 × 40 = 655360) spans ten 65536-element chunks: its segment has several stage-1 blocks
        base = nn.Sequential(nn.Conv2d(3, 64, 3, padding=1), nn.BatchNorm2d(64), nn.ReLU(), nn.Flatten(), nn.Linear(64 * 16 * 16, 40)).to(dev)
        oracle = copy.deepcopy(base)
        oopt = FusedLARS(groups(oracle), lr=0.5)

        def build(state=None, model_sd=None):
            m = copy.deepcopy(base)
            if model_sd is not None:
                m.load_state_dict(model_sd)
            o = make_sharded_fused_lars(groups(m), lr=0.5, max_grad_norm=bound)
            if state is not None:
                o.load_state_dict(state)
            m = m.with_bagua([o], FusedGradientAllReduceAlgorithm(o))
            assert all(b.allreduce_variant.startswith("fused_lars_") for b in m.bagua_buckets), [b.allreduce_variant for b in m.bagua_buckets]
            return m, o

        def train(m, o, its, rebucket_at=None):
            for it in its:
                if it == rebucket_at:
                    m.bagua_ddp._reset_buckets()
                for g in o.param_groups:
                    g["lr"] = lr_at(it)
                o.zero_grad()
                m(batch(it)).pow(2).mean().backward()
                o.step()

        model, opt = build()
        train(model, opt, range(8))
        torch.cuda.synchronize()
        sd, msd = copy.deepcopy(opt.state_dict()), {k: v.clone() for k, v in model.state_dict().items()}
        assert sd["sharded_fused"] == "lars" and sd["steps"] == 8
        train(model, opt, range(8, 16))
        torch.cuda.synchronize()
        final = torch.cat([p.detach().reshape(-1) for p in model.parameters()])

        model2, opt2 = build(sd, msd)
        train(model2, opt2, range(8, 16), rebucket_at=12)
        torch.cuda.synchronize()
        final2 = torch.cat([p.detach().reshape(-1) for p in model2.parameters()])
        assert torch.equal(final2, final), f"resumed / re-bucketed run differs: max {(final2 - final).abs().max().item()}"

        for it in range(16):
            for g in oopt.param_groups:
                g["lr"] = lr_at(it)
            oopt.zero_grad()
            oracle(batch(it)).pow(2).mean().backward()
            if world > 1:
                for p in oracle.parameters():
                    dist.all_reduce(p.grad)
                    p.grad /= world
            if bound is not None:
                torch.nn.utils.clip_grad_norm_(oracle.parameters(), bound)
            oopt.step()
        want = torch.cat([p.detach().reshape(-1) for p in oracle.parameters()])
        torch.testing.assert_close(final, want, rtol=1e-4, atol=2e-5)
        if bound is not None:
            assert opt.last_grad_norm is not None
        out[str(bound)] = final.cpu()
    return out


def test_self_peer_lars_training_matches_fused_lars():
    run_distributed(_lars_train_worker, world=1, use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
def test_lars_training_on_real_peers():
    n = min(torch.cuda.device_count(), 8)
    if n < 2:
        pytest.skip("needs 2 or more GPUs")
    res = run_distributed(_lars_train_worker, world=n, use_cuda=True, timeout=300)
    for r in res[1:]:
        for k in res[0]:
            assert torch.equal(r[k], res[0][k])
