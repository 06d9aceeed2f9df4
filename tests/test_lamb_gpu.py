"""LAMB on the GPU.

* ``FusedLAMB`` (the two multi-tensor kernels) against the float64 oracle of ``tests/lamb_oracle.py``.
* The in-bucket kernels (phase A ``shard_grad``, the moments, the per-parameter ratio exchange, apply + all-gather) on virtual peer
  worlds of P = 1 … 8 ranks, with a bucket whose slices cut parameters anywhere.
* ``make_sharded_fused_lamb`` end to end in self-peer mode (and on 2+ real GPUs) against ``FusedLAMB`` without bagua.
"""
import copy
import math

import pytest
import torch

from tests import lamb_oracle as lo
from tests.mp_utils import run_distributed
from tests.optim_oracle import check
from tests.test_virtual_peer_gpu import _code, _f32, _owned_slice_sum, _world

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


# ---------------------------------------------------------------------------------------------------------------------
# FusedLAMB
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [0, 1, 65535, 65536, 65537, 2 * 65536 + 3]
PAD = 32


def _padded(n, dtype, gen, scale=1.0):
    """A tensor of n elements inside a larger buffer whose margins hold sentinel values."""
    buf = torch.full((n + 2 * PAD,), 7.0, device="cuda", dtype=dtype)
    t = buf[PAD:PAD + n]
    t.copy_((torch.randn(n, device="cuda", generator=gen) * scale).to(dtype))
    return buf, t


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_fused_lamb_matches_oracle(dtype):
    from bagua_b200.ops.optim import FusedLAMB

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
    # the decay group holds every tensor of several 65536-element chunks and the channels_last one: their ratio is a fixed-order sum
    # over several blocks (stage 2), and it is applied
    groups = [{"params": params[2:], "weight_decay": 0.01}, {"params": params[:2], "weight_decay": 0.0}]
    opt = FusedLAMB(groups, lr=1e-2, betas=(0.9, 0.999), eps=1e-6)
    mixed = dtype != torch.float32
    for step in range(1, 4):
        for p in params:
            if p is cl:
                p.grad = (torch.randn(p.shape, device="cuda", generator=gen) * 0.1).to(dtype)   # contiguous: a copy in the layout
            elif step > 1:
                p.grad.copy_((torch.randn(p.numel(), device="cuda", generator=gen) * 0.1).to(dtype))
        def flat(t):   # memory order, as the kernels walk it
            return torch.as_strided(t, (t.numel(),), (1,))

        before = {}
        for p in params:
            st = opt.state[p]
            w = st["master"] if "master" in st else p.detach().float()
            zeros = torch.zeros(p.numel(), device="cuda")
            g = p.grad.contiguous(memory_format=torch.channels_last) if p is cl else p.grad
            before[p] = (flat(w).clone(), flat(g).clone(), flat(st["exp_avg"]).clone() if "exp_avg" in st else zeros,
                         flat(st["exp_avg_sq"]).clone() if "exp_avg_sq" in st else zeros)
        opt.step()
        torch.cuda.synchronize()
        for gi, group in enumerate(groups):
            hp = lo.Lamb(lr=1e-2, step=step, weight_decay=group["weight_decay"])
            for p in group["params"]:
                w_new, a_new, b_new, r, tol_w, tol_a, tol_b = lo.lamb([before[p]], hp)[0]
                if group["weight_decay"] != 0 and p.numel() > 65536:
                    assert r != 1.0, "a multi-chunk parameter must get a real trust ratio"
                st = opt.state[p]
                check(flat(st["exp_avg"]), a_new, tol_a, f"exp_avg {dtype} n={p.numel()} step {step}")
                check(flat(st["exp_avg_sq"]), b_new, tol_b, f"exp_avg_sq {dtype} n={p.numel()} step {step}")
                if mixed:
                    check(flat(st["master"]), w_new, tol_w, f"master {dtype} n={p.numel()} step {step}")
                    assert torch.equal(flat(p.detach()), flat(st["master"]).to(dtype)), "model copy = master rounded once"
                else:
                    check(flat(p.detach()), w_new, tol_w, f"param {dtype} n={p.numel()} step {step}")
                assert torch.count_nonzero(p.grad).item() == 0, "zero_grad_in_step clears the gradient"
        for b in bufs:
            assert torch.all(b[:PAD] == 7.0) and torch.all(b[-PAD:] == 7.0), "write outside a tensor"


# ---------------------------------------------------------------------------------------------------------------------
# in-bucket kernels on a virtual peer world
# ---------------------------------------------------------------------------------------------------------------------
WORLDS = [1, 2, 3, 4, 8]
# about 12 parameters packed back to back: tiny ones share 16-byte vectors, one is large enough to straddle several slices, one is zero
SIZES_BUCKET = [1, 3, 7, 1, 513, 2, 20000, 5, 1, 777, 4099, 3, 2 * 65536 + 5]
BIG_PARAM = 12   # more than two 65536-element chunks, straddles the slices at P ≥ 2: segments of several stage-1 blocks
ZERO_PARAM = 9


class _Rank:
    def __init__(self, C, w, r, dtype, numel, grads, weights, box, rbox, w0, cfg, clip):
        from bagua_b200.ops.optim import multi_tensor_plan

        es = torch.empty(0, dtype=dtype).element_size()
        P, dev = w.world, w.device
        per = 16 // es
        vpr = (numel * es // 16 + P - 1) // P
        self.lo, self.hi, length = r * vpr * per, min((r + 1) * vpr * per, numel), vpr * per
        self.shard = torch.zeros(length, device=dev)
        self.master = torch.zeros(length, device=dev)
        if self.hi > self.lo:
            self.master[: self.hi - self.lo].copy_(w0[self.lo:self.hi].float())
        self.m1, self.m2 = torch.zeros(length, device=dev), torch.zeros(length, device=dev)
        self.gpart = torch.zeros(1, C.MAX_COMM_BLOCKS, dtype=torch.float64, device=dev)
        self.out = torch.zeros(2, device=dev)
        nbytes = numel * es
        self.a = C.ShardGradOp(w.comms[r], grads.buf, 0, nbytes, _code(dtype), self.shard.data_ptr(), self.gpart.data_ptr(), 1.0 / P, True, False, cfg)
        self.norm = C.GradNormOp(w.comms[r], box.buf, 0, self.gpart.data_ptr(), self.gpart.numel(), 0, self.out.data_ptr()) if clip else None
        coef = self.out[1:].data_ptr() if clip else 0
        T = len(SIZES_BUCKET)
        self.segs, views, off = [], [[], [], [], []], 0
        for t, n in enumerate(SIZES_BUCKET):
            a, b = max(off, self.lo), min(off + n, self.hi)
            if a < b:
                self.segs.append((a - self.lo, b - self.lo, t))
                for lst, buf in zip(views, (self.master, self.shard, self.m1, self.m2)):
                    lst.append(buf[a - self.lo: b - self.lo])
            off += n
        self.seg_ptr, self.seg_nblk = [0] * T, [0] * T
        if self.segs:
            self.plan = multi_tensor_plan(views)
            self.partials = torch.zeros(max(1, self.plan.n_blocks), 2, dtype=torch.float64, device=dev)
            self.moments = C.LambMomentsOp(*self.plan.args(), coef, self.partials.data_ptr())
            blk = 0
            for a, b, t in self.segs:
                nb = (b - a + 65535) // 65536
                self.seg_ptr[t], self.seg_nblk[t] = (self.partials.data_ptr() + 16 * blk, nb)
                blk += nb
        else:
            self.partials = torch.zeros(1, 2, dtype=torch.float64, device=dev)
            self.moments = C.LambMomentsOp(0, 0, 0, 0, 0, 0, 65536, coef, self.partials.data_ptr())
        self.ptrs = torch.tensor(self.seg_ptr, dtype=torch.int64, device=dev)
        self.nblk = torch.tensor(self.seg_nblk, dtype=torch.int32, device=dev)
        self.ratio = torch.zeros(T, device=dev)
        self.sums = torch.zeros(T, 2, dtype=torch.float64, device=dev)
        self.rop = C.LambRatioOp(w.comms[r], rbox.buf, 0, self.ptrs.data_ptr(), self.nblk.data_ptr(), T, self.ratio.data_ptr(), self.sums.data_ptr())
        self.table = torch.tensor([v for s in self.segs for v in s] or [0, 0, 0], dtype=torch.int32, device=dev)
        self.b = C.ShardLambOp(w.comms[r], weights.buf, 0, nbytes, _code(dtype), self.master.data_ptr(), self.m1.data_ptr(), self.m2.data_ptr(),
                               self.table.data_ptr(), len(self.segs), self.ratio.data_ptr(), False, cfg)


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("wd,clip", [(0.01, False), (0.0, False), (0.01, True)])
def test_in_bucket_lamb_matches_oracle(C, P, dtype, wd, clip):
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
        ranks.append(_Rank(C, w, r, dtype, numel, grads, weights, box, rbox, w0, w.cfg(6), clip))
        ranks[r].moments.set_hyper(1e-2, 0.9, 0.999, 1e-6, wd)
        ranks[r].b.set_hyper(1e-2, 0.9, 0.999, 1e-6, wd)
    assert any(len([s for s in rk.segs if s[2] == 6]) for rk in ranks)
    for step in range(1, 4):
        gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        for g in gs:
            g[payload:] = 0
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
        ref = _owned_slice_sum(gs, _f32(1.0 / P))
        w.run(None, ops=[rk.a for rk in ranks])
        for r in range(P):
            assert torch.count_nonzero(grads.view(r, torch.uint8, nbytes)).item() == 0, "gradient bucket must be cleared"
        coef = 1.0
        if clip:
            for rk in ranks:
                rk.norm.set_max_norm(0.5 * math.sqrt(float(ref.double().square().sum())))   # clips
            w.run(None, ops=[rk.norm for rk in ranks])
            coef = float(ranks[0].out[1])
            assert coef < 1.0
        before = [(rk.master.clone(), rk.m1.clone(), rk.m2.clone()) for rk in ranks]
        w.run(None, ops=[rk.moments for rk in ranks])
        w.run(None, ops=[rk.rop for rk in ranks])
        # the per-parameter sums: the fixed-order oracle fed with the kernel's segment partials, identical bits on every rank
        want = torch.zeros(len(SIZES_BUCKET), 2, dtype=torch.float64)
        for rk in ranks:
            part = rk.partials.cpu()
            local = torch.zeros(len(SIZES_BUCKET), 2, dtype=torch.float64)
            blk = 0
            for a, b, t in rk.segs:
                nb = (b - a + 65535) // 65536
                for k in range(nb):
                    local[t] += part[blk + k]
                blk += nb
            want += local
        for rk in ranks:
            assert torch.equal(rk.sums.cpu(), want), (P, dtype, step)
            assert torch.equal(rk.ratio.cpu(), ranks[0].ratio.cpu()), "every rank must compute the same ratio bits"
        # the whole-parameter state before the step, assembled from the ranks' shards
        full = {k: torch.zeros(numel, dtype=torch.float64) for k in ("w", "g", "a", "b")}
        for rk, (m, a, b) in zip(ranks, before):
            n = rk.hi - rk.lo
            for k, t in zip(("w", "g", "a", "b"), (m, rk.shard, a, b)):
                full[k][rk.lo:rk.hi] = t[:n].cpu().double()
        params, off = [], 0
        for n in SIZES_BUCKET:
            params.append(tuple(full[k][off:off + n] for k in ("w", "g", "a", "b")))
            off += n
        res = lo.lamb(params, lo.Lamb(lr=1e-2, step=step, weight_decay=wd, coef=coef))
        # Σw² against the exact sum (w² of an fp32 w is exact in float64): only the order of the additions differs, so the gap is
        # within the a-priori bound of a float64 sum in any order. Σu² against the oracle's u: the fp32 rounding of each u, plus that.
        hp = lo.Lamb(lr=1e-2, step=step, weight_decay=wd, coef=coef)
        for t, (pw, pg, pa, pb) in enumerate(params):
            sq = [x * x for x in pw.tolist()]
            assert abs(float(want[t, 0]) - math.fsum(sq)) <= lo.sum_bound(sq), (P, dtype, step, t, float(want[t, 0]), math.fsum(sq))
            u, tol_u = lo.direction(pw, pg, pa, pb, hp)
            su = [x * x for x in (u.abs() + tol_u).tolist()]
            gap = float((2.0 * u.abs() * tol_u + tol_u * tol_u).sum()) + lo.sum_bound(su)
            assert abs(float(want[t, 1]) - float(u.square().sum())) <= gap, (P, dtype, step, t, float(want[t, 1]), float(u.square().sum()), gap)
        if P == 1:
            assert int(ranks[0].nblk[BIG_PARAM]) == 3, "the big parameter's segment spans three stage-1 blocks"
        if wd != 0:
            assert float(ranks[0].ratio[BIG_PARAM]) != 1.0
        if step == 1:
            assert float(ranks[0].ratio[ZERO_PARAM]) == 1.0, "an all-zero parameter gets r = 1"
        w.run(None, ops=[rk.b for rk in ranks])
        got = torch.zeros(numel, dtype=torch.float32)
        for rk in ranks:
            got[rk.lo:rk.hi] = rk.master[: rk.hi - rk.lo].cpu()
        off = 0
        for t, (n, out) in enumerate(zip(SIZES_BUCKET, res)):
            check(got[off:off + n], out[0], out[4], f"master P={P} {dtype} wd={wd} step {step} param {t}")
            off += n
        assert torch.count_nonzero(got[payload:]).item() == 0, "the padding stays zero"
        model = got.to(dtype).to(w.device)
        for r in range(P):
            assert torch.equal(weights.view(r, dtype, numel), model), "published weights = owner's master rounded once"


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def _lamb_train_worker(rank, world):
    """A small transformer encoder with a wide head, a decay and a no-decay group: make_sharded_fused_lamb against FusedLAMB without bagua for
    20 steps, with and without clipping; a checkpoint after step 10 resumes bit-identically; re-bucketing mid-run keeps the state."""
    import torch.distributed as dist
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.ops.optim import FusedLAMB
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lamb

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False

    def groups(m):
        return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 0.01},
                {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]

    def batch(it):
        g = torch.Generator(device=dev).manual_seed(100 * it + rank)
        return torch.randn(4, 10, 32, device=dev, generator=g)

    out = {}
    for bound in (None, 0.05):
        torch.manual_seed(9)
        # the head's weight (32 × 4200) spans three 65536-element chunks: its segment has several stage-1 blocks
        base = nn.Sequential(nn.TransformerEncoderLayer(32, 4, 64, dropout=0.0, batch_first=True), nn.Linear(32, 4200)).to(dev)
        oracle = copy.deepcopy(base)
        oopt = FusedLAMB(groups(oracle), lr=1e-3)

        def build(state=None, model_sd=None):
            m = copy.deepcopy(base)
            if model_sd is not None:
                m.load_state_dict(model_sd)
            o = make_sharded_fused_lamb(groups(m), lr=1e-3, max_grad_norm=bound)
            if state is not None:
                o.load_state_dict(state)
            m = m.with_bagua([o], FusedGradientAllReduceAlgorithm(o))
            assert all(b.allreduce_variant.startswith("fused_lamb_") for b in m.bagua_buckets), [b.allreduce_variant for b in m.bagua_buckets]
            return m, o

        def train(m, o, its, rebucket_at=None):
            for it in its:
                if it == rebucket_at:
                    m.bagua_ddp._reset_buckets()
                o.zero_grad()
                m(batch(it)).pow(2).mean().backward()
                o.step()

        model, opt = build()
        train(model, opt, range(10))
        torch.cuda.synchronize()
        sd, msd = copy.deepcopy(opt.state_dict()), {k: v.clone() for k, v in model.state_dict().items()}
        train(model, opt, range(10, 20))
        torch.cuda.synchronize()
        final = torch.cat([p.detach().reshape(-1) for p in model.parameters()])

        model2, opt2 = build(sd, msd)
        train(model2, opt2, range(10, 20), rebucket_at=15)
        torch.cuda.synchronize()
        final2 = torch.cat([p.detach().reshape(-1) for p in model2.parameters()])
        assert torch.equal(final2, final), f"resumed / re-bucketed run differs: max {(final2 - final).abs().max().item()}"

        for it in range(20):
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


def test_self_peer_lamb_training_matches_fused_lamb():
    run_distributed(_lamb_train_worker, world=1, use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
def test_lamb_training_on_real_peers():
    n = min(torch.cuda.device_count(), 8)
    if n < 2:
        pytest.skip("needs 2 or more GPUs")
    res = run_distributed(_lamb_train_worker, world=n, use_cuda=True, timeout=300)
    for r in res[1:]:
        for k in res[0]:
            assert torch.equal(r[k], res[0][k])
