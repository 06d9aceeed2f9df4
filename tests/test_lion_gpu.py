"""Lion on the GPU, bit for bit against the fp32 replay (``bagua_b200.ops.optim.lion_reference_step_``, run on the CPU).

* ``FusedLion`` (the multi-tensor kernel) in fp32, bf16 and fp16: sizes 0, 1 and the chunk edges, misaligned views with sentinels,
  an ``lr`` change, zero-gradient elements and a NaN element.
* ``AllReduceLionOp`` and ``ShardLionOp`` on virtual peer worlds of P = 1 … 8 ranks with ragged slices: masters and ``exp_avg``
  against the replay on the owned-slice sum, the published weights, the cleared bucket, the sentinels past the bucket, a clip
  coefficient, an overflowed loss-scaled step, and loss scaling at scale 1 against the op without it.
* ``make_sharded_fused_lion`` end to end in self-peer mode (and on 2+ real GPUs): plain, clipped, accumulating, with an EMA and
  fp16 loss scaling with a forced overflow, against the replay driven by the gradients of a model without bagua; a checkpoint
  resume and a re-bucketing give bit-identical weights.
"""
import copy

import pytest
import torch

from bagua_b200.ops.optim import lion_reference_step_
from tests.mp_utils import run_distributed
from tests.test_virtual_peer_gpu import _code, _f32, _owned_slice_sum, _world

pytestmark = pytest.mark.gpu

BETAS = (0.9, 0.99)


def _bits(t):
    """The fp32 bit patterns of ``t``, every NaN as the canonical one (the payload depends on where a NaN arose)."""
    t = t.detach().cpu().float()
    b = t.view(torch.int32).clone()
    b[torch.isnan(t)] = 0x7FC00000
    return b


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


# ---------------------------------------------------------------------------------------------------------------------
# FusedLion
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [0, 1, 65535, 65536, 65537, 2 * 65536 + 3]
PAD = 32
LRS = [3e-3, 3e-3, 1e-3]   # an lr change between the second and the third step


def _padded(n, dtype, gen, misalign, scale=1.0):
    """n elements inside a buffer whose margins hold sentinels; ``misalign`` starts the view one element past a 16-byte boundary."""
    buf = torch.full((n + 2 * PAD,), 7.0, device="cuda", dtype=dtype)
    t = buf[PAD + misalign:PAD + misalign + n]
    t.copy_((torch.randn(n, device="cuda", generator=gen) * scale).to(dtype))
    return buf, t


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_fused_lion_is_the_replay_bit_for_bit(dtype):
    from bagua_b200.ops.optim import FusedLion

    gen = torch.Generator(device="cuda").manual_seed(3)
    params, bufs = [], []
    for i, n in enumerate(SIZES):
        wb, w = _padded(n, dtype, gen, misalign=i % 2)
        gb, g = _padded(n, dtype, gen, misalign=i % 2, scale=0.1)
        p = torch.nn.Parameter(torch.empty(0, device="cuda", dtype=dtype))
        p.data, p.grad = w, g
        params.append(p)
        bufs += [wb, gb]
    groups = [{"params": params[:3], "weight_decay": 0.1}, {"params": params[3:], "weight_decay": 0.0}]
    opt = FusedLion(groups, lr=LRS[0], betas=BETAS)
    mixed = dtype != torch.float32
    big = params[-1]
    ref = {p: (p.detach().float().cpu(), torch.zeros(p.numel())) for p in params}
    for step, lr in enumerate(LRS):
        for g in opt.param_groups:
            g["lr"] = lr
        for p in params:
            if step > 0:
                p.grad.copy_((torch.randn(p.numel(), device="cuda", generator=gen) * 0.1).to(dtype))
        big.grad[:100] = 0          # with m = 0 at the first step: u = 0, sign 0, the weight only decays
        if step == 1:
            big.grad[1000] = float("nan")
        grads = {p: p.grad.detach().cpu() for p in params}
        opt.step()
        torch.cuda.synchronize()
        for group in groups:
            for p in group["params"]:
                w, m = ref[p]
                lion_reference_step_(w, m, grads[p], lr, BETAS, group["weight_decay"])
                st = opt.state[p]
                assert _same(st["exp_avg"], m), f"exp_avg {dtype} n={p.numel()} step {step}"
                got = st["master"].cpu() if mixed else p.detach().cpu()
                assert _same(got, w), f"weights {dtype} n={p.numel()} step {step}"
                if mixed:
                    assert _same(p, w.to(dtype)), "model copy = master rounded once"
                assert torch.count_nonzero(p.grad).item() == 0, "zero_grad_in_step clears the gradient"
        for b in bufs:
            assert torch.all(b[:PAD] == 7.0) and torch.all(b[-PAD + 1:] == 7.0), "write outside a tensor"
    w = opt.state[big]["master"] if mixed else big.detach()
    assert torch.isnan(w[1000]) and int(torch.isnan(w).sum()) == 1, "a NaN gradient element poisons its own weight only"


# ---------------------------------------------------------------------------------------------------------------------
# in-bucket kernels on a virtual peer world
# ---------------------------------------------------------------------------------------------------------------------
WORLDS = [1, 2, 3, 4, 8]
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
TAIL = 64   # bytes past the bucket in every symmetric buffer: sentinels no kernel may touch


def _numel(dtype):
    return (1 << 15) + 16 // torch.empty(0, dtype=dtype).element_size() * 5   # slices of unequal length


def _shard(numel, es, P, r):
    per = 16 // es
    vpr = (numel * es // 16 + P - 1) // P
    return r * vpr * per, min((r + 1) * vpr * per, numel), vpr * per


def _lion_world(C, P, dtype, mode, lr=2e-3, wd=0.1, steps=3, overflow_step=None):
    """``steps`` Lion steps on a virtual world of P ranks. mode: "fused" (AllReduceLionOp), "plain" / "clip" / "scaled" (ShardGradOp,
    then the norm exchange for clip and scaled, then ShardLionOp). Each step is checked against the replay on every rank; returns
    the published weights after each step."""
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    numel = _numel(dtype)
    nbytes = numel * es
    torch.manual_seed(17)
    w0 = torch.randn(numel, device=w.device).to(dtype)
    grads, weights = w.alloc(nbytes + TAIL), w.alloc(nbytes + TAIL)
    box = w.alloc(2 * C.MAX_PEERS * 8)
    ranks = []
    for r in range(P):
        weights.view(r, torch.uint8, nbytes + TAIL)[nbytes:].fill_(0xA5)
        grads.view(r, torch.uint8, nbytes + TAIL)[nbytes:].fill_(0x5A)
        weights.view(r, dtype, numel).copy_(w0)
        lo, hi, length = _shard(numel, es, P, r)
        rk = {"lo": lo, "hi": hi, "master": torch.zeros(length, device=w.device), "m": torch.zeros(length, device=w.device),
              "shard": torch.zeros(length, device=w.device), "part": torch.zeros(1, C.MAX_COMM_BLOCKS, dtype=torch.float64, device=w.device),
              "out": torch.zeros(3, device=w.device), "t": torch.zeros(1, dtype=torch.int32, device=w.device),
              "scale": torch.ones(1, device=w.device), "unit": torch.ones(1, device=w.device)}
        if hi > lo:
            rk["master"][: hi - lo].copy_(w0[lo:hi].float())
        comm, cfg, code = w.comms[r], w.cfg(6), _code(dtype)
        if mode == "fused":
            rk["ops"] = [C.AllReduceLionOp(comm, grads.buf, weights.buf, 0, 0, nbytes, code, rk["master"].data_ptr(), rk["m"].data_ptr(), 1.0 / P, True,
                                           False, cfg)]
        else:
            a = C.ShardGradOp(comm, grads.buf, 0, nbytes, code, rk["shard"].data_ptr(), rk["part"].data_ptr(), 1.0 / P, True, False, cfg)
            coef = rk["out"][1:].data_ptr() if mode != "plain" else rk["unit"].data_ptr()
            b = C.ShardLionOp(comm, weights.buf, 0, nbytes, code, rk["shard"].data_ptr(), coef, rk["master"].data_ptr(), rk["m"].data_ptr(), False, cfg)
            rk["ops"] = [a]
            if mode == "clip":
                rk["ops"].append(C.GradNormOp(comm, box.buf, 0, rk["part"].data_ptr(), rk["part"].numel(), 0, rk["out"].data_ptr()))
                rk["ops"][-1].set_max_norm(20.0)
            elif mode == "scaled":
                n = C.LossScaleNormOp(comm, box.buf, 0, rk["part"].data_ptr(), rk["part"].numel(), 0, rk["out"].data_ptr(), rk["t"].data_ptr())
                n.set_scale_ptr(rk["scale"].data_ptr())
                rk["ops"].append(n)
                b.set_device_step(coef, rk["t"].data_ptr())
            rk["ops"].append(b)
        for op in rk["ops"]:
            if hasattr(op, "set_hyper"):
                op.set_hyper(lr, BETAS[0], BETAS[1], wd)
        ranks.append(rk)
    published = []
    for step in range(steps):
        gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        gs[0][:64] = 0
        if step == overflow_step:
            gs[P - 1][5] = float("inf")
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
        red = _owned_slice_sum(gs, _f32(1.0 / P))
        before = [(rk["master"].clone(), rk["m"].clone()) for rk in ranks]
        for k in range(len(ranks[0]["ops"])):
            w.run(None, ops=[rk["ops"][k] for rk in ranks])
        torch.cuda.synchronize()
        pub = weights.view(0, dtype, numel).clone()
        got = torch.zeros(numel)
        for r, rk in enumerate(ranks):
            assert torch.equal(weights.view(r, dtype, numel), pub), "every rank holds the same published weights"
            assert torch.all(weights.view(r, torch.uint8, nbytes + TAIL)[nbytes:] == 0xA5), "write past the weights"
            assert torch.all(grads.view(r, torch.uint8, nbytes + TAIL)[nbytes:] == 0x5A), "write past the gradient bucket"
            assert grads.view(r, dtype, numel).abs().max().item() == 0.0, "the gradient bucket is cleared on the way out"
        if step == overflow_step:
            assert float(ranks[0]["out"][2]) == 1.0, "the overflow is voted"
            for rk, (m0, e0) in zip(ranks, before):
                assert torch.equal(rk["master"], m0) and torch.equal(rk["m"], e0), "a skipped step changes no state bit"
            assert torch.equal(pub, published[-1] if published else w0), "a skipped step publishes nothing new"
            published.append(pub)
            continue
        for rk, (m0, e0) in zip(ranks, before):
            lo, hi = rk["lo"], rk["hi"]
            if hi <= lo:
                continue
            n = hi - lo
            if mode != "fused":
                assert torch.equal(rk["shard"][:n].cpu(), red[lo:hi]), "phase A: the shard is the owned-slice sum"
            coef = None if mode == "fused" else (rk["unit"] if mode == "plain" else rk["out"][1]).cpu().reshape(())
            if mode == "clip":
                assert float(coef) < 1.0, "the bound clips"
            wm, em = m0[:n].cpu(), e0[:n].cpu()
            lion_reference_step_(wm, em, red[lo:hi], lr, BETAS, wd, coef)
            assert torch.equal(rk["master"][:n].cpu(), wm), (P, dtype, mode, step)
            assert torch.equal(rk["m"][:n].cpu(), em), (P, dtype, mode, step)
            got[lo:hi] = wm
        assert torch.equal(pub.cpu(), got.to(dtype)), "published weights = the owners' masters rounded once"
        published.append(pub)
    w.check()
    return published


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_allreduce_lion_is_the_replay_on_the_owned_slice_sum(C, P, dtype):
    _lion_world(C, P, dtype, "fused")


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["plain", "clip"])
def test_shard_lion_is_the_replay_with_the_coefficient(C, P, dtype, mode):
    _lion_world(C, P, dtype, mode)


@pytest.mark.parametrize("P", [1, 3, 8])
def test_shard_lion_overflow_is_skipped_on_every_rank(C, P):
    _lion_world(C, P, torch.float16, "scaled", overflow_step=1)


@pytest.mark.parametrize("P", [1, 2, 8])
def test_loss_scaling_at_scale_one_is_bit_identical(C, P):
    plain = _lion_world(C, P, torch.bfloat16, "plain")
    scaled = _lion_world(C, P, torch.bfloat16, "scaled")
    assert all(torch.equal(a, b) for a, b in zip(plain, scaled))


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def _net(dev, dtype):
    import torch.nn as nn

    return nn.Sequential(nn.Linear(48, 96), nn.GELU(), nn.LayerNorm(96), nn.Linear(96, 10)).to(dev, dtype)


def _groups(m):
    return [{"params": [p for p in m.parameters() if p.dim() > 1], "weight_decay": 0.1},
            {"params": [p for p in m.parameters() if p.dim() <= 1], "weight_decay": 0.0}]


def _batch(dev, rank, it, k, dtype):
    g = torch.Generator(device=dev).manual_seed(1000 * it + 10 * k + rank)
    return torch.randn(16, 48, device=dev, generator=g).to(dtype)


def _lr_at(it):
    return 2e-3 if it < 6 else 1e-3


def _lion_train_worker(rank, world, variant):
    """make_sharded_fused_lion against the replay driven by a model without bagua: the replay's gradient is the oracle model's
    (all-reduced and averaged across the ranks, summed over K micro-batches with ``accumulate``), times the coefficient the sharded
    optimizer's norm exchange produced (clip, loss scaling). Plain runs are also compared with FusedLion. A checkpoint after step 6
    resumes, and a re-bucketing at step 9, with bit-identical weights."""
    import torch.distributed as dist

    import bagua_b200 as bagua
    from bagua_b200.amp import ShardedGradScaler
    from bagua_b200.ops.optim import FusedLion
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lion

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.use_deterministic_algorithms(True)
    dtype = torch.float16 if variant == "scaled" else torch.bfloat16
    K = 4 if variant == "accumulate" else 1
    kw = {"plain": {}, "clip": {"max_grad_norm": 0.05}, "accumulate": {"accumulate_grads": True}, "ema": {"ema_decay": 0.8},
          "scaled": {"loss_scaling": True}}[variant]
    steps, overflow = 12, (3 if variant == "scaled" else None)
    torch.manual_seed(9)
    base = _net(dev, dtype)
    oracle = copy.deepcopy(base)

    def build(state=None, model_sd=None):
        m = copy.deepcopy(base)
        if model_sd is not None:
            m.load_state_dict(model_sd)
        o = make_sharded_fused_lion(_groups(m), lr=_lr_at(0), betas=BETAS, **kw)
        if state is not None:
            o.load_state_dict(state)
        m = m.with_bagua([o], FusedGradientAllReduceAlgorithm(o))
        assert all(b.allreduce_variant.startswith("fused_lion_") for b in m.bagua_buckets), [b.allreduce_variant for b in m.bagua_buckets]
        return m, o

    scaler = ShardedGradScaler(init_scale=256.0, growth_interval=100) if variant == "scaled" else None

    def loss_of(m, it, k):
        return m(_batch(dev, rank, it, k, dtype)).float().pow(2).mean()

    def train(m, o, its, rebucket_at=None, log=None):
        for it in its:
            if it == rebucket_at:
                m.bagua_ddp._reset_buckets()
            for g in o.param_groups:
                g["lr"] = _lr_at(it)
            o.zero_grad()
            for k in range(K):
                loss = loss_of(m, it, k)
                if scaler is not None:
                    if it == overflow:
                        loss = loss * float("inf")
                    scaler.scale(loss).backward()
                else:
                    loss.backward()
            if scaler is not None:
                scale = float(scaler.get_scale())
                scaler.step(o)
                scaler.update()
            else:
                scale = 1.0
                o.step()
            if log is not None:
                clip = o._bucketing.clip
                coef = clip["out"][1].detach().cpu().reshape(()) if clip is not None else None
                skipped = bool(o.last_step_skipped.item()) if scaler is not None else False
                log.append((coef, scale, skipped))

    model, opt = build()
    log = []
    train(model, opt, range(6), log=log)
    torch.cuda.synchronize()
    sd, msd = copy.deepcopy(opt.state_dict()), {k: v.clone() for k, v in model.state_dict().items()}
    assert sd["sharded_fused"] == "lion"
    train(model, opt, range(6, steps), log=log)
    torch.cuda.synchronize()
    final = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    if variant == "plain":
        model2, opt2 = build(sd, msd)
        train(model2, opt2, range(6, steps), rebucket_at=9)
        torch.cuda.synchronize()
        final2 = torch.cat([p.detach().reshape(-1) for p in model2.parameters()])
        assert torch.equal(final2, final), f"resumed / re-bucketed run differs: max {(final2.float() - final.float()).abs().max().item()}"

    # the replay: fp32 masters and moments per parameter, fed the oracle model's gradient
    names = [n for n, _ in oracle.named_parameters()]
    wd = {id(p): g["weight_decay"] for g in _groups(oracle) for p in g["params"]}
    state = {n: (p.detach().float().cpu().reshape(-1), torch.zeros(p.numel())) for n, p in oracle.named_parameters()}
    ema = {n: w.clone() for n, (w, _) in state.items()}
    for it in range(steps):
        coef, scale, skipped = log[it]
        assert skipped == (it == overflow), (it, skipped)
        total = {}
        for k in range(K):
            for p in oracle.parameters():
                p.grad = None
            (loss_of(oracle, it, k) * scale).backward()
            for n, p in oracle.named_parameters():
                g = p.grad.float().reshape(-1)
                if world > 1:
                    dist.all_reduce(g)
                    g = torch.mul(g, torch.tensor(1.0 / world, dtype=torch.float32, device=dev))
                total[n] = torch.add(total[n], g.cpu()) if k else g.cpu()
        if skipped:
            continue
        for n, p in oracle.named_parameters():
            w, m = state[n]
            lion_reference_step_(w, m, total[n], _lr_at(it), BETAS, wd[id(p)], coef)
            if variant == "ema":
                ema[n].add_(torch.mul(torch.sub(w, ema[n]), torch.tensor(1.0 - 0.8, dtype=torch.float32)))
            with torch.no_grad():
                p.copy_(w.reshape(p.shape).to(dtype))
    want = torch.cat([p.detach().reshape(-1) for p in oracle.parameters()])
    if world <= 2:   # two ranks add their two gradients in either order: the same fp32 sum
        assert torch.equal(final, want), f"{variant}: max {(final.float() - want.float()).abs().max().item()}"
    else:   # the kernels add the ranks' gradients in another order (in the switch with multimem): u may cross 0 elsewhere
        diff = (final.float() - want.float()).abs()
        assert float(diff.max()) <= 2 * sum(_lr_at(it) for it in range(steps)) + 1e-2 and float((diff > 1e-2).double().mean()) < 0.01
    if variant == "ema":
        got = list(opt.ema_state_dict().values())
        assert len(got) == len(names)
        for n, e in zip(names, got):
            assert torch.equal(e.reshape(-1), ema[n]), n
    if variant == "plain" and world == 1:   # FusedLion without bagua, fed the same batches
        flat = copy.deepcopy(base)
        fo = FusedLion(_groups(flat), lr=_lr_at(0), betas=BETAS)
        for it in range(steps):
            for g in fo.param_groups:
                g["lr"] = _lr_at(it)
            fo.zero_grad()
            loss_of(flat, it, 0).backward()
            fo.step()
        assert torch.equal(torch.cat([p.detach().reshape(-1) for p in flat.parameters()]), final), "FusedLion differs"
    return final.cpu()


VARIANTS = ["plain", "clip", "accumulate", "ema", "scaled"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_self_peer_lion_training_is_the_replay(variant):
    run_distributed(_lion_train_worker, world=1, args=(variant,), use_cuda=True, extra_env={"BAGUA_SELF_PEER": "1"}, timeout=300)


@pytest.mark.multigpu
@pytest.mark.parametrize("variant", ["plain", "clip"])
def test_lion_training_on_real_peers(variant):
    n = min(torch.cuda.device_count(), 8)
    if n < 2:
        pytest.skip("needs 2 or more GPUs")
    res = run_distributed(_lion_train_worker, world=n, args=(variant,), use_cuda=True, timeout=300)
    for r in res[1:]:
        assert torch.equal(r, res[0]), "every rank must hold the same weights"
