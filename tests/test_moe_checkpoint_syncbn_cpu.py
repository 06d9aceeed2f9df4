"""MoE gating/dispatch (index form vs the reference's dense one-hot formulation), expert-parallel training on gloo,
MoE-aware checkpoints, and SyncBatchNorm against single-process BatchNorm over the concatenated batch."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from tests.mp_utils import run_distributed


def _dense_reference(tokens, gate, E, C):
    """The reference's formulation (sharded_moe.py:352-374) from dense combine weights."""
    cw, mask = gate.dense()
    dispatched = torch.einsum("sec,sm->ecm", mask.type_as(tokens), tokens)
    return cw, mask, dispatched


@pytest.mark.parametrize("k", [1, 2])
def test_index_gating_matches_dense_formulation(k):
    from bagua_b200.ops import moe as moe_ops
    from bagua_b200.parallel.moe.sharded_moe import top1gating_indices, top2gating_indices

    torch.manual_seed(0)
    S, E, M = 64, 4, 8
    logits = torch.randn(S, E)
    tokens = torch.randn(S, M, requires_grad=True)
    g = top1gating_indices(logits, 1.0, 4) if k == 1 else top2gating_indices(logits, 1.0)
    C = g.capacity
    assert C == (math.ceil(S / E) if k == 1 else math.ceil(2 * S / E))
    # every (expert, slot) pair is used at most once and slots are < capacity
    flat = (g.expert_idx * C + g.slot_idx)[g.slot_idx >= 0]
    assert flat.unique().numel() == flat.numel() and int(g.slot_idx.max()) < C
    cw, mask, dispatched_ref = _dense_reference(tokens.detach(), g, E, C)
    disp = moe_ops.dispatch(tokens, g.expert_idx, g.slot_idx, E, C, None, 1, E).reshape(E, C, M)
    torch.testing.assert_close(disp, dispatched_ref)
    expert_out = torch.randn(1, E, C, M, requires_grad=True)
    w = g.weights.clone().requires_grad_(True)
    comb = moe_ops.combine(expert_out, g.expert_idx, g.slot_idx, w, E, C, None, 1, E)
    comb_ref = torch.einsum("sec,ecm->sm", cw, expert_out.detach().reshape(E, C, M))
    torch.testing.assert_close(comb, comb_ref, rtol=1e-5, atol=1e-6)
    # gradients of the row scatter/gather equal autograd through the dense einsums
    (disp.sum() + comb.pow(2).sum()).backward()
    t2 = tokens.detach().clone().requires_grad_(True)
    e2 = expert_out.detach().clone().requires_grad_(True)
    cw2 = cw.clone().requires_grad_(True)
    ref = torch.einsum("sec,sm->ecm", mask.float(), t2).sum() + torch.einsum("sec,ecm->sm", cw2, e2.reshape(E, C, M)).pow(2).sum()
    ref.backward()
    torch.testing.assert_close(tokens.grad, t2.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(expert_out.grad, e2.grad, rtol=1e-5, atol=1e-6)
    gw_ref = torch.stack([cw2.grad[torch.arange(S), g.expert_idx[:, j], g.slot_idx[:, j].clamp(min=0)] * (g.slot_idx[:, j] >= 0) for j in range(k)], dim=1)
    torch.testing.assert_close(w.grad, gw_ref, rtol=1e-5, atol=1e-6)
    # l_aux and exp_counts as defined by the reference
    gates = F.softmax(logits, dim=1)
    mask1 = F.one_hot(gates.argmax(1), E)
    assert torch.equal(g.exp_counts, mask1.sum(0))
    l_ref = (gates.mean(0) * mask1.float().mean(0)).sum() * E if k == 1 else (gates.mean(0) * mask1.float().mean(0)).mean() * E * E
    torch.testing.assert_close(g.l_aux, l_ref)


def test_top1_capacity_overflow_drops_tokens():
    from bagua_b200.parallel.moe.sharded_moe import top1gating_indices

    logits = torch.zeros(32, 4)
    logits[:, 0] = 10.0  # everybody wants expert 0
    g = top1gating_indices(logits, 1.0, 4)
    kept = (g.slot_idx >= 0).sum().item()
    assert kept == g.capacity == 8 and (g.weights[g.slot_idx < 0] == 0).all()


def _moe_worker(rank, world, ckpt_dir):
    import torch.distributed as dist
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.checkpoint import load_checkpoint, save_checkpoint
    from bagua_b200.parallel.algorithms import gradient_allreduce
    from bagua_b200.parallel.moe import MoE

    bagua.init_process_group()

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.inp = nn.Linear(16, 32)
            self.moe = MoE(32, nn.Linear(32, 32), num_local_experts=2, k=2)
            self.out = nn.Linear(32, 4)

        def forward(self, x):
            h, l_aux, counts = self.moe(F.relu(self.inp(x)))
            return self.out(h), l_aux, counts

    torch.manual_seed(100 + rank)  # experts start different per rank; shared weights are broadcast by with_bagua
    model = Net()
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    model = model.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    names = {n for n, _ in model.bagua_ddp.bagua_build_params()}
    assert not any("bagua_experts" in n for n in names) and "moe.bagua_moe.gate.wg.weight" in names
    for it in range(4):
        g = torch.Generator().manual_seed(rank * 10 + it)
        x, y = torch.randn(16, 16, generator=g), torch.randint(0, 4, (16,), generator=g)
        opt.zero_grad()
        out, l_aux, counts = model(x)
        (F.cross_entropy(out, y) + 0.01 * l_aux).backward()
        opt.step()
        assert counts.device.type == "cpu" and counts.numel() == 2 * world
    shared = torch.cat([p.detach().reshape(-1) for n, p in model.named_parameters() if "bagua_experts" not in n])
    expert = torch.cat([p.detach().reshape(-1) for n, p in model.named_parameters() if "bagua_experts" in n])
    save_checkpoint(7, ckpt_dir, model, opt)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        for p in model.parameters():
            p.add_(1.0)
    it = load_checkpoint(ckpt_dir, model, opt)
    after = model.state_dict()
    assert it == 7 and all(torch.equal(before[k], after[k]) for k in before)
    files = sorted(os.listdir(os.path.join(ckpt_dir, "iter_0000007"))) if rank == 0 else []
    return shared, expert, files


def test_moe_training_and_checkpoint(tmp_path):
    res = run_distributed(_moe_worker, world=2, args=(str(tmp_path),), timeout=300)
    assert torch.equal(res[0][0], res[1][0])          # non-expert parameters are data-parallel → identical
    assert not torch.equal(res[0][1], res[1][1])      # experts are local to their rank
    files = res[0][2]
    assert "mp_rank_00_model_states.pt" in files
    assert {f"expert_{i}_mp_rank_00_model_states.pt" for i in range(4)} <= set(files)
    assert {f"expert_parallel_rank_{r}_mp_rank_00_optim_states.pt" for r in range(2)} <= set(files)
    assert open(tmp_path / "latest_checkpointed_iteration.txt").read().strip() == "7"


def test_plain_checkpoint_roundtrip(tmp_path):
    from bagua_b200.checkpoint import load_checkpoint, save_checkpoint

    m = torch.nn.Linear(4, 4)
    opt = torch.optim.Adam(m.parameters())
    m(torch.randn(2, 4)).sum().backward()
    opt.step()
    sched = torch.optim.lr_scheduler.StepLR(opt, 1)
    assert load_checkpoint(str(tmp_path), m) == 0  # nothing there yet
    save_checkpoint(3, str(tmp_path), m, opt, sched)
    m2 = torch.nn.Linear(4, 4)
    opt2 = torch.optim.Adam(m2.parameters())
    assert load_checkpoint(str(tmp_path), m2, opt2, torch.optim.lr_scheduler.StepLR(opt2, 1)) == 3
    assert torch.equal(m.weight, m2.weight) and len(opt2.state_dict()["state"]) == 2


def _syncbn_worker(rank, world):
    import bagua_b200 as bagua
    from bagua_b200.contrib.sync_batchnorm import SyncBatchNorm

    bagua.init_process_group()
    torch.manual_seed(0)
    full = torch.randn(4 * world, 3, 5, 5)
    ref_bn = torch.nn.BatchNorm2d(3)
    net = torch.nn.Sequential(torch.nn.BatchNorm2d(3))
    net = SyncBatchNorm.convert_sync_batchnorm(net)
    assert isinstance(net[0], SyncBatchNorm)
    x = full[4 * rank : 4 * rank + 4].clone().requires_grad_(True)
    xf = full.clone().requires_grad_(True)
    y = net(x)
    yf = ref_bn(xf)
    w = torch.linspace(0.5, 1.5, y.numel() * world).view(4 * world, 3, 5, 5)
    (y * w[4 * rank : 4 * rank + 4]).sum().backward()
    (yf * w).sum().backward()
    torch.testing.assert_close(y, yf[4 * rank : 4 * rank + 4], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(x.grad, xf.grad[4 * rank : 4 * rank + 4], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(net[0].running_mean, ref_bn.running_mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(net[0].running_var, ref_bn.running_var, rtol=1e-4, atol=1e-5)
    net.eval()
    assert torch.isfinite(net(x.detach())).all()
    return True


def test_sync_batchnorm_equals_global_batchnorm():
    assert all(run_distributed(_syncbn_worker, world=2))


def _bf16_moe_worker(rank, world):
    """Regression: a bf16 model whose MoE gate must stay fp32 trains under with_bagua (casting the gate inside ``forward`` used to
    re-create the parameter and break the engine's 'backend tensor == parameter grad' contract)."""
    import bagua_b200 as bagua
    from bagua_b200 import models
    from bagua_b200.parallel.algorithms import gradient_allreduce

    bagua.init_process_group()
    torch.manual_seed(0)
    cfg = models.GPT2MoEConfig(vocab_size=128, n_positions=16, n_embd=32, n_layer=2, n_head=2, num_experts=2 * world)
    model = models.GPT2MoE(cfg, world_size=world).to(torch.bfloat16)
    gate_dtypes = {p.dtype for n, p in model.named_parameters() if n.endswith("wg.weight")}
    assert gate_dtypes == {torch.float32}
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    model = model.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    idx = torch.randint(0, 128, (2, 16), generator=torch.Generator().manual_seed(rank))
    for _ in range(3):
        opt.zero_grad()
        loss, _ = model(idx, idx)
        loss.backward()
        opt.step()
    gate = [p for n, p in model.named_parameters() if n.endswith("wg.weight")][0]
    return float(loss), gate.detach().clone()


def test_bf16_model_with_fp32_gate_trains_under_with_bagua():
    res = run_distributed(_bf16_moe_worker, world=2, timeout=240)
    assert all(l == l for l, _ in res)                                  # finite
    assert torch.equal(res[0][1], res[1][1])                            # the gate is data-parallel: identical on both ranks


def test_sharded_fused_optimizer_state_is_world_size_independent():
    """In-bucket fused SGD / Adam keep fp32 master weights and moments in 1/N shards next to the buckets.  ``state_dict()``
    consolidates them per parameter name (all-gather), ``load_state_dict()`` re-shards for the current layout: saved from 2
    ranks with one bucket, restored into 3 ranks with two buckets, every shard equals the slice of the same flat vectors.  The
    collective is replaced by a local concatenation; channels_last parameters keep their logical order in the checkpoint."""
    from bagua_b200.parallel.algorithms.gradient_allreduce import make_sharded_fused_adam, make_sharded_fused_sgd
    from bagua_b200.tensor import dense_strides

    torch.manual_seed(1)
    params = {"conv.weight": torch.randn(4, 3, 2, 2).to(memory_format=torch.channels_last), "conv.bias": torch.randn(4), "fc.weight": torch.randn(6, 8)}
    per = 4  # fp32 buckets: 16 bytes = 4 elements

    class Op:
        def __init__(self):
            self.s = 0

        def steps(self):
            return self.s

        def set_steps(self, s):
            self.s = s

        def set_hyper(self, *a):
            self.hyper = a

    def build(world, bucket_names, factory, n_state):
        """``world`` optimizers (one per rank) with shard records for the given bucketing; state filled from per-name truth."""
        ranks = [factory([torch.nn.Parameter(torch.zeros(1))], lr=0.1) for _ in range(world)]
        truth, recs = {}, [[] for _ in range(world)]
        for bi, names in enumerate(bucket_names):
            layout, off = [], 0
            for n in names:
                t = params[n]
                layout.append((n, off, t.numel(), tuple(t.shape), tuple(dense_strides(t))))
                off += t.numel()
            numel = (off + per - 1) // per * per
            vpr = (numel // per + world - 1) // world
            length = vpr * per
            for r in range(world):
                lo, hi = r * length, min((r + 1) * length, numel)
                state = tuple(torch.zeros(length) for _ in range(n_state))
                recs[r].append({"bucket": str(bi), "group": None, "numel": numel, "lo": lo, "hi": max(lo, hi), "layout": layout, "state": state,
                                "step_ops": (Op(),), "weights": torch.zeros(numel)})
        for r, opt in enumerate(ranks):
            opt._bucketing.hyper_ops = [(rec["step_ops"][0], 0) for rec in recs[r]]
            for rec in recs[r]:
                opt._register_shard(rec)
            # all-gather double: the same record of every rank, in rank order
            opt._gather = lambda t, group, r=r: [other_rec["state"][idx] for other_rec, idx in _locate(t, recs)]
        return ranks, recs

    def _locate(t, recs):
        for r, rr in enumerate(recs):
            for bi, rec in enumerate(rr):
                for idx, st in enumerate(rec["state"]):
                    if st is t:
                        return [(recs[q][bi], idx) for q in range(len(recs))]
        raise AssertionError("tensor is not a registered shard")

    for factory, keys in ((make_sharded_fused_sgd, ("master", "momentum_buffer")), (make_sharded_fused_adam, ("master", "exp_avg", "exp_avg_sq"))):
        src, src_recs = build(2, [["conv.weight", "conv.bias", "fc.weight"]], factory, len(keys))
        from bagua_b200.parallel.algorithms.gradient_allreduce import shard_of

        truth = {k: {n: torch.randn_like(params[n].contiguous()) for n in params} for k in keys}
        for r in range(2):
            for rec in src_recs[r]:
                for k, t in zip(keys, rec["state"]):
                    t.copy_(shard_of(truth[k], rec["layout"], rec["numel"], rec["lo"], rec["hi"], t.numel()))
                rec["step_ops"][0].set_steps(17)
        sds = [o.state_dict() for o in src]
        assert src[0].collective_state_dict and sds[0]["steps"] == 17 and sds[0]["param_groups"][0]["lr"] == 0.1
        for n in params:
            for k in keys:
                assert torch.equal(sds[0]["state"][n][k], truth[k][n]) and torch.equal(sds[1]["state"][n][k], truth[k][n])
        dst, dst_recs = build(3, [["fc.weight"], ["conv.bias", "conv.weight"]], factory, len(keys))
        sds[0]["param_groups"][0]["lr"] = 0.025
        for r, o in enumerate(dst):
            o.load_state_dict(sds[0])
            assert o.param_groups[0]["lr"] == 0.025
            for rec in dst_recs[r]:
                assert rec["step_ops"][0].steps() == 17
                for k, t in zip(keys, rec["state"]):
                    assert torch.equal(t, shard_of(truth[k], rec["layout"], rec["numel"], rec["lo"], rec["hi"], t.numel()))
        again = dst[1].state_dict()
        for n in params:
            for k in keys:
                assert torch.equal(again["state"][n][k], truth[k][n])
        # a state loaded before with_bagua() is kept and applied bucket by bucket when the algorithm builds the ops
        late = factory([torch.nn.Parameter(torch.zeros(1))], lr=0.1)
        late.load_state_dict(sds[0])
        assert not late.collective_state_dict and late.param_groups[0]["lr"] == 0.025
        _, fresh = build(3, [["fc.weight"], ["conv.bias", "conv.weight"]], factory, len(keys))
        for rec in fresh[2]:
            late._register_shard(rec)
            for k, t in zip(keys, rec["state"]):
                assert torch.equal(t, shard_of(truth[k], rec["layout"], rec["numel"], rec["lo"], rec["hi"], t.numel())) and rec["step_ops"][0].steps() == 17
