"""The whole engine on the NVSwitch code path with ONE GPU: ``BAGUA_SELF_PEER=1`` builds the group's ``PeerEngine`` with this
GPU as its only peer, so ``with_bagua`` creates the very same native bucket programs as on 8 GPUs (fused
reduce-scatter→optimizer→all-gather, ByteGrad, peer average, low-precision ring, fused async average, MoE scatter/gather,
GEMM with the combine epilogue) and a world of one makes every result checkable against plain single-process training.

The workers are the multi-GPU ones of ``tests/test_peer_gpu.py`` (they run again, unchanged, on 2…8 real GPUs there); the
P = 2…8 arithmetic of the kernels themselves is covered on one GPU by ``tests/test_virtual_peer_gpu.py``.
"""
import copy

import pytest
import torch

from tests import test_peer_gpu as multi
from tests.mp_utils import run_distributed

pytestmark = pytest.mark.gpu

SELF = {"BAGUA_SELF_PEER": "1"}


def _run(fn, *args, env=None):
    e = dict(SELF)
    e.update(env or {})
    return run_distributed(fn, world=1, args=args, use_cuda=True, extra_env=e, timeout=300)


def test_self_peer_allreduce_variants_and_blocking_api():
    res = _run(multi._allreduce_worker)
    assert "multicast" in res[0]


def test_self_peer_bytegrad_kernel_vs_pipeline():
    _run(multi._bytegrad_worker)


@pytest.mark.parametrize("name", ["gradient_allreduce", "bytegrad", "decentralized", "decentralized_shift_one", "low_precision_decentralized", "qadam", "async"])
def test_self_peer_algorithms_run_native_ops(name):
    _run(_algorithm_vs_local_training, name)


def _algorithm_vs_local_training(rank, world, name):
    """Each algorithm family through ``with_bagua`` at world = 1 on the peer-kernel path; averaging with oneself is the identity,
    so the trained weights must match plain local training (quantised families: within the quantisation noise)."""
    import torch.nn as nn

    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms import Algorithm, q_adam

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    torch.manual_seed(3)
    base = nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 32)).to(dev)
    model, oracle = copy.deepcopy(base), copy.deepcopy(base)
    if name == "qadam":
        opt = q_adam.QAdamOptimizer(model.parameters(), lr=1e-3, warmup_steps=3)
        oopt = q_adam.QAdamOptimizer(oracle.parameters(), lr=1e-3, warmup_steps=3)
        algo = q_adam.QAdamAlgorithm(opt)
    else:
        opt = torch.optim.SGD(model.parameters(), lr=0.05)
        oopt = torch.optim.SGD(oracle.parameters(), lr=0.05)
        kw = {"sync_interval_ms": 5} if name == "async" else {}
        algo = Algorithm.init("decentralized", peer_selection_mode="shift_one") if name == "decentralized_shift_one" else Algorithm.init(name, **kw)
    model = model.with_bagua([opt], algo)
    kinds = set()
    for it in range(8):
        x = torch.randn(16, 64, device=dev, generator=torch.Generator(device=dev).manual_seed(it))
        opt.zero_grad()
        model(x).square().mean().backward()
        opt.step()
        if name == "qadam" and it >= 3:
            # the oracle's compressed stage: m = b1*m + (1-b1)*g on the host side of the test
            b1 = 0.9
            oopt.zero_grad()
            oracle(x).square().mean().backward()
            for p in oracle.parameters():
                oopt.state[p]["exp_avg"].mul_(b1).add_(p.grad, alpha=1 - b1)
            oopt.step()
        else:
            oopt.zero_grad()
            oracle(x).square().mean().backward()
            oopt.step()
        kinds |= {b.backend_bucket.print_ops() for b in model.bagua_buckets}
    if name == "async":
        import time

        time.sleep(0.1)   # let a few background rounds land
        rounds = model.bagua_buckets[0]._async_op.native_op.rounds()
        model.bagua_algorithm.abort(model)
        assert rounds >= 1, "the background loop must have launched the fused averaging kernel"
    torch.cuda.synchronize()
    expected = {
        "gradient_allreduce": "allreduce", "bytegrad": "bytegrad_fused", "decentralized": "allreduce", "decentralized_shift_one": "peer_average_shift_one",
        "low_precision_decentralized": "low_precision_ring_fused", "qadam": "qadam_momentum_bytegrad_fused", "async": "async_model_average_fused",
    }[name]
    assert any(expected in k for k in kinds), (name, kinds)
    assert not any("python" in k for k in kinds if name != "decentralized"), (name, kinds)   # no GIL-taking op in front of the kernels
    if name == "qadam":
        # compare the communicated quantity — the first moments — not the weights: Adam divides by sqrt(v) with v frozen after the
        # warm-up, so one quantisation level of noise in m moves weights with a tiny v by arbitrary amounts (inherent to QAdam)
        mine = torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in model.parameters()])
        want = torch.cat([oopt.state[p]["exp_avg"].reshape(-1) for p in oracle.parameters()])
        assert (mine - want).abs().max().item() <= 6 * (want.max() - want.min()).item() / 255, (mine - want).abs().max().item()
        return True
    mine = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    want = torch.cat([p.detach().reshape(-1) for p in oracle.parameters()])
    tol = {"bytegrad": 2e-2, "low_precision_decentralized": 2e-2}.get(name, 1e-5)
    assert (mine - want).abs().max().item() <= tol * max(1.0, want.abs().max().item()), (name, (mine - want).abs().max().item())
    eng = bagua.communication._get_default_group().peer_engine()
    assert eng is not None and eng.comm.error_code() == 0
    return True


def test_self_peer_fused_sgd_matches_torch_and_survives_rebucketing():
    _run(_fused_sgd_rebucket_worker)


def _fused_sgd_rebucket_worker(rank, world):
    """SGD(momentum, nesterov, weight decay) inside the bucket kernel vs torch.optim.SGD, with the buckets rebuilt in the middle of
    training (what the autotune service does every 100 steps): momentum, fp32 master weights and step count must carry over."""
    import bagua_b200 as bagua
    from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_sgd

    bagua.init_process_group()
    dev = torch.device("cuda", rank)
    for dtype in (torch.float32, torch.bfloat16):
        torch.manual_seed(9)
        base = torch.nn.Sequential(torch.nn.Linear(512, 1024), torch.nn.ReLU(), torch.nn.Linear(1024, 1024), torch.nn.ReLU(), torch.nn.Linear(1024, 64)).to(dev)
        oracle = copy.deepcopy(base)                       # fp32 oracle
        model = copy.deepcopy(base).to(dtype)
        opt = make_sharded_fused_sgd(model.parameters(), lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-4)
        oopt = torch.optim.SGD(oracle.parameters(), lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-4)
        model = model.with_bagua([opt], FusedGradientAllReduceAlgorithm(opt))
        assert all(b.allreduce_variant.startswith("fused_sgd") for b in model.bagua_buckets)
        for it in range(8):
            if it == 4:
                n_before = len(opt._bucketing.shards)
                model.bagua_ddp._reset_buckets()           # re-bucket mid-training
                assert len(opt._bucketing.shards) == n_before and len(opt._bucketing.hyper_ops) == n_before, "old shards must be dropped, not accumulated"
                assert opt._pending_state is None
            x = torch.randn(32, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(it))
            opt.zero_grad()
            model(x.to(dtype)).float().pow(2).mean().backward()
            opt.step()
            oopt.zero_grad()
            # the oracle sees the same (dtype-rounded) weights' gradients only approximately in bf16: compare masters loosely there
            oracle(x).pow(2).mean().backward()
            oopt.step()
        torch.cuda.synchronize()
        sd = opt.state_dict()
        assert sd["steps"] == 8
        mine = torch.cat([sd["state"][n]["master"].reshape(-1) for n, _ in model.named_parameters()]).to(dev)
        want = torch.cat([p.detach().reshape(-1) for p in oracle.parameters()])
        if dtype == torch.float32:
            torch.testing.assert_close(mine, want, rtol=1e-4, atol=1e-5)
        else:
            assert (mine - want).abs().max().item() < 5e-2
    return True


def test_self_peer_fused_adam_matches_adamw():
    _run(multi._fused_adam_worker)


def test_self_peer_sharded_optimizer_state_roundtrip():
    _run(multi._sharded_state_worker)


def test_self_peer_moe_dispatch_combine_vs_all_to_all():
    _run(multi._moe_worker)


def test_self_peer_moe_gemm_with_combine_epilogue():
    _run(multi._fused_combine_worker)


def test_self_peer_syncbn_cuda_path():
    _run(multi._syncbn_worker)


def test_self_peer_blocking_allgather_reduce_scatter():
    _run(multi._peer_collectives_worker)


def test_self_peer_graphed_step_with_bucket_kernels():
    _run(multi._graphed_step_worker)
