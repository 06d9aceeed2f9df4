"""The Lion float64 oracle (``tests/lion_oracle.py``) on the CPU: the fp32 replay that ``FusedLion`` runs on CPU tensors stays inside
the per-element bound over a fixed gradient sequence, every emulated defect leaves it, and a NaN gradient element poisons its own
weight only."""
import pytest
import torch

from bagua_b200.ops.optim import FusedLion, lion_reference_step_
from tests.lion_oracle import VARIANTS, Lion, emulate_fp32, excess, oracle

STEPS = 12


def _sequence(seed, n=4096, nan_at=None):
    """A fixed gradient sequence with magnitudes over several decades, a block of exact zeros and, optionally, one NaN."""
    g = torch.Generator().manual_seed(seed)
    w0 = torch.randn(n, generator=g) * 0.05
    scales = torch.logspace(-4, 1, n, dtype=torch.float32)
    xs = []
    for k in range(STEPS):
        x = torch.randn(n, generator=g) * scales
        x[:64] = 0.0   # m stays 0 there: sign(u) = 0, the weight only decays
        if nan_at is not None and k == STEPS // 2:
            x[nan_at] = float("nan")
        xs.append(x)
    return w0, xs


def _hps(wd=0.1):
    return [Lion(lr=3e-3 if k < STEPS // 2 else 1e-3, betas=(0.9, 0.99), weight_decay=wd) for k in range(STEPS)]


def _replay(w0, xs, hps, coefs=None):
    w, m = w0.clone(), torch.zeros_like(w0)
    for k, (x, hp) in enumerate(zip(xs, hps)):
        coef = None if coefs is None else torch.tensor(coefs[k], dtype=torch.float32)
        lion_reference_step_(w, m, x, hp.lr, hp.betas, hp.weight_decay, coef)
    return w, m


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_fp32_replay_stays_inside_the_bound(seed):
    w0, xs = _sequence(seed)
    coefs = [1.0 if k % 3 else 0.37 for k in range(STEPS)]   # a clip coefficient on some steps
    hps = _hps()
    w, m = _replay(w0, xs, hps, coefs)
    ew, em = emulate_fp32(w0, torch.zeros_like(w0), xs, hps, coefs)
    assert torch.equal(w, ew) and torch.equal(m, em), "the optimizer's replay and the oracle's emulation must agree bit for bit"
    W, M, tw, tm = oracle(w0, torch.zeros_like(w0), xs, hps, coefs)
    assert excess(w, W, tw) <= 1.0 and excess(m, M, tm) <= 1.0
    assert torch.equal(w[:64], emulate_fp32(w0[:64], torch.zeros(64), [x[:64] for x in xs], hps, coefs)[0])
    # the bound is not loose: the 2·lr slack applies only where |u| is within the rounding error of u
    assert float((tw > 1e-5).double().mean()) < 0.05


@pytest.mark.parametrize("variant", VARIANTS)
def test_bound_catches_emulated_defects(variant):
    nan_at = 100 if variant == "sign_nan_zero" else None
    w0, xs = _sequence(7, nan_at=nan_at)
    hps = _hps()
    W, M, tw, tm = oracle(w0, torch.zeros_like(w0), xs, hps)
    w, m = emulate_fp32(w0, torch.zeros_like(w0), xs, hps, variant=variant)
    assert max(excess(w, W, tw), excess(m, M, tm)) > 1.0, variant


def test_nan_gradient_element_poisons_its_own_weight_only():
    w0, xs = _sequence(3, nan_at=200)
    hps = _hps()
    w, m = _replay(w0, xs, hps)
    assert torch.isnan(w[200]) and torch.isnan(m[200])
    rest = torch.ones_like(w, dtype=torch.bool)
    rest[200] = False
    assert not torch.isnan(w[rest]).any() and not torch.isnan(m[rest]).any()
    W, M, tw, tm = oracle(w0, torch.zeros_like(w0), xs, hps)
    assert excess(w, W, tw) <= 1.0 and excess(m, M, tm) <= 1.0


def test_fused_lion_on_cpu_is_the_replay():
    w0, xs = _sequence(5, n=300)
    p = torch.nn.Parameter(w0.clone().reshape(10, 30))
    opt = FusedLion([p], lr=2e-3, betas=(0.95, 0.98), weight_decay=0.05)
    for x in xs:
        p.grad = x.reshape(10, 30).clone()
        opt.step()
    w, m = emulate_fp32(w0, torch.zeros_like(w0), xs, Lion(lr=2e-3, betas=(0.95, 0.98), weight_decay=0.05))
    assert torch.equal(p.detach().reshape(-1), w) and torch.equal(opt.state[p]["exp_avg"].reshape(-1), m)


@pytest.mark.parametrize("kw", [dict(lr=-1e-4), dict(weight_decay=-0.1), dict(betas=(1.0, 0.99)), dict(betas=(0.9, -0.1))])
def test_fused_lion_rejects_invalid_hyperparameters(kw):
    with pytest.raises(ValueError):
        FusedLion([torch.nn.Parameter(torch.zeros(3))], **kw)
