"""The LAMB float64 oracle (``tests/lamb_oracle.py``) on the CPU: an fp32 emulation of the kernels' arithmetic stays inside its
bound, and each deliberately wrong update leaves it."""
import pytest
import torch

from tests import lamb_oracle as lo
from tests.optim_oracle import excess


def _bucket(seed, sizes=(1, 3, 7, 300, 4099)):
    gen = torch.Generator().manual_seed(seed)
    params = []
    for n in sizes:
        w = torch.randn(n, generator=gen)
        g = torch.randn(n, generator=gen) * 0.3
        m1 = torch.randn(n, generator=gen) * 0.05
        m2 = torch.rand(n, generator=gen) * 0.01
        params.append((w, g, m1, m2))
    params.append((torch.zeros(64), torch.randn(64, generator=gen), torch.zeros(64), torch.zeros(64)))   # all-zero weights: r = 1
    return params


def _worst(params, hp, variant=None):
    got = lo.emulate_fp32(params, hp)
    want = lo.lamb(params, hp, variant)
    worst = 0.0
    for (w, a, b), (w_n, a_n, b_n, r, tol_w, tol_a, tol_b) in zip(got, want):
        worst = max(worst, excess(w, w_n, tol_w), excess(a, a_n, tol_a), excess(b, b_n, tol_b))
    return worst


HP = dict(lr=2e-2, step=3, coef=0.37)


@pytest.mark.parametrize("wd", [0.01, 0.0])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_fp32_emulation_inside_bound(seed, wd):
    assert _worst(_bucket(seed), lo.Lamb(weight_decay=wd, **HP)) <= 1.0


def test_zero_parameter_gets_ratio_one():
    out = lo.lamb(_bucket(0), lo.Lamb(**HP))
    assert out[-1][3] == 1.0 and all(o[3] != 1.0 for o in out[:-1])


@pytest.mark.parametrize("variant", lo.VARIANTS)
def test_broken_variants_leave_bound(variant):
    wd = 0.0 if variant == "ratio_without_decay" else 0.01
    hp = lo.Lamb(weight_decay=wd, **HP)
    assert max(_worst(_bucket(s), hp, variant) for s in range(3)) > 1.0, variant
