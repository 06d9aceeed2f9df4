"""The float64 optimizer oracle of tests/optim_oracle.py: an fp32 emulation of the kernels' update stays inside its bound, and every
deliberately broken update leaves it — so the GPU tests that use the bound would notice each of those mistakes in a kernel."""
import pytest
import torch

from tests import optim_oracle as oracle

N = 4096


def _inputs(seed):
    gen = torch.Generator().manual_seed(seed)
    w = torch.randn(N, generator=gen) * oracle.wide(N, gen, -3, 1, zeros=0.0, positive=True)
    g = oracle.wide(N, gen)
    m = oracle.wide(N, gen, -6, 2)
    v = oracle.wide(N, gen, -20, 3, zeros=0.2, positive=True)  # zero second moments: denominator = eps
    return w, g, m, v


def _f(x):
    return torch.tensor(x, dtype=torch.float32)


def _sgd_f32(w, g, m, hp):
    """csrc/multi_tensor.cu sgd_update in fp32 arithmetic, one rounding per operation."""
    lr, mu, damp, wd, s = map(_f, (hp.lr, hp.momentum, hp.dampening, hp.weight_decay, hp.grad_scale))
    d = g * s + wd * w
    if mu != 0:
        m = d if hp.first_step else mu * m + (1 - damp) * d
        d = d + mu * m if hp.nesterov else m
    return w - lr * d, m


def _adam_f32(w, g, m, v, hp):
    lr, b1, b2, eps, wd, s = map(_f, (hp.lr, hp.betas[0], hp.betas[1], hp.eps, hp.weight_decay, hp.grad_scale))
    bc1, bc2 = 1 - b1 ** hp.step, 1 - b2 ** hp.step  # fp32 pow: not the host's powf, within an ulp of it
    g = g * s
    if hp.adamw:
        w = w * (1 - lr * wd)
    else:
        g = g + wd * w
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    return w - (lr / bc1) * (m / (torch.sqrt(v) / torch.sqrt(bc2) + eps)), m, v


SGD_CASES = [
    oracle.Sgd(lr=0.1),
    oracle.Sgd(lr=0.1, momentum=0.9, first_step=True),
    oracle.Sgd(lr=0.05, momentum=0.9, dampening=0.1, weight_decay=1e-4),
    oracle.Sgd(lr=0.05, momentum=0.9, nesterov=True, weight_decay=0.1, grad_scale=2.0 ** -16),
]
ADAM_CASES = [oracle.Adam(lr=1e-3, step=t, adamw=aw, weight_decay=0.1, grad_scale=gs) for t in (1, 2, 10, 10 ** 4) for aw in (False, True)
              for gs in (1.0, 2.0 ** -16)]


@pytest.mark.parametrize("hp", SGD_CASES)
def test_fp32_sgd_update_is_inside_the_bound(hp):
    for seed in range(3):
        w, g, m, _ = _inputs(seed)
        wn, mn = _sgd_f32(w, g, m, hp)
        ow, om, tw, tm = oracle.sgd(w, g, m, hp)
        assert oracle.excess(wn, ow, tw) <= 1.0
        if om is not None:
            assert oracle.excess(mn, om, tm) <= 1.0


@pytest.mark.parametrize("hp", ADAM_CASES)
def test_fp32_adam_update_is_inside_the_bound(hp):
    for seed in range(3):
        w, g, m, v = _inputs(seed)
        wn, mn, vn = _adam_f32(w, g, m, v, hp)
        ow, om, ov, tw, tm, tv = oracle.adam(w, g, m, v, hp)
        assert oracle.excess(wn, ow, tw) <= 1.0
        assert oracle.excess(mn, om, tm) <= 1.0
        assert oracle.excess(vn, ov, tv) <= 1.0


# inputs chosen so that the variant matters: momentum and decay on, a scaled gradient, a later step
SGD_BROKEN = {
    "dampening_on_first_step": oracle.Sgd(lr=0.1, momentum=0.9, dampening=0.1, first_step=True),
    "nesterov_with_old_momentum": oracle.Sgd(lr=0.1, momentum=0.9, nesterov=True),
    "no_grad_scale": oracle.Sgd(lr=0.1, momentum=0.9, grad_scale=2.0 ** -16),
    "weight_decay_after_momentum": oracle.Sgd(lr=0.1, momentum=0.9, weight_decay=1e-4),
}
ADAM_BROKEN = {
    "eps_inside_sqrt": oracle.Adam(lr=1e-3, step=10),
    "bias_correction_of_previous_step": oracle.Adam(lr=1e-3, step=10),
    "l2_decay_in_adamw": oracle.Adam(lr=1e-3, step=10, adamw=True, weight_decay=1e-2),
    "no_grad_scale": oracle.Adam(lr=1e-3, step=10, grad_scale=2.0 ** -16),
}


def test_the_broken_variants_are_the_listed_ones():
    assert set(SGD_BROKEN) == set(oracle.SGD_VARIANTS) and set(ADAM_BROKEN) == set(oracle.ADAM_VARIANTS)


@pytest.mark.parametrize("variant", oracle.SGD_VARIANTS)
def test_every_broken_sgd_update_leaves_the_bound(variant):
    hp = SGD_BROKEN[variant]
    w, g, m, _ = _inputs(7)
    ow, om, tw, tm = oracle.sgd(w, g, m, hp)
    bw, bm, _, _ = oracle.sgd(w, g, m, hp, variant=variant)
    # what a kernel with this mistake would store: its fp32 result
    worst = max(oracle.excess(bw.float(), ow, tw), oracle.excess(bm.float(), om, tm))
    assert worst > 1.0, (variant, worst)


@pytest.mark.parametrize("variant", oracle.ADAM_VARIANTS)
def test_every_broken_adam_update_leaves_the_bound(variant):
    hp = ADAM_BROKEN[variant]
    w, g, m, v = _inputs(8)
    ow, om, ov, tw, tm, tv = oracle.adam(w, g, m, v, hp)
    bw, bm, bv, _, _, _ = oracle.adam(w, g, m, v, hp, variant=variant)
    worst = max(oracle.excess(bw.float(), ow, tw), oracle.excess(bm.float(), om, tm), oracle.excess(bv.float(), ov, tv))
    assert worst > 1.0, (variant, worst)


def test_half_ulp_of_the_low_precision_dtypes():
    x = torch.tensor([1.0, 1.5, 2.0 ** -130, 3e-8, 1000.0], dtype=torch.float64)
    assert oracle.half_ulp(x, torch.bfloat16).tolist() == [2.0 ** -8, 2.0 ** -8, 2.0 ** -134, 2.0 ** -33, 2.0]
    assert oracle.half_ulp(x, torch.float16).tolist() == [2.0 ** -11, 2.0 ** -11, 2.0 ** -25, 2.0 ** -25, 2.0 ** -2]
    assert oracle.half_ulp(x, torch.float32).tolist() == [0.0] * 5
