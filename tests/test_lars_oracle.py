"""The LARS float64 oracle (``tests/lars_oracle.py``) on the CPU.

* Its rule, chained over several steps at a constant learning rate, equals an independent formulation: apex
  ``LARC(clip=False, eps=0)`` around ``torch.optim.SGD(momentum)`` with the weight decay folded into the gradient (written out
  below); under a learning-rate change the two momentum forms part, and the check sees it.
* An fp32 emulation of the kernels' arithmetic stays inside its bound over a few steps with a changing ``lr``, two parameter
  groups and ``coef ≠ 1``, and each deliberately wrong update leaves it."""
import math

import pytest
import torch

from tests import lars_oracle as lo

# fp32 values, as the launchers receive them, so that both formulations use the same numbers
MU, WD, ETA, COEF = (lo.f32(x) for x in (0.9, 5e-4, 1e-3, 0.37))


def _params(seed, sizes=(3, 7, 300, 4099)):
    gen = torch.Generator().manual_seed(seed)
    ws = [torch.randn(n, generator=gen) for n in sizes]
    ws.append(torch.zeros(64))   # all-zero weights: trust 1
    return ws


def _grads(seed, ws, steps):
    gen = torch.Generator().manual_seed(1000 + seed)
    return [[torch.randn(w.numel(), generator=gen) * 0.3 for w in ws] for _ in range(steps)]


def _larc_sgd(ws, grads, lrs, wd_groups, coef):
    """apex LARC(clip=False, eps=0) wrapping torch.optim.SGD(momentum=MU) in float64: per parameter with weight decay, the
    gradient becomes ``trust·(g + wd·w)`` with ``trust = eta·‖w‖/(‖g‖ + wd·‖w‖)`` (when both norms are nonzero) and the inner
    SGD runs without weight decay. LARC adapts every parameter it sees; the MLPerf form exempts the weight_decay = 0 group, which
    is therefore stepped by the plain SGD (no LARC) here."""
    params = [torch.nn.Parameter(w.double().clone()) for w in ws]
    groups = [{"params": [params[i] for i in idx], "weight_decay": wd} for idx, wd in wd_groups]
    sgd = torch.optim.SGD(groups, lr=lrs[0], momentum=MU)
    index = {id(p): i for i, p in enumerate(params)}
    for step_grads, lr in zip(grads, lrs):
        for g in sgd.param_groups:
            g["lr"] = lr
        with torch.no_grad():
            for grp in sgd.param_groups:
                wd = grp["weight_decay"]
                for p in grp["params"]:
                    g = step_grads[index[id(p)]].double() * lo.f32(coef)
                    if wd != 0:
                        pn, gn = float(p.norm()), float(g.norm())
                        if pn != 0 and gn != 0:
                            adaptive = lo.f32(ETA) * pn / (gn + pn * lo.f32(wd))
                            g = (g + lo.f32(wd) * p) * adaptive
                    p.grad = g
            saved = [grp["weight_decay"] for grp in sgd.param_groups]
            for grp in sgd.param_groups:
                grp["weight_decay"] = 0
            sgd.step()
            for grp, wd in zip(sgd.param_groups, saved):
                grp["weight_decay"] = wd
    return [p.detach() for p in params]


# the oracle rounds trust and lr·trust to fp32 as the kernels do, LARC/SGD in float64 does not: a few 2^-24 of each step
RTOL, ATOL = 1e-9, 2e-9


def _oracle_chain(ws, grads, lrs, wd_groups, coef, variant=None):
    w = [x.double() for x in ws]
    v = [torch.zeros_like(x) for x in w]
    prev = None
    for step_grads, lr in zip(grads, lrs):
        for idx, wd in wd_groups:
            hp = lo.Lars(lr=lr, momentum=MU, weight_decay=wd, trust_coefficient=ETA, coef=coef, prev_lr=prev)
            res = lo.lars([(w[i], step_grads[i], v[i]) for i in idx], hp, variant)
            for i, (wn, vn, *_) in zip(idx, res):
                w[i], v[i] = wn, vn
        prev = lr
    return w


GROUPS = [([0, 2, 3, 4], WD), ([1], 0.0)]


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_equals_larc_sgd_at_constant_lr(seed):
    ws = _params(seed)
    grads = _grads(seed, ws, 4)
    lrs = [lo.f32(0.8)] * 4
    got = _oracle_chain(ws, grads, lrs, GROUPS, COEF)
    want = _larc_sgd(ws, grads, lrs, GROUPS, COEF)
    for a, b in zip(got, want):
        torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL)


def test_lr_change_tells_the_momentum_forms_apart():
    ws = _params(0)
    grads = _grads(0, ws, 4)
    lrs = [lo.f32(x) for x in (0.8, 0.8, 0.2, 0.1)]
    got = _oracle_chain(ws, grads, lrs, GROUPS, COEF)
    want = _larc_sgd(ws, grads, lrs, GROUPS, COEF)
    assert max(float((a - b).abs().max()) for a, b in zip(got, want)) > 1e-6
    # the torch form of the oracle is the LARC/SGD trajectory
    torch_form = _oracle_chain(ws, grads, lrs, GROUPS, COEF, "torch_momentum")
    for a, b in zip(torch_form, want):
        torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL)


def _states(seed, steps=4):
    """Kernel-side states of a few fp32-emulated steps: for each step, per group, the ``(w, g, v)`` before it and its hp."""
    ws = [w.float() for w in _params(seed)]
    vs = [torch.zeros_like(w) for w in ws]
    grads = _grads(seed, ws, steps)
    lrs = [0.8, 0.8, 0.3, 0.1][:steps]
    out, prev = [], None
    for step_grads, lr in zip(grads, lrs):
        for idx, wd in GROUPS:
            hp = lo.Lars(lr=lr, momentum=MU, weight_decay=wd, trust_coefficient=ETA, coef=COEF, prev_lr=prev)
            params = [(ws[i], step_grads[i], vs[i]) for i in idx]
            out.append((params, hp))
            for i, (wn, vn, _) in zip(idx, lo.emulate_fp32(params, hp)):
                ws[i], vs[i] = wn, vn
        prev = lr
    return out


def _worst(states, variant=None):
    worst = 0.0
    for params, hp in states:
        for (w, v, tr), (w_n, v_n, tr_n, tol_w, tol_v) in zip(lo.emulate_fp32(params, hp), lo.lars(params, hp, variant)):
            worst = max(worst, lo.excess(w, w_n, tol_w), lo.excess(v, v_n, tol_v))
    return worst


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_fp32_emulation_inside_bound(seed):
    assert _worst(_states(seed)) <= 1.0


def test_trust_rules():
    hp = lo.Lars(lr=0.1, weight_decay=1e-4, trust_coefficient=1e-3)
    assert lo.trust(4.0, 9.0, hp) == lo.f32(1e-3 * 2.0 / (3.0 + lo.f32(1e-4) * 2.0))
    assert lo.trust(0.0, 9.0, hp) == 1.0 and lo.trust(4.0, 0.0, hp) == 1.0
    assert math.isnan(lo.trust(float("nan"), 9.0, hp)) and math.isnan(lo.trust(4.0, float("nan"), hp))
    assert lo.trust(4.0, float("inf"), hp) == 0.0
    assert lo.trust(4.0, 9.0, lo.Lars(lr=0.1, weight_decay=0.0)) == 1.0


def test_nan_sum_gives_nan_weights_for_the_whole_parameter():
    w, g, v = torch.randn(100), torch.randn(100), torch.zeros(100)
    g[7] = float("nan")
    (w_n, v_n, tr, _, _), = lo.lars([(w, g, v)], lo.Lars(lr=0.1))
    assert math.isnan(tr) and bool(torch.isnan(w_n).all())


@pytest.mark.parametrize("variant", lo.VARIANTS)
def test_broken_variants_leave_bound(variant):
    states = _states(0)
    if variant == "nan_trust_one":   # a NaN gradient element: the whole parameter must turn NaN, not just that element
        params, hp = states[0]
        (w, g, v), *rest = params
        g = g.clone()
        g[1] = float("nan")
        states = [([(w, g, v)] + rest, hp)]
    assert _worst(states, variant) > 1.0, variant
