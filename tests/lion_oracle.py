"""Float64 oracle of a sequence of Lion steps (``csrc/lion.cuh``) with a per-element error bound, in the style of ``lars_oracle.py``.

The rule, with the constants as the launchers receive them (each worked out in double and rounded to fp32 once)::

    g = coef·x;  u = b1·m + c1·g;  w ← w·d − lr·sign(u);  m ← b2·m + c2·g
    b1 = f32(β1), c1 = f32(1 − β1), b2 = f32(β2), c2 = f32(1 − β2), lr = f32(lr), d = f32(1 − lr·wd)

``sign`` is +1 / −1, 0 for ±0 and NaN for NaN. The oracle follows one element through the whole gradient sequence in float64.
The momentum does not depend on the sign decisions, so its error stays a sum of fp32 rounding terms: ``e_m ← b2·e_m +
C·2^-24·(b2·|m| + c2·|g|)``, and ``u`` inherits ``b1·e_m`` plus its own roundings. The weight carries ``d·e_w`` plus the roundings of
``w·d − lr·s``, plus ``2·lr`` at every step where ``|u|`` lies within the error of ``u`` (the fp32 sign may differ there). So the bound
stays per element and tight everywhere else. ``variant`` selects a deliberately wrong update; ``tests/test_lion_oracle.py`` shows
that each of them leaves the bound.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from tests.lars_oracle import excess  # noqa: F401  (NaN-aware: a NaN on one side only is an infinite excess)
from tests.optim_oracle import FLOOR, U32, C

VARIANTS = ("momentum_before_interpolation", "betas_swapped", "coupled_weight_decay", "sign_nan_zero")


@dataclass
class Lion:
    lr: float = 1e-4
    betas: tuple = (0.9, 0.99)
    weight_decay: float = 0.0


def constants(hp: Lion):
    """``(lr, b1, c1, b2, c2, d)`` as Python floats holding the fp32 values the kernels use."""
    b1, b2, lr, wd = float(hp.betas[0]), float(hp.betas[1]), float(hp.lr), float(hp.weight_decay)
    return tuple(float(torch.tensor(v, dtype=torch.float32)) for v in (lr, b1, 1.0 - b1, b2, 1.0 - b2, 1.0 - lr * wd))


def _sign(u: torch.Tensor, nan_zero: bool = False) -> torch.Tensor:
    s = torch.sign(u)   # torch's sign maps NaN to 0
    return s if nan_zero else torch.where(torch.isnan(u), u, s)


def _steps(hps, n):
    return list(hps) if isinstance(hps, (list, tuple)) else [hps] * n


def oracle(w0, m0, xs, hps, coefs=None):
    """Float64 trajectory of ``len(xs)`` Lion steps from fp32 ``w0`` / ``m0`` over the gradients ``xs`` (as the kernel reads them)
    with the per-step coefficients ``coefs`` (default 1). ``hps``: one :class:`Lion` or one per step (an lr schedule). Returns
    ``(w, m, tol_w, tol_m)`` in float64."""
    w, m = w0.detach().double().clone(), m0.detach().double().clone()
    ew, em = torch.zeros_like(w), torch.zeros_like(m)
    seen = torch.zeros_like(w, dtype=torch.bool)   # only exact zeros so far: m and u are exact zeros in fp32 too
    for k, (x, hp) in enumerate(zip(xs, _steps(hps, len(xs)))):
        lr, b1, c1, b2, c2, d = constants(hp)
        coef = 1.0 if coefs is None else float(torch.tensor(coefs[k], dtype=torch.float32))
        g = x.detach().double() * coef
        u = b1 * m + c1 * g
        eu = b1 * em + C * U32 * (b1 * m.abs() + c1 * g.abs()) + FLOOR
        seen |= g != 0
        flip = seen & (u.abs() <= eu)
        s = _sign(u)
        ew = d * ew + C * U32 * (d * (w.abs() + ew) + lr) + torch.where(flip, 2.0 * lr, 0.0) + FLOOR
        w = w * d - lr * s
        em = b2 * em + C * U32 * (b2 * m.abs() + c2 * g.abs()) + FLOOR
        m = b2 * m + c2 * g
    return w, m, ew, em


def emulate_fp32(w0, m0, xs, hps, coefs=None, variant: str = None):
    """The kernels' arithmetic in fp32 on the CPU, one separately rounded torch op per product and sum, or with the defect
    ``variant``. Returns ``(w, m)`` in fp32."""
    f = torch.float32
    w, m = w0.detach().to(f).clone(), m0.detach().to(f).clone()
    for k, (x, hp) in enumerate(zip(xs, _steps(hps, len(xs)))):
        lr, b1, c1, b2, c2, d = (torch.tensor(v, dtype=f) for v in constants(hp))
        if variant == "betas_swapped":
            b1, c1, b2, c2 = b2, c2, b1, c1
        g = x.detach().to(f) if coefs is None else torch.mul(x.detach().to(f), torch.tensor(coefs[k], dtype=f))
        if variant == "coupled_weight_decay":   # L2 decay in the gradient instead of the decoupled factor
            g = torch.add(g, torch.mul(torch.tensor(float(hp.weight_decay), dtype=f), w))
            d = torch.tensor(1.0, dtype=f)
        if variant == "momentum_before_interpolation":
            m = torch.add(torch.mul(b2, m), torch.mul(c2, g))
        u = torch.add(torch.mul(b1, m), torch.mul(c1, g))
        w = torch.sub(torch.mul(w, d), torch.mul(lr, _sign(u, nan_zero=variant == "sign_nan_zero")))
        if variant != "momentum_before_interpolation":
            m = torch.add(torch.mul(b2, m), torch.mul(c2, g))
    return w, m

