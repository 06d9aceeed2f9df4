"""Float64 oracle of one LAMB step (``csrc/lamb.cuh``) with a per-element error bound, in the style of ``optim_oracle.py``.

Each call starts from the kernel's own state before the step: fp32 master weights, both moments, the gradient as the kernel reads
it (the fp32 shard, or the parameter's gradient in its dtype) and the clipping coefficient ``coef``. Hyperparameters are used as
the launchers receive them: fp32 ``lr``, betas, ``eps``, ``weight_decay`` and ``coef``; ``1 - beta`` is evaluated in fp32 and the
bias corrections are ``1 - beta^t`` rounded to fp32.

Bound, per element of a parameter: the Adam-like terms of ``optim_oracle.adam`` for the direction ``u`` (``C·2^-24`` times ``u``
evaluated on absolute values, the second moment's error through the square root, one fp32 ulp of ``beta^t``), carried through
``lr·r``, plus ``lr·r·|u|`` times the ratio's relative error: ``‖tol_u‖₂ / ‖u‖₂`` (how far the fp32 directions can move ``‖u‖``;
``‖w‖`` is exact) plus two fp32 ulps (the fp64 norms' quotient rounded to fp32 once). ``variant`` selects a deliberately wrong
update; ``tests/test_lamb_oracle.py`` shows that each of them leaves the bound.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from tests.optim_oracle import FLOOR, U32, C, _bias_correction, _d, f32

VARIANTS = ("local_segment_ratio", "bucket_ratio", "ratio_without_decay", "norms_after_update", "bias_correction_of_previous_step",
            "eps_inside_sqrt", "l2_decay_in_gradient", "no_coef")


@dataclass
class Lamb:
    lr: float
    step: int
    betas: tuple = (0.9, 0.999)
    eps: float = 1e-6
    weight_decay: float = 0.01
    coef: float = 1.0


def _direction(w, g, m1, m2, hp: Lamb, variant):
    b1, b2, eps, wd, s = f32(hp.betas[0]), f32(hp.betas[1]), f32(hp.eps), f32(hp.weight_decay), f32(hp.coef)
    t = hp.step - 1 if variant == "bias_correction_of_previous_step" else hp.step
    bc1, dbc1 = _bias_correction(b1, t)
    bc2, dbc2 = _bias_correction(b2, t)
    omb1, omb2 = f32(1.0 - b1), f32(1.0 - b2)
    gs = g * (1.0 if variant == "no_coef" else s)
    Mg = gs.abs()
    if variant == "l2_decay_in_gradient":
        gs, Mg = gs + wd * w, Mg + wd * w.abs()
    m1n, m2n = b1 * m1 + omb1 * gs, b2 * m2 + omb2 * gs * gs
    Mm1, Mm2 = b1 * m1.abs() + omb1 * Mg, b2 * m2.abs() + omb2 * Mg * Mg
    denom = torch.sqrt(m2n / bc2 + eps) if variant == "eps_inside_sqrt" else torch.sqrt(m2n) / (bc2 ** 0.5) + eps
    adam = (m1n / bc1) / denom
    u = adam if variant == "l2_decay_in_gradient" else adam + wd * w
    tol_m1, tol_m2 = C * U32 * Mm1 + FLOOR, C * U32 * Mm2 + FLOOR
    Mu = (Mm1 / bc1) / denom + wd * w.abs()
    denom_err = adam.abs() * (torch.sqrt(m2n.abs() + tol_m2) - torch.sqrt(m2n.abs())) / (bc2 ** 0.5) / denom
    pow_err = adam.abs() * (dbc1 / bc1 + dbc2 / (2.0 * bc2))
    tol_u = C * U32 * Mu + denom_err + pow_err + FLOOR
    return u, m1n, m2n, tol_u, tol_m1, tol_m2


def direction(w, g, m1, m2, hp: Lamb):
    """The update direction ``u`` of one parameter and its per-element bound ``tol_u`` (float64): what Σu² is made of."""
    u, _, _, tol_u, _, _ = _direction(_d(w), _d(g), _d(m1), _d(m2), hp, None)
    return u, tol_u


def sum_bound(terms) -> float:
    """A-priori bound on how far a float64 sum of the non-negative ``terms``, added in ANY order, lies from the exact sum:
    ``(n − 1)·2^-53·Σ terms`` (Higham, "Accuracy and Stability of Numerical Algorithms", eq. 4.4)."""
    n = len(terms)
    return max(n - 1, 0) * 2.0 ** -53 * math.fsum(terms) * (1.0 + 1e-12)


def _ratio(w2, u2, wd, variant):
    if (wd == 0.0 and variant != "ratio_without_decay") or not (w2 > 0.0 and u2 > 0.0):
        return 1.0
    return (w2 ** 0.5) / (u2 ** 0.5)


def lamb(params, hp: Lamb, variant: str = None):
    """One LAMB step of the parameters of ONE bucket (one parameter group): ``params`` is a list of ``(w, g, m1, m2)``, each the
    WHOLE parameter (flat). Returns a list of ``(w, m1, m2, r, tol_w, tol_m1, tol_m2)`` in float64 (``r`` a float)."""
    lr, wd = f32(hp.lr), f32(hp.weight_decay)
    dirs = [_direction(_d(w), _d(g), _d(a), _d(b), hp, variant) for w, g, a, b in params]
    bucket_w2 = sum(float(_d(w).square().sum()) for w, *_ in params)
    bucket_u2 = sum(float(d[0].square().sum()) for d in dirs)
    out = []
    for (w, *_), (u, m1n, m2n, tol_u, tol_m1, tol_m2) in zip(params, dirs):
        w = _d(w)
        if variant == "local_segment_ratio":   # this rank's part of the parameter only
            k = max(1, w.numel() // 2)
            r = _ratio(float(w[:k].square().sum()), float(u[:k].square().sum()), wd, variant)
        elif variant == "bucket_ratio":
            r = _ratio(bucket_w2, bucket_u2, wd, variant)
        elif variant == "norms_after_update":
            r = _ratio(float((w - lr * u).square().sum()), float(u.square().sum()), wd, variant)
        else:
            r = _ratio(float(w.square().sum()), float(u.square().sum()), wd, variant)
        un = float(u.norm())
        rel_r = (float(tol_u.norm()) / un if un > 0 else 0.0) + 2.0 * U32 if r != 1.0 else 0.0
        w_new = w - lr * r * u
        tol_w = C * U32 * (w.abs() + lr * r * (u.abs() + tol_u)) + lr * r * tol_u + lr * r * u.abs() * rel_r + FLOOR
        out.append((w_new, m1n, m2n, r, tol_w, tol_m1, tol_m2))
    return out


def emulate_fp32(params, hp: Lamb):
    """The kernels' arithmetic in fp32 on the CPU (every operation rounded as lamb.cuh rounds it, fp64 norms): the positive control
    of the bound. Returns ``[(w, m1, m2)]`` in fp32."""
    f = torch.float32
    b1, b2 = torch.tensor(hp.betas[0], dtype=f), torch.tensor(hp.betas[1], dtype=f)
    eps, wd, lr, s = (torch.tensor(x, dtype=f) for x in (hp.eps, hp.weight_decay, hp.lr, hp.coef))
    bc1 = torch.tensor(1.0 - float(b1) ** hp.step, dtype=f)
    bc2 = torch.tensor(1.0 - float(b2) ** hp.step, dtype=f)
    inv_bc1 = torch.tensor(1.0 / float(bc1), dtype=f)
    rs_bc2 = torch.tensor(1.0 / float(bc2) ** 0.5, dtype=f)
    out = []
    for w, g, a, b in params:
        w, g, a, b = w.to(f), g.to(f) * s, a.to(f), b.to(f)
        a = b1 * a + (1 - b1) * g
        b = b2 * b + ((1 - b2) * g) * g
        u = (a * inv_bc1) / (torch.sqrt(b) * rs_bc2 + eps) + wd * w
        w2, u2 = float(w.double().square().sum()), float(u.double().square().sum())
        r = torch.tensor((w2 ** 0.5) / (u2 ** 0.5) if float(wd) != 0 and w2 > 0 and u2 > 0 else 1.0, dtype=f)
        out.append((w - (lr * r) * u, a, b))
    return out
