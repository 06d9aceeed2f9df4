"""Float64 oracle of one LARS step (``csrc/lars.cuh``) with a per-element error bound, in the style of ``lamb_oracle.py``.

Each call starts from the kernel's own state before the step: fp32 master weights ``w``, the momentum ``v`` (which holds the
lr-scaled step), the gradient as the kernel reads it (the fp32 shard, or the parameter's gradient in its dtype) and the
clip / unscale coefficient ``coef``. Hyperparameters are used as the launchers receive them, in fp32. The rule::

    g̃ = coef·g;  W = Σw², G = Σg̃² over the whole parameter
    trust = eta·√W / (√G + wd·√W) when wd ≠ 0 and W > 0 and G > 0 (rounded to fp32 once); NaN when W or G is NaN; else 1
    v ← μ·v + (lr·trust)·(g̃ + wd·w);  w ← w − v

Bound, per element: ``C·2^-24`` times the magnitudes that enter ``v`` (``μ|v| + lr·trust·(|g̃| + wd·|w|)``; the trust's own
relative error — one rounding of ``g̃`` through ``√G``, one fp32 rounding of the quotient, one of ``lr·trust`` — is a few
``2^-24`` and sits inside ``C``), plus ``C·2^-24·(|w| + |v_new|)`` for ``w``. ``variant`` selects a deliberately wrong update;
``tests/test_lars_oracle.py`` shows that each of them leaves the bound.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

from tests.optim_oracle import FLOOR, U32, C, _d, f32, half_ulp

VARIANTS = ("torch_momentum", "trust_without_decay_term", "adapt_without_decay", "per_shard_norms", "norms_before_coef", "nan_trust_one")


@dataclass
class Lars:
    lr: float
    momentum: float = 0.9
    weight_decay: float = 5e-4
    trust_coefficient: float = 1e-3
    coef: float = 1.0
    prev_lr: Optional[float] = None   # lr of the step that produced v; only the torch_momentum variant reads it (None: = lr)


def trust(w2: float, g2: float, hp: Lars, variant: str = None) -> float:
    """The trust of a parameter from its global Σw², Σg̃² (float64), rounded to fp32 once."""
    wd, eta = f32(hp.weight_decay), f32(hp.trust_coefficient)
    if math.isnan(w2) or math.isnan(g2):
        return 1.0 if variant == "nan_trust_one" else float("nan")
    if (wd == 0.0 and variant != "adapt_without_decay") or not (w2 > 0.0 and g2 > 0.0):
        return 1.0
    sw = math.sqrt(w2)
    den = math.sqrt(g2) if variant in ("trust_without_decay_term", "adapt_without_decay") else math.sqrt(g2) + wd * sw
    return f32(eta * sw / den)


def lars(params, hp: Lars, variant: str = None):
    """One LARS step of the parameters of ONE parameter group: ``params`` is a list of ``(w, g, v)``, each the WHOLE parameter
    (flat). Returns a list of ``(w, v, trust, tol_w, tol_v)`` in float64 (``trust`` a float)."""
    lr, mu, wd, s = f32(hp.lr), f32(hp.momentum), f32(hp.weight_decay), f32(hp.coef)
    out = []
    for w, g, v in params:
        w, g, v = _d(w), _d(g), _d(v)
        gt = g * s
        gn = g if variant == "norms_before_coef" else gt
        if variant == "per_shard_norms":   # this rank's part of the parameter only
            k = max(1, w.numel() // 2)
            tr = trust(float(w[:k].square().sum()), float(gn[:k].square().sum()), hp, variant)
        else:
            tr = trust(float(w.square().sum()), float(gn.square().sum()), hp, variant)
        lt = f32(lr * tr) if not math.isnan(tr) else float("nan")
        d = gt + wd * w
        if variant == "torch_momentum":   # torch.optim.SGD keeps v/lr and scales the whole buffer by the CURRENT lr
            prev = f32(hp.prev_lr) if hp.prev_lr is not None else lr
            v_new = lr * (mu * (v / prev) + tr * d)
        else:
            v_new = mu * v + lt * d
        w_new = w - v_new
        mag = mu * v.abs() + abs(lt) * (gt.abs() + wd * w.abs())
        tol_v = C * U32 * mag + FLOOR
        tol_w = tol_v + C * U32 * (w.abs() + v_new.abs()) + FLOOR
        out.append((w_new, v_new, tr, tol_w, tol_v))
    return out


def emulate_fp32(params, hp: Lars):
    """The kernels' arithmetic in fp32 on the CPU (every operation rounded as lars.cuh rounds it, fp64 norms): the positive
    control of the bound. Returns ``[(w, v, trust)]`` in fp32."""
    f = torch.float32
    lr, mu, wd, s = (torch.tensor(x, dtype=f) for x in (hp.lr, hp.momentum, hp.weight_decay, hp.coef))
    out = []
    for w, g, v in params:
        w, v = w.to(f), v.to(f)
        gt = g.to(f) * s
        tr = torch.tensor(trust(float(w.double().square().sum()), float(gt.double().square().sum()), hp), dtype=f)
        lt = lr * tr
        v = mu * v + lt * (gt + wd * w)
        out.append((w - v, v, float(tr)))
    return out


def excess(actual: torch.Tensor, expected: torch.Tensor, tol: torch.Tensor) -> float:
    """``optim_oracle.excess`` that also compares NaNs: a NaN on one side only is an infinite excess, NaN on both sides none."""
    a = actual.detach().to(torch.float64).reshape(expected.shape)
    na, ne = torch.isnan(a), torch.isnan(expected)
    if bool((na != ne).any()):
        return math.inf
    keep = ~ne
    if not bool(keep.any()):
        return 0.0
    a, e, t = a[keep], expected[keep], tol[keep]
    bound = t + half_ulp(e.abs() + t, actual.dtype)
    return float(((a - e).abs() / bound).max())
