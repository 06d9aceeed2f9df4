"""Float64 oracle of one optimizer step of the kernels in ``csrc/multi_tensor.cu``, with a per-element error bound.

Each call starts from the kernel's own state before the step (fp32 master or parameter, moments or momentum, the gradient
as stored in its dtype), so errors never compound and the bound stays at a few fp32 ulps however many steps a test runs.
Hyperparameters are used as the launchers receive them: fp32 ``lr``, ``momentum``, ``dampening``, ``weight_decay``,
``eps``, betas and ``grad_scale``; ``1 - dampening`` and ``1 - beta`` are evaluated in fp32, and the bias corrections are
``1 - beta^t`` rounded to fp32 as ``make_adam`` (``csrc/bindings.cpp``) computes them.

Bound, per element: ``C * 2^-24 * M + FLOOR``, where ``M`` is the same formula evaluated on absolute values (so cancellation
in the exact result does not shrink the bound below the rounding error of its terms).  ``C`` covers a handful of fp32
roundings along the chain plus FMA contraction, ``sqrtf`` and the division.  ``powf`` is not correctly rounded, so the Adam
bound also carries what one fp32 ulp of ``beta^t`` does to the update, and the bound of the second moment carried through the
square root of the denominator (it matters where ``g + wd * w`` cancels).  A low-precision result stored without an fp32 copy
adds half an ulp of its dtype (:func:`check`).  ``variant`` selects a deliberately wrong update; the CPU suite shows that every
one of them leaves the bound (``tests/test_optimizer_oracle.py``).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

C = 12.0
U32 = 2.0 ** -24
FLOOR = 2.0 ** -122  # 16x the smallest normal fp32: results that underflow into (or flush from) the subnormal range

SGD_VARIANTS = ("dampening_on_first_step", "nesterov_with_old_momentum", "no_grad_scale", "weight_decay_after_momentum")
ADAM_VARIANTS = ("eps_inside_sqrt", "bias_correction_of_previous_step", "l2_decay_in_adamw", "no_grad_scale")


def f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


@dataclass
class Sgd:
    lr: float
    momentum: float = 0.0
    dampening: float = 0.0
    weight_decay: float = 0.0
    nesterov: bool = False
    first_step: bool = False
    grad_scale: float = 1.0


@dataclass
class Adam:
    lr: float
    step: int
    betas: tuple = (0.9, 0.999)
    eps: float = 1e-8
    weight_decay: float = 0.0
    adamw: bool = False
    grad_scale: float = 1.0


def _d(t):
    return t.detach().to(torch.float64)


def sgd(w, g, m, hp: Sgd, variant: str = None):
    """One SGD step.  ``w``: fp32 master or parameter, ``g``: gradient as stored, ``m``: momentum before the step (ignored when
    ``hp.momentum == 0`` or on the first step).  Returns ``(w, m, tol_w, tol_m)`` in float64 (``m``/``tol_m`` None without
    momentum)."""
    w, g = _d(w), _d(g)
    lr, mu, wd, s = f32(hp.lr), f32(hp.momentum), f32(hp.weight_decay), f32(hp.grad_scale)
    omd = f32(1.0 - f32(hp.dampening))
    if variant == "no_grad_scale":
        s = 1.0
    gs = g * s
    d = gs if variant == "weight_decay_after_momentum" else gs + wd * w
    Md = gs.abs() + wd * w.abs()
    m_new = tol_m = None
    upd, Mu = d, Md
    if mu != 0.0:
        m = _d(m)
        if hp.first_step:
            m_new, Mm = (omd * d if variant == "dampening_on_first_step" else d), Md
        else:
            m_new, Mm = mu * m + omd * d, mu * m.abs() + omd * Md
        if hp.nesterov:
            upd = d + mu * (m if variant == "nesterov_with_old_momentum" else m_new)
            Mu = Md + mu * Mm
        else:
            upd, Mu = m_new, Mm
        if variant == "weight_decay_after_momentum":
            upd = upd + wd * w
        tol_m = C * U32 * Mm + FLOOR
    w_new = w - lr * upd
    tol_w = C * U32 * (w.abs() + lr * Mu) + FLOOR
    return w_new, m_new, tol_w, tol_m


def _bias_correction(beta: float, t: int) -> tuple:
    """``(1 - beta^t, |d bc|)`` as make_adam computes it in fp32, and what one fp32 ulp of ``beta^t`` changes in it."""
    p = f32(beta ** t)
    return f32(1.0 - p), 2.0 * U32 * p


def adam(w, g, m1, m2, hp: Adam, variant: str = None):
    """One Adam/AdamW step.  Returns ``(w, m1, m2, tol_w, tol_m1, tol_m2)`` in float64."""
    w, g, m1, m2 = _d(w), _d(g), _d(m1), _d(m2)
    lr, b1, b2, eps, wd, s = f32(hp.lr), f32(hp.betas[0]), f32(hp.betas[1]), f32(hp.eps), f32(hp.weight_decay), f32(hp.grad_scale)
    t = hp.step - 1 if variant == "bias_correction_of_previous_step" else hp.step
    bc1, dbc1 = _bias_correction(b1, t)
    bc2, dbc2 = _bias_correction(b2, t)
    omb1, omb2 = f32(1.0 - b1), f32(1.0 - b2)
    if variant == "no_grad_scale":
        s = 1.0
    gs = g * s
    Mg = gs.abs()
    w0 = w
    if hp.adamw:
        w = w * (1.0 - lr * wd)
        if variant == "l2_decay_in_adamw":
            gs = gs + wd * w0
    else:
        gs = gs + wd * w
        Mg = Mg + wd * w.abs()
    m1n = b1 * m1 + omb1 * gs
    m2n = b2 * m2 + omb2 * gs * gs
    Mm1 = b1 * m1.abs() + omb1 * Mg
    Mm2 = b2 * m2.abs() + omb2 * Mg * Mg
    if variant == "eps_inside_sqrt":
        denom = torch.sqrt(m2n / bc2 + eps)
    else:
        denom = torch.sqrt(m2n) / (bc2 ** 0.5) + eps
    step_size = lr / bc1
    upd = step_size * (m1n / denom)
    w_new = w - upd
    tol_m1, tol_m2 = C * U32 * Mm1 + FLOOR, C * U32 * Mm2 + FLOOR
    # rounding of every term; the error of the second moment through the denominator (large where g + wd*w cancels);
    # one ulp of beta^t in either bias correction
    Mupd = step_size * Mm1 / denom
    denom_err = upd.abs() * (torch.sqrt(m2n.abs() + tol_m2) - torch.sqrt(m2n.abs())) / (bc2 ** 0.5) / denom
    pow_err = upd.abs() * (dbc1 / bc1 + dbc2 / (2.0 * bc2))
    tol_w = C * U32 * (w0.abs() + Mupd) + denom_err + pow_err + FLOOR
    return w_new, m1n, m2n, tol_w, tol_m1, tol_m2


def wide(n: int, gen: torch.Generator, lo: float = -30.0, hi: float = 4.0, zeros: float = 0.05, positive: bool = False) -> torch.Tensor:
    """fp32 values of random sign whose magnitudes are log-uniform in [10^lo, 10^hi], with a share of exact zeros, on the
    generator's device."""
    dev = gen.device
    mag = torch.pow(10.0, lo + (hi - lo) * torch.rand(n, generator=gen, dtype=torch.float64, device=dev))
    sign = 1.0 if positive else torch.where(torch.rand(n, generator=gen, device=dev) < 0.5, -1.0, 1.0).to(torch.float64)
    x = (mag * sign).float()
    x[torch.rand(n, generator=gen, device=dev) < zeros] = 0.0
    return x


_LOWP = {torch.bfloat16: (8, -126), torch.float16: (11, -14)}


def half_ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Half an ulp of ``dtype`` at ``|x|`` (float64), 0 for fp32."""
    if dtype not in _LOWP:
        return torch.zeros_like(x)
    bits, emin = _LOWP[dtype]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - bits)


def excess(actual: torch.Tensor, expected: torch.Tensor, tol: torch.Tensor) -> float:
    """Largest ``|actual - expected| / tol`` (> 1 means out of bounds); ``actual`` is rounded to its own dtype, whose half ulp
    widens the bound."""
    a = actual.detach().to(torch.float64).reshape(expected.shape)
    bound = tol + half_ulp(expected.abs() + tol, actual.dtype)
    return float(((a - expected).abs() / bound).max()) if a.numel() else 0.0


def check(actual, expected, tol, what: str = ""):
    a = actual.detach().to(torch.float64).reshape(expected.shape)
    bound = tol + half_ulp(expected.abs() + tol, actual.dtype)
    bad = (a - expected).abs() > bound
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bounds; first at flat index {i}: got "
                             f"{float(a.flatten()[i])!r}, oracle {float(expected.flatten()[i])!r}, bound {float(bound.flatten()[i])!r}")
