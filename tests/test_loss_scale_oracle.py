"""Numpy / float64 oracle of dynamic loss scaling in the in-bucket sharded optimizers, checked against ``torch.amp.GradScaler``.

:func:`exchange` is ``loss_scale_norm_kernel`` (``csrc/peer_kernels.cu``): the fixed-order sum ``S`` of every rank's Σx² over the
still-scaled averaged gradient, the overflow vote, the unscaled norm, the gradient coefficient and the effective step count.
:func:`step` layers the skip rule on the per-step optimizer oracle (``tests/optim_oracle.py``). The GPU tests compare the kernels
with these; here a few steps of stock ``GradScaler`` semantics on CPU tensors are reproduced, and each deliberately wrong variant
must be caught."""
import numpy as np
import pytest
import torch

from tests import optim_oracle as oo

VARIANTS = ("step_advances_on_skip", "clip_on_scaled_norm", "first_step_consumed_by_skip")
F = np.float32


def exchange(rank_sums, scale, max_norm, t, variant=None):
    """``rank_sums``: per rank, this rank's Σ over its partials plus its parameters outside the buckets (float64), in rank order.
    Returns ``(total, coef, found_inf, t)`` with the kernel's roundings: ``total`` and ``coef`` are fp32."""
    S = np.float64(0.0)
    with np.errstate(all="ignore"):
        for s in rank_sums:
            S = S + np.float64(s)
        found = not np.isfinite(S)
        inv = np.float64(1.0) / np.float64(F(scale))
        total = F(np.sqrt(S) * inv)
        clip = F(1.0)
        if max_norm is not None and np.isfinite(max_norm):
            norm = F(np.sqrt(S)) if variant == "clip_on_scaled_norm" else total
            c = F(F(1.0) / F(norm + F(1e-6))) * F(max_norm)
            clip = c if not c > F(1.0) else F(1.0)   # a NaN norm gives a NaN coefficient, as in torch
        coef = F(F(inv) * clip)
    if variant == "step_advances_on_skip":
        return total, coef, found, t + 1
    return total, coef, found, t + (0 if found else 1)


def step(kind, state, g, hyper, vote, launches=0, variant=None):
    """One optimizer step under the vote ``(total, coef, found_inf, t)`` of :func:`exchange`; ``g`` is the scaled gradient shard,
    ``state = (w, m)`` (SGD) or ``(w, m1, m2)`` (Adam) before the step. Returns ``(new state in float64, tolerances)`` — the state
    itself (and ``None``) on a skipped step. ``launches``: steps attempted before this one, for the wrong first-step rule."""
    _, coef, found, t = vote
    if found:
        return state, None
    if kind == "sgd":
        first = launches == 0 if variant == "first_step_consumed_by_skip" else t == 1
        w, m, tol_w, tol_m = oo.sgd(state[0], g, state[1], oo.Sgd(first_step=first, grad_scale=float(coef), **hyper))
        return (w, m), (tol_w, tol_m)
    w, m1, m2, tol_w, tol_1, tol_2 = oo.adam(state[0], g, state[1], state[2], oo.Adam(step=t, grad_scale=float(coef), **hyper))
    return (w, m1, m2), (tol_w, tol_1, tol_2)


# ---------------------------------------------------------------------------------------------------------------------
# against torch.amp.GradScaler on CPU tensors
# ---------------------------------------------------------------------------------------------------------------------
N = 257
PLAN = ["inf", "ok", "ok", "nan", "ok", "ok", "ok", "ok"]   # overflow on the very first step, and again later
BOUND = 0.5


def _grads():
    g = torch.Generator().manual_seed(3)
    return [torch.randn(N, generator=g) * (0.02 if i % 2 else 0.2) for i in range(len(PLAN))]   # norms on both sides of BOUND


def _torch_run(kind, clip):
    """Stock GradScaler: unscale_ → clip_grad_norm_ → step (skipped on overflow) → update. Returns per step the state after it."""
    torch.manual_seed(1)
    p = torch.nn.Parameter(torch.randn(N))
    opt = (torch.optim.SGD([p], lr=0.1, momentum=0.9, dampening=0.5, weight_decay=1e-3) if kind == "sgd"
           else torch.optim.AdamW([p], lr=1e-2, weight_decay=0.01))
    scaler = torch.amp.GradScaler("cpu", init_scale=2.0 ** 10, growth_interval=2)
    w0, out = p.detach().clone(), []
    for what, g in zip(PLAN, _grads()):
        scaler.scale(torch.zeros(1))   # creates the scale tensor, as scaling the loss does
        scale = float(scaler.get_scale())
        sg = g * scale
        if what != "ok":
            sg[5] = float(what)
        p.grad = sg.clone()
        scaler.unscale_(opt)
        norm = torch.nn.utils.clip_grad_norm_([p], BOUND) if clip else None
        scaler.step(opt)
        scaler.update()
        st = opt.state.get(p, {})
        out.append({"scale": scale, "sg": sg, "w": p.detach().clone(), "norm": norm,
                    "t": int(st.get("step", 0)) if kind == "adam" else None,
                    "new_scale": float(scaler.get_scale()),
                    "state": tuple(st[k].clone() if k in st else torch.zeros(N) for k in (("momentum_buffer",) if kind == "sgd" else ("exp_avg", "exp_avg_sq")))})
    return w0, out


def _oracle_run(kind, clip, variant=None):
    """The oracle over the same gradients; returns the first disagreement with torch, or None."""
    w0, ref = _torch_run(kind, clip)
    hyper = dict(lr=0.1, momentum=0.9, dampening=0.5, weight_decay=1e-3) if kind == "sgd" else dict(lr=1e-2, weight_decay=0.01, adamw=True)
    state = (w0.clone(), torch.zeros(N)) if kind == "sgd" else (w0.clone(), torch.zeros(N), torch.zeros(N))
    t, scale, good = 0, 2.0 ** 10, 0
    for i, r in enumerate(ref):
        if scale != r["scale"]:
            return f"step {i}: scale {scale} vs torch {r['scale']}"
        sg = r["sg"]
        half = N // 2   # two "ranks", each with the Σx² of its half
        sums = [float(sg[:half].double().square().sum()), float(sg[half:].double().square().sum())]
        vote = exchange(sums, scale, BOUND if clip else None, t, variant)
        total, coef, found, t = vote
        if found != (PLAN[i] != "ok"):
            return f"step {i}: vote {found}"
        new, tol = step(kind, state, sg, hyper, vote, launches=i, variant=variant)
        after = (r["w"],) + r["state"]          # torch's state after its step: the next oracle step starts from it
        if found:
            if new is not state or not all(torch.equal(a, b) for a, b in zip(after, state)):
                return f"step {i}: a skipped step changed the state"
        else:
            if clip and abs(float(total) - float(r["norm"])) > 2e-6 * float(r["norm"]):
                return f"step {i}: norm {total} vs torch {float(r['norm'])}"
            # torch rounds the gradient three times (unscale, clip, update) where the kernels multiply by one coefficient
            for name, got, want, tl in zip(("weights", "momentum / exp_avg", "exp_avg_sq"), after, new, tol):
                slack = 64 * oo.U32 * (want.abs() + 1e-3)
                if oo.excess(got, want, tl + slack) > 1.0:
                    return f"step {i}: {name} differ from torch by {oo.excess(got, want, tl + slack):.1f} bounds"
        if kind == "adam" and t != r["t"]:
            return f"step {i}: step count {t} vs torch {r['t']}"
        state = after
        # torch._amp_update_scale_: back off on overflow, grow after growth_interval clean steps
        good = 0 if found else good + 1
        if found:
            scale *= 0.5
        elif good == 2:
            scale, good = scale * 2.0, 0
        if scale != r["new_scale"]:
            return f"step {i}: scale after update {scale} vs torch {r['new_scale']}"
    return None


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_oracle_reproduces_torch_grad_scaler(kind, clip):
    assert _oracle_run(kind, clip) is None


def test_every_broken_variant_is_caught():
    assert "step count" in (_oracle_run("adam", False, "step_advances_on_skip") or "")
    assert _oracle_run("adam", True, "clip_on_scaled_norm") is not None
    assert _oracle_run("sgd", True, "clip_on_scaled_norm") is not None
    got = _oracle_run("sgd", False, "first_step_consumed_by_skip") or ""
    assert "momentum" in got or "weights" in got, got


def test_exchange_roundings_and_vote():
    # the vote is on S alone: finite squares cannot overflow fp64, a single inf or NaN element makes S non-finite
    big = float(np.finfo(np.float32).max)
    total, coef, found, t = exchange([big * big * 1e6, 3.0], 2.0 ** 16, None, 4)
    assert not found and t == 5 and np.isfinite(coef) and coef == F(2.0 ** -16)
    for bad in (np.inf, np.nan):
        total, coef, found, t = exchange([1.0, bad, 2.0], 1024.0, 1.0, 4)
        assert found and t == 4 and not np.isfinite(total)
    # unscaled norm and coefficient: torch's reciprocal in double, clip with torch's operation order, one fp32 product
    total, coef, found, t = exchange([9.0, 16.0], 8.0, 0.25, 0)
    assert total == F(5.0 / 8.0) and t == 1
    want_clip = torch.clamp(0.25 / (torch.tensor(5.0 / 8.0) + 1e-6), max=1.0).numpy()
    assert coef == F(F(1.0 / 8.0) * F(want_clip))
    assert exchange([9.0, 16.0], 8.0, 100.0, 0)[1] == F(0.125)   # not clipped: the coefficient only unscales
    # with the wrong rule the bound is compared with the scaled norm
    assert exchange([9.0, 16.0], 8.0, 1.0, 0, "clip_on_scaled_norm")[1] != exchange([9.0, 16.0], 8.0, 1.0, 0)[1]
