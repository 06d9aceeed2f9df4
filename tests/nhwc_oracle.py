"""Float64 oracle of the fused NHWC conv epilogues in ``csrc/nhwc_fused.cu``, computed with torch on the tensors' own device.

T is bf16 or fp16; every tensor is logically NCHW and stored channels_last, exactly as the kernels see it.

* bias + ReLU forward: ``y = relu(round_T(x + b))``. ``relu`` keeps NaN (``relu(NaN) = NaN``), as torch does. The kernel adds
  in fp32 and rounds once to T; for two T values that equals rounding the exact sum once to T.
* bias + ReLU + 2x2/2 max-pool forward: the window maximum ``m`` is taken over the *pre-bias* x, ``out = relu(round_T(m + b))``.
  The argmax (0..3 = dy * 2 + dx) is the first maximum in scan order (0,0), (0,1), (1,0), (1,1); a window holding a NaN gives
  the last NaN (torch.max_pool2d's rule ``val > max || isnan(val)``).
* backward: ``gout = g`` where ``!(y <= 0)`` (NaN passes, as torch's ``threshold_backward``), else 0; the pool's ``gin`` holds
  ``g`` where ``!(out <= 0)`` at the argmax position and 0 at the other three. Both are selections, so they match bit for bit.
* bias gradient: the float64 sum of the masked gradient, rounded once to T. The kernels add fp32 partial sums: each thread over
  the rows it visits, then the threads of a block that own the same channels (shared-memory atomics), then the blocks (global
  atomics). Its error is at most ``(terms per thread + threads per channel in a block + blocks) * 2^-24 * sum|masked g|``
  before the final rounding (:func:`bias_grad_bound`). With *exact* data (:func:`make_exact`) every partial sum is exact in fp32
  in any order, so the bias gradient equals the rounded float64 sum bit for bit: a dropped or doubled row or block shows.

The pool's tie rule differs from eager torch in one place: two different x in a window can become equal after ``round_T(x + b)``.
The kernel compares before adding the bias and routes the gradient to the larger x; ``max_pool2d(relu(x + b))`` sees a tie and
routes it to the first of the tied values. Both produce the same forward output.
"""
from __future__ import annotations

import torch

U32 = 2.0 ** -24
HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}      # half an ulp, relative to the value
TINY = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24}         # smallest subnormal of T
WINDOW = ((0, 0), (0, 1), (1, 0), (1, 1))                               # argmax q = dy * 2 + dx

THREADS = 256          # kThreads in csrc/nhwc_fused.cu
GRID_CAP = 132 * 8     # grid_for's cap


def cl(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous(memory_format=torch.channels_last)


def relu(s: torch.Tensor) -> torch.Tensor:
    """ReLU that keeps NaN."""
    return torch.where(s <= 0, torch.zeros_like(s), s)


def bias_relu_fwd(x: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return cl(relu((x.double() + b.double().view(1, -1, 1, 1)).to(x.dtype)))


def pool_fwd(x: torch.Tensor, b: torch.Tensor):
    """``(out, idx)``: uint8 argmax positions in scan order, NaN rule of torch.max_pool2d."""
    xd = x.double()
    win = [xd[:, :, dy::2, dx::2] for dy, dx in WINDOW]
    m = win[0]
    idx = torch.zeros(m.shape, dtype=torch.uint8, device=x.device)
    for q in range(1, 4):
        take = (win[q] > m) | torch.isnan(win[q])
        m = torch.where(take, win[q], m)
        idx = torch.where(take, torch.full_like(idx, q), idx)
    return cl(relu((m + b.double().view(1, -1, 1, 1)).to(x.dtype))), cl(idx)


def _masked(g: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return torch.where(y <= 0, torch.zeros_like(g), g)


def bias_relu_bwd(g: torch.Tensor, y: torch.Tensor):
    """``(gout, Σ gout, Σ |gout|)``, sums in float64 per channel."""
    gout = cl(_masked(g, y))
    gd = gout.double()
    return gout, gd.sum((0, 2, 3)), gd.abs().sum((0, 2, 3))


def pool_bwd(g: torch.Tensor, out: torch.Tensor, idx: torch.Tensor, H: int, W: int):
    """``(gin, Σ masked g, Σ |masked g|)``."""
    N, C = g.shape[:2]
    gm = _masked(g, out)
    gin = torch.zeros((N, C, H, W), dtype=g.dtype, device=g.device)
    for q, (dy, dx) in enumerate(WINDOW):
        gin[:, :, dy::2, dx::2] = torch.where(idx == q, gm, torch.zeros_like(gm))
    gd = gm.double()
    return cl(gin), gd.sum((0, 2, 3)), gd.abs().sum((0, 2, 3))


# ---- launch geometry of the kernels (grid_for in csrc/nhwc_fused.cu) -----------------------------------------------------------
def grid_for(items: int) -> int:
    return max(1, min(-(-items // THREADS), GRID_CAP))


def bias_relu_fwd_passes(rows: int, C: int) -> int:
    """Grid-stride iterations of the busiest thread of bias_relu_fwd_kernel."""
    vecs = rows * C // 8
    return -(-vecs // (grid_for(vecs // 2 + 1) * THREADS))


def pool_fwd_passes(N: int, H: int, W: int, C: int) -> int:
    vecs = N * (H // 2) * (W // 2) * (C // 8)
    return -(-vecs // (grid_for(vecs) * THREADS))


def bias_relu_bwd_geometry(rows: int, C: int):
    """``(passes, depth)``: row iterations of a thread and the summation depth of the bias gradient (terms per thread + rows
    per block + blocks)."""
    rpb = THREADS // (C // 8)
    grid = grid_for(rows // rpb * THREADS // 4 + 1)
    passes = -(-rows // (grid * rpb))
    return passes, passes + rpb + grid


def pool_bwd_geometry(N: int, H: int, W: int, C: int):
    cpv = C // 8
    vecs = N * (H // 2) * (W // 2) * cpv
    grid = grid_for(vecs // 2 + 1)
    passes = -(-vecs // (grid * THREADS))
    return passes, passes + THREADS // cpv + grid


def bias_grad_bound(exact: torch.Tensor, abs_sum: torch.Tensor, depth: int, dtype: torch.dtype) -> torch.Tensor:
    """Largest distance of the kernel's bias gradient (fp32 tree of ``depth`` levels, rounded once to T) from the float64 sum."""
    err = depth * U32 * abs_sum
    return err + HALF_ULP[dtype] * (exact.abs() + err) + TINY[dtype]


def assert_same(got: torch.Tensor, want: torch.Tensor, what: str = ""):
    """Equal values (±0 equal, NaN equal NaN), same dtype and shape."""
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    torch.testing.assert_close(got, want, rtol=0, atol=0, equal_nan=True, msg=lambda m: f"{what}: {m}")


def assert_bits(got: torch.Tensor, want: torch.Tensor, what: str = ""):
    """Same bits (for NaN-free selections of g, where even the sign of zero is determined)."""
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    gi, wi = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    bad = (gi != wi).sum().item()
    assert bad == 0, f"{what}: {bad} of {got.numel()} elements differ in their bits"


def check_bias_grad(got: torch.Tensor, exact: torch.Tensor, abs_sum: torch.Tensor, depth: int, exact_data: bool, what: str = ""):
    if exact_data:
        assert_same(got, exact.to(got.dtype), what)
        return
    err = (got.double() - exact).abs()
    bound = bias_grad_bound(exact, abs_sum, depth, got.dtype)
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{what}: bias gradient off by {worst:.3g} x its bound"


# ---- data families -------------------------------------------------------------------------------------------------------------
def make_exact(shape, dtype, device, gen: torch.Generator):
    """Small integers for x and b, multiples of 2^-4 for g: exact in T, every fp32 partial sum exact (|Σ g| < 2^20 for up to
    2^21 rows per channel), many pool ties and many ``x + b == 0`` ReLU edges."""
    N, C, H, W = shape
    x = torch.randint(-4, 5, shape, generator=gen, device=device).to(dtype)
    b = torch.randint(-4, 5, (C,), generator=gen, device=device).to(dtype)
    return cl(x), b


def make_normal(shape, dtype, device, gen: torch.Generator):
    N, C, H, W = shape
    x = torch.randn(shape, generator=gen, device=device).to(dtype)
    b = torch.randn((C,), generator=gen, device=device).to(dtype)
    return cl(x), b


def make_grad(shape, dtype, device, gen: torch.Generator, exact: bool):
    if exact:
        return cl((torch.randint(-8, 9, shape, generator=gen, device=device).double() * 2.0 ** -4).to(dtype))
    return cl(torch.randn(shape, generator=gen, device=device).to(dtype))


FAMILIES = {"exact": make_exact, "normal": make_normal}
