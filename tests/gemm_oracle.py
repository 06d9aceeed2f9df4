"""Float64 oracle of the grouped wgmma GEMM (``csrc/gemm_wgmma.cu``) and of the MoE gather / scatter (``csrc/moe_kernels.cu``),
computed with torch on the tensors' own device.

GEMM: ``out[g] = round_bf16(act(A[g] · B[g]^T + bias[g]))`` with bf16 A [G, M, K], B [G, N, K] and an fp32 bias [G, N]. The
kernel multiplies exactly (a bf16 product fits in fp32), accumulates in fp32 over K/16 wgmma k16 steps, adds the bias in fp32,
applies the tanh form of GELU in fp32 (``gelu_tanh``) and converts to bf16 with round-to-nearest-even. The hardware promises
neither an order nor a rounding mode inside a k16 step, so the oracle gives a bound per element rather than bits
(:func:`gemm_bound`), with ``P = |A| · |B|^T`` (float64) and ``u = 2^-24``:

* accumulation: ``E_acc = C_ACC · (K/16) · 2u · P``. Every k16 step adds one partial sum to the accumulator; a step may lose
  up to ``C_ACC = 2`` ulps (``2u`` relative, a truncating adder) of a value no larger than ``P``, and there are ``K/16`` steps.
* bias add: one fp32 rounding, ``u · (P + |bias|)``.
* GELU: the error before it is multiplied by ``max |gelu_tanh'| < GELU_SLOPE = 1.13``; evaluating it in fp32 adds at most
  ``C_GELU · u · |x|``. Derivation: ``u = k0 (x + k1 x^3)`` has no cancellation (both terms share the sign of x), so a few
  roundings and the fp32 constants give ``|du| <= 5u |u|``, which moves the result by at most ``0.5 |x| sech^2(u) |du| <=
  1.2u |x|``; ``tanhf`` (2 ulps, <= 4u absolute), ``1 + t`` and ``0.5 · x · (…)`` add ``0.5 |x| · 6u + 2u |gelu|`` — in all
  under ``6.2u · |x|``; ``C_GELU = 8`` keeps a margin.
* bf16 conversion: round to nearest is within half an ulp, ``2^-8 · (|ref| + E)`` where E is everything above, plus the
  smallest bf16 subnormal. A truncating conversion can be a whole ulp off and leaves this bound.

Integer data (:func:`int_operands`): small integers in A, B and the bias, chosen so that every product and every partial
sum is an integer below 2^20. fp32 holds those exactly, so any summation order and any rounding mode of the adders give the
exact sum, and the one conversion to bf16 (round to nearest even) gives the bits of ``ref.to(torch.bfloat16)``: without GELU
the GPU test compares with ``torch.equal``. Outputs reach a few thousand, so the conversion really rounds (bf16 holds
integers exactly only up to 256).

Gather: ``out[s] = round_T(Σ_k w[s,k] · row[s,k])`` over the choices k whose slot is valid (``slot >= 0``); rows are as stored
in T, weights fp32. The kernel accumulates ``w · row`` in fp32, K terms, with or without FMA contraction: ``|err| <= K · 2u ·
Σ_k |w| |row|`` (:func:`gather_bound`), plus half an ulp of T for 16-bit outputs. Scatter with ``scale`` is one fp32 multiply
and one rounding: ``(row.float() * scale).to(T)`` bit for bit (:func:`scatter_ref`).
"""
from __future__ import annotations

import math

import torch

U32 = 2.0 ** -24
C_ACC = 2.0
GELU_SLOPE = 1.13
C_GELU = 8.0
HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}
TINY = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24, torch.float32: 0.0}
INT_LIMIT = 2 ** 20

GELU_K0 = math.sqrt(2.0 / math.pi)
GELU_K1 = 0.044715

BM, BK, WGMMA_K = 128, 64, 16


def block_n(N: int) -> int:
    """The BN instantiation ``launch_grouped_gemm_tn`` picks."""
    return 256 if N % 256 == 0 else 128


def stages(BN: int) -> int:
    """``GemmCfg<BN>::STAGES``."""
    return 4 if BN == 256 else 6


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.tanh(GELU_K0 * (x + GELU_K1 * x * x * x)))


def _bias64(bias, G: int, N: int, like: torch.Tensor) -> torch.Tensor:
    if bias is None:
        return torch.zeros(G, 1, N, dtype=torch.float64, device=like.device)
    return bias.float().double().view(G, 1, N)


def ref_gemm(a: torch.Tensor, b: torch.Tensor, bias=None, act: str = "none") -> torch.Tensor:
    """float64 ``act(a @ b^T + bias)`` from the bf16 operands as stored and the bias as the kernel reads it (fp32)."""
    G, N = b.shape[0], b.shape[1]
    pre = torch.bmm(a.double(), b.double().transpose(1, 2)) + _bias64(bias, G, N, a)
    return gelu_tanh(pre) if act == "gelu" else pre


def gemm_bound(a: torch.Tensor, b: torch.Tensor, bias=None, act: str = "none", ref: torch.Tensor = None) -> torch.Tensor:
    """Largest distance of the kernel's bf16 output from :func:`ref_gemm`, per element (see the module docstring)."""
    G, N, K = b.shape
    if ref is None:
        ref = ref_gemm(a, b, bias, act)
    P = torch.bmm(a.double().abs(), b.double().abs().transpose(1, 2))
    err = C_ACC * (K / WGMMA_K) * 2 * U32 * P + U32 * (P + _bias64(bias, G, N, a).abs())
    if act == "gelu":
        pre = P + _bias64(bias, G, N, a).abs()           # |x| <= P + |bias|, whatever the sign of the cancellation
        err = GELU_SLOPE * err + C_GELU * U32 * (pre + err)
    return err + HALF_ULP[torch.bfloat16] * (ref.abs() + err) + TINY[torch.bfloat16]


def check_gemm(out: torch.Tensor, a, b, bias=None, act: str = "none", what: str = ""):
    """``out`` within :func:`gemm_bound` of :func:`ref_gemm` everywhere (NaN fails)."""
    ref = ref_gemm(a, b, bias, act)
    bound = gemm_bound(a, b, bias, act, ref=ref)
    ratio = (out.double() - ref).abs() / bound
    worst = ratio.nan_to_num(float("inf")).max().item()
    assert worst <= 1.0, f"{what}: off by {worst:.3g} x the bound at {divmod(int(ratio.nan_to_num(float('inf')).argmax()), out.shape[-1])}"


def int_range(K: int, bias_max: int = 256) -> int:
    """Largest magnitude m <= 16 of the integer operands with ``K · m^2 + bias_max < 2^20``."""
    m = 16
    while K * m * m + bias_max >= INT_LIMIT:
        m -= 1
    assert m >= 1, K
    return m


def int_operands(G: int, M: int, N: int, K: int, gen: torch.Generator, device="cpu"):
    """``(a, b, bias)``: integers in [-m, m] for the operands (bf16) and in [-256, 256] for the bias (fp32), see :func:`int_range`.
    Every partial sum of the GEMM is an integer of magnitude below 2^20, hence exact in fp32."""
    m = int_range(K)
    a = torch.randint(-m, m + 1, (G, M, K), generator=gen, device=gen.device).to(torch.bfloat16)
    b = torch.randint(-m, m + 1, (G, N, K), generator=gen, device=gen.device).to(torch.bfloat16)
    bias = torch.randint(-256, 257, (G, N), generator=gen, device=gen.device).float()
    return a.to(device), b.to(device), bias.to(device)


# ---- MoE gather / scatter ---------------------------------------------------------------------------------------------------------
def gather_ref(picked: torch.Tensor, weights, valid: torch.Tensor) -> torch.Tensor:
    """float64 ``Σ_k w[s,k] · picked[s,k]`` over the valid choices; ``picked`` [S, K, M] as stored, ``weights`` [S, K] fp32 or None."""
    w = torch.ones(valid.shape, dtype=torch.float64, device=picked.device) if weights is None else weights.double()
    w = w * valid.double()
    return (picked.double() * w.unsqueeze(-1)).sum(1)


def gather_bound(picked: torch.Tensor, weights, valid: torch.Tensor, dtype: torch.dtype, ref: torch.Tensor = None) -> torch.Tensor:
    """``K · 2u · Σ_k |w| |row|`` (fp32 accumulation, with or without FMA) plus half an ulp of ``dtype`` for the final rounding."""
    K = valid.shape[1]
    if ref is None:
        ref = gather_ref(picked, weights, valid)
    mag = gather_ref(picked.abs(), None if weights is None else weights.abs(), valid)
    err = K * 2 * U32 * mag
    return err + HALF_ULP[dtype] * (ref.abs() + err) + TINY[dtype]


def check_gather(out: torch.Tensor, picked: torch.Tensor, weights, valid: torch.Tensor, what: str = ""):
    """``out`` within :func:`gather_bound` of :func:`gather_ref` everywhere (an fp32 bound is 0 where every choice is dropped)."""
    ref = gather_ref(picked, weights, valid)
    bound = gather_bound(picked, weights, valid, out.dtype, ref=ref)
    err = (out.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the bound, worst error {err.max().item():.3g}"


def routing(P: int, S: int, K: int, E_local: int, C: int, gen: torch.Generator):
    """Per source rank: ``(expert_idx, slot_idx)`` [S, K] int64 on the CPU, K distinct experts per token, slots filled in token
    order up to the capacity C; every token with ``s % 5 == 3`` has all its choices dropped, and the second choice of every
    seventh token is dropped."""
    E = P * E_local
    eidx, sidx = [], []
    for _ in range(P):
        e = torch.stack([torch.randperm(E, generator=gen)[:K] for _ in range(S)])
        slot = torch.full((S, K), -1, dtype=torch.int64)
        fill = [0] * E
        for s in range(S):
            for k in range(K):
                ex = int(e[s, k])
                if fill[ex] < C and s % 5 != 3 and not (s % 7 == 0 and k == 1):
                    slot[s, k] = fill[ex]
                    fill[ex] += 1
        eidx.append(e)
        sidx.append(slot)
    return eidx, sidx


def scatter_ref(row: torch.Tensor, scale) -> torch.Tensor:
    """What the scatter stores for one (token, choice): the row as is, or ``round_T(fp32(row) · fp32(scale))``."""
    if scale is None:
        return row
    return (row.float() * scale.float()).to(row.dtype)
