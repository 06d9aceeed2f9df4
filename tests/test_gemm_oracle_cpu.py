"""The float64 oracle of the grouped wgmma GEMM and the MoE gather (tests/gemm_oracle.py), checked without a GPU.

* The bound is safe: an fp32 emulation of ``grouped_gemm_tn_kernel`` (each k16 slice summed in fp32, accumulated in fp32 over the
  persistent tile schedule, bias in fp32, bf16 with round-to-nearest-even) stays inside :func:`gemm_bound` on several data
  families, and gives the bits of ``ref.to(bf16)`` on integer data.
* The checks are not vacuous: each emulated defect leaves the bound on some element, or breaks bit equality on integer data.
* ``grouped_gemm_tn`` and ``grouped_linear`` reject malformed inputs before anything native is called.
"""
import math

import pytest
import torch

from tests import gemm_oracle as go

NUM_SMS = 5   # small persistent grid: CTAs walk several tiles, as 132 SMs do at MoE sizes


# ---- fp32 emulation of grouped_gemm_tn_kernel -------------------------------------------------------------------------------------
def _bf16_trunc(v: torch.Tensor) -> torch.Tensor:
    return (v.contiguous().view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


def emulate_gemm(a, b, bias=None, act="none", num_sms=NUM_SMS, defect=None):
    """The kernel's arithmetic and tile schedule in fp32 on the host; ``defect`` injects one bug."""
    G, M, K = a.shape
    N = b.shape[1]
    BN = go.block_n(N)
    BN_coord = 256 if defect == "bn256_columns" else BN
    tiles_m, tiles_n = M // go.BM, N // BN
    num_tiles = tiles_m * tiles_n * G
    grid = min(num_tiles, num_sms)
    num_kb = K // go.BK
    a32, b32 = a.float(), b.float()
    bias32 = bias.float() if bias is not None else None
    out = torch.full((G, M, N), float("nan"), dtype=torch.bfloat16)     # torch.empty: unwritten elements are garbage
    for cta in range(grid):
        acc = torch.zeros(go.BM, BN)
        for i, tile in enumerate(range(cta, num_tiles, grid)):
            m0 = (tile % tiles_m) * go.BM
            r = tile // tiles_m
            n0 = (r % tiles_n) * BN_coord
            g = r // tiles_n
            if not (defect == "stale_accumulator" and i > 0):
                acc = torch.zeros(go.BM, BN)
            A = a32[g, m0:m0 + go.BM]
            B = torch.zeros(BN, K)                                           # TMA fills rows past N with zeros
            rows = b32[g, n0:n0 + BN]
            B[:rows.shape[0]] = rows
            kbs = list(range(num_kb))
            if defect == "dropped_k_block":
                kbs.remove(num_kb - 1)
            if defect == "doubled_k_block":
                kbs.append(num_kb - 1)
            for kb in kbs:
                for k in range(go.BK // go.WGMMA_K):
                    lo = kb * go.BK + k * go.WGMMA_K
                    acc = acc + A[:, lo:lo + go.WGMMA_K] @ B[:, lo:lo + go.WGMMA_K].T
            v = acc.clone()
            if bias32 is not None:
                cols = torch.arange(n0, n0 + BN).clamp_max(N - 1)
                gb = g
                if defect == "bias_next_column":
                    cols = (cols | 1).clamp_max(N - 1)                       # b0 = brow[col + 1]: the even column takes its neighbour's bias
                if defect == "bias_next_group":
                    gb = (g + 1) % G
                if defect == "bias_previous_group":
                    gb = (g - 1) % G
                v = v + bias32[gb, cols]
            if act == "gelu":
                v = 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0))) if defect == "erf_gelu" else go.gelu_tanh(v)
            o = _bf16_trunc(v) if defect == "truncating_bf16" else v.to(torch.bfloat16)
            if defect == "rows_r_and_r_plus_8_swapped":
                o = o.view(go.BM // 16, 2, 8, BN).flip(1).reshape(go.BM, BN)
            w = min(BN, N - n0)
            if w > 0:
                out[g, m0:m0 + go.BM, n0:n0 + w] = o[:, :w]
    return out


def _within(out, a, b, bias, act) -> bool:
    ref = go.ref_gemm(a, b, bias, act)
    return bool(((out.double() - ref).abs() <= go.gemm_bound(a, b, bias, act, ref=ref)).all())


def _family(name, G, M, N, K, gen):
    if name == "int":
        return go.int_operands(G, M, N, K, gen)
    a = torch.randn(G, M, K, generator=gen)
    b = torch.randn(G, N, K, generator=gen) / math.sqrt(K)
    bias = torch.randn(G, N, generator=gen)
    if name == "uniform":
        a, b, bias = a.abs(), b.abs(), bias.abs()
    elif name == "large":
        a, b, bias = a * 2.0 ** 20, b * 2.0 ** 20, bias * 2.0 ** 40
    elif name == "small":
        a, b, bias = a * 2.0 ** -20, b * 2.0 ** -20, bias * 2.0 ** -40
    elif name == "mixed":                                                    # magnitudes over 2^±8 and both signs: heavy cancellation
        a = a * torch.exp2(torch.randint(-8, 9, a.shape, generator=gen).float())
        b = b * torch.exp2(torch.randint(-8, 9, b.shape, generator=gen).float())
    return a.to(torch.bfloat16), b.to(torch.bfloat16), bias


# (G, M, N, K): BN = 128 with 3 column tiles and BN = 256 with 2, several tiles per CTA, num_kb around STAGES
SHAPES = [(3, 256, 384, 7 * 64), (2, 384, 512, 5 * 64), (1, 128, 128, 64)]
FAMILIES = ["normal", "uniform", "large", "small", "mixed", "int"]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("act", ["none", "gelu"])
def test_fp32_emulation_stays_inside_the_bound(family, act):
    gen = torch.Generator().manual_seed(11)
    for G, M, N, K in SHAPES:
        a, b, bias = _family(family, G, M, N, K, gen)
        for bb in (bias, None):
            out = emulate_gemm(a, b, bb, act)
            assert _within(out, a, b, bb, act), (family, act, G, M, N, K, bb is None)
            if family == "int" and act == "none":
                assert torch.equal(out, go.ref_gemm(a, b, bb).to(torch.bfloat16)), (G, M, N, K)


def test_integer_operands_keep_every_partial_sum_exact():
    gen = torch.Generator().manual_seed(12)
    for K in (64, 704, 4096, 8192):
        a, b, bias = go.int_operands(1, 128, 128, K, gen)
        assert a.float().abs().max() * b.float().abs().max() * K + bias.abs().max() < go.INT_LIMIT
        assert torch.equal(a.float(), a.float().round()) and torch.equal(b.float(), b.float().round())
    a, b, bias = go.int_operands(2, 128, 256, 448, gen)
    ref = go.ref_gemm(a, b, bias)
    assert (ref.abs() > 256).float().mean() > 0.5          # most outputs need rounding to bf16: RNE vs truncation shows


GEMM_DEFECTS = ["dropped_k_block", "doubled_k_block", "stale_accumulator", "bias_next_column", "bias_next_group", "bias_previous_group",
                "rows_r_and_r_plus_8_swapped", "bn256_columns", "truncating_bf16"]


@pytest.mark.parametrize("defect", GEMM_DEFECTS + ["erf_gelu"])
def test_each_emulated_gemm_defect_is_caught(defect):
    """Caught = on normal data some element leaves the bound, or on integer data the bits differ (without GELU) / some element
    leaves the bound (with GELU) — the checks of the GPU test."""
    act = "gelu" if defect == "erf_gelu" else "none"
    G, M, N, K = 3, 256, 384, 7 * 64                     # BN = 128: 18 tiles on 5 CTAs, so every CTA walks a second tile
    gen = torch.Generator().manual_seed(13)
    caught = []
    for family in ("normal", "int"):
        a, b, bias = _family(family, G, M, N, K, gen)
        out = emulate_gemm(a, b, bias, act, defect=defect)
        if family == "int" and act == "none":
            caught.append(not torch.equal(out, go.ref_gemm(a, b, bias).to(torch.bfloat16)))
        else:
            caught.append(not _within(out, a, b, bias, act))
        assert _within(emulate_gemm(a, b, bias, act), a, b, bias, act)
    assert any(caught), defect


def test_truncation_and_erf_gelu_also_leave_the_bound_on_random_data():
    """The two subtle epilogue defects are not only visible on integer data: half an ulp is the rounding allowance."""
    gen = torch.Generator().manual_seed(14)
    a, b, bias = _family("normal", 2, 256, 256, 256, gen)
    assert not _within(emulate_gemm(a, b, bias, defect="truncating_bf16"), a, b, bias, "none")
    assert not _within(emulate_gemm(a, b, bias, "gelu", defect="erf_gelu"), a, b, bias, "gelu")


def test_gelu_slope_constant_bounds_the_derivative():
    x = torch.linspace(-12, 12, 200001, dtype=torch.float64, requires_grad=True)
    (d,) = torch.autograd.grad(go.gelu_tanh(x).sum(), x)
    assert d.abs().max().item() < go.GELU_SLOPE


# ---- MoE gather -------------------------------------------------------------------------------------------------------------------
def emulate_gather(bufs, r, eidx, sidx, weights, E_local, local_layout, defect=None):
    """``moe_gather_kernel`` for source rank r on the host: bufs[p] is rank p's buffer [P, E_local, C, M]; fp32 accumulation."""
    S, K = eidx.shape
    M = bufs[0].shape[-1]
    dtype = bufs[0].dtype
    acc = torch.zeros(S, M)
    picked = torch.zeros(S, K, M, dtype=dtype)
    ks = range(K - 1) if defect == "dropped_choice" else range(K)
    for s in range(S):
        for k in ks:
            slot = int(sidx[s, k])
            if slot < 0:
                if defect != "dropped_row_not_zero":
                    continue
                slot = 0
            e = int(eidx[s, k])
            owner, el = e // E_local, e % E_local
            frm, major = (r, owner) if local_layout else (owner, r)
            if defect == "from_major_swapped":
                frm, major = major, frm
            row = bufs[frm][major, el, slot]
            kw = (k + 1) % K if defect == "weight_of_next_choice" else (k - 1) % K if defect == "weight_of_previous_choice" else k
            w = 1.0 if weights is None else float(weights[s, kw])      # an fp32 value, exact as a double
            acc[s] = acc[s] + torch.tensor(w, dtype=torch.float32) * row.float()
            picked[s, k] = row
    return acc.to(dtype), picked


def _produced(P, E_local, C, M, dtype, gen, integer):
    """``prod[o][r]`` [E_local, C, M]: what the experts of owner o made of source rank r's slots."""
    if integer:
        return [[torch.randint(-64, 65, (E_local, C, M), generator=gen).to(dtype) for _ in range(P)] for _ in range(P)]
    return [[torch.randn(E_local, C, M, generator=gen).to(dtype) for _ in range(P)] for _ in range(P)]


def _place(prod, local_layout):
    """Pull layout: owner o holds [source r][expert][slot]; local layout (the GEMM push): source r holds [owner o][expert][slot]."""
    P = len(prod)
    if local_layout:
        return [torch.stack([prod[o][r] for o in range(P)]) for r in range(P)]
    return [torch.stack([prod[o][r] for r in range(P)]) for o in range(P)]


def _expected_picked(prod, r, eidx, sidx, E_local):
    S, K = eidx.shape
    M = prod[0][0].shape[-1]
    picked = torch.zeros(S, K, M, dtype=prod[0][0].dtype)
    for s in range(S):
        for k in range(K):
            if sidx[s, k] >= 0:
                e = int(eidx[s, k])
                picked[s, k] = prod[e // E_local][r][e % E_local, int(sidx[s, k])]
    return picked


def _pow2_weights(S, K, gen):
    return torch.exp2(torch.randint(-3, 2, (S, K), generator=gen).float())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("local_layout", [False, True])
def test_gather_emulation_matches_the_oracle(dtype, local_layout):
    P, S, K, E_local, C, M = 3, 40, 2, 2, 16, 16
    gen = torch.Generator().manual_seed(21)
    eidx, sidx = go.routing(P, S, K, E_local, C, gen)
    for integer in (True, False):
        prod = _produced(P, E_local, C, M, dtype, gen, integer)
        bufs = _place(prod, local_layout)
        for r in range(P):
            valid = sidx[r] >= 0
            want = _expected_picked(prod, r, eidx[r], sidx[r], E_local)
            for weights in (None, _pow2_weights(S, K, gen) if integer else torch.rand(S, K, generator=gen)):
                out, picked = emulate_gather(bufs, r, eidx[r], sidx[r], weights, E_local, local_layout)
                assert torch.equal(picked, want)
                ref = go.gather_ref(want, weights, valid)
                if integer:
                    assert torch.equal(out, ref.to(dtype))
                go.check_gather(out, want, weights, valid)


@pytest.mark.parametrize("defect", ["from_major_swapped", "weight_of_next_choice", "weight_of_previous_choice", "dropped_choice",
                                    "dropped_row_not_zero"])
def test_each_emulated_gather_defect_is_caught(defect):
    P, S, K, E_local, C, M, dtype = 3, 40, 3, 2, 24, 16, torch.bfloat16
    gen = torch.Generator().manual_seed(22)
    eidx, sidx = go.routing(P, S, K, E_local, C, gen)
    local_layout = defect == "from_major_swapped"
    prod = _produced(P, E_local, C, M, dtype, gen, integer=True)
    bufs = _place(prod, local_layout)
    caught = False
    for r in range(P):
        valid = sidx[r] >= 0
        want = _expected_picked(prod, r, eidx[r], sidx[r], E_local)
        weights = _pow2_weights(S, K, gen)
        out, picked = emulate_gather(bufs, r, eidx[r], sidx[r], weights, E_local, local_layout, defect=defect)
        caught |= not torch.equal(picked, want) or not torch.equal(out, go.gather_ref(want, weights, valid).to(dtype))
    assert caught, defect


def test_scatter_with_scale_is_one_multiply_and_one_rounding():
    gen = torch.Generator().manual_seed(23)
    row = torch.randn(64, generator=gen).to(torch.bfloat16)
    sc = torch.rand((), generator=gen)
    want = (row.double() * sc.double()).float().to(torch.bfloat16)      # the fp32 product of two fp32 values is the rounded exact one
    assert torch.equal(go.scatter_ref(row, sc), want)
    assert go.scatter_ref(row, None) is row


# ---- input validation: everything is rejected before the native library is touched ------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    import bagua_b200.ops.gemm as gemm

    def refuse():
        raise AssertionError("native() called for an input that must be rejected first")

    monkeypatch.setattr(gemm, "native", refuse)
    return gemm


def _ab(G=2, M=128, N=256, K=64, dtype=torch.bfloat16):
    return torch.zeros(G, M, K, dtype=dtype), torch.zeros(G, N, K, dtype=dtype)


def _gemm_cases():
    a, b = _ab()
    bias = torch.zeros(2, 256)
    return [
        ("cpu", (a, b, bias), ValueError, "CUDA"),
        ("fp16_a", (a.half(), b, bias), TypeError, "a must be bfloat16"),
        ("fp32_b", (a, b.float(), bias), TypeError, "b must be bfloat16"),
        ("devices", (a.to("meta"), b, None), ValueError, "b is on cpu"),
        ("bias_device", (a, b, bias.to("meta")), ValueError, "bias is on meta"),
        ("G_mismatch", (a, b[:1], bias), ValueError, "b must be"),
        ("K_mismatch", (a, b[:, :, :32].contiguous(), bias), ValueError, "b must be"),
        ("bias_N", (a, b, torch.zeros(256)), ValueError, "bias must be"),
        ("bias_1N", (a, b, torch.zeros(1, 256)), ValueError, "bias must be"),
        ("bias_GN1", (a, b, torch.zeros(2, 257)), ValueError, "bias must be"),
        ("bias_int", (a, b, torch.zeros(2, 256, dtype=torch.int32)), TypeError, "bias must be"),
        ("a_noncontig", (a.transpose(1, 2).contiguous().transpose(1, 2), b, bias), ValueError, "a must be contiguous"),
        ("b_noncontig", (a, b.transpose(1, 2).contiguous().transpose(1, 2), bias), ValueError, "b must be contiguous"),
        ("G0", (a[:0], b[:0], None), ValueError, "at least one group"),
        ("2d", (a[0], b[0], None), ValueError, "3-D"),
    ]


@pytest.mark.parametrize("case", [c[0] for c in _gemm_cases()])
def test_grouped_gemm_tn_rejects_malformed_inputs_before_any_native_call(no_native, case):
    _, args, exc, msg = next(c for c in _gemm_cases() if c[0] == case)
    with pytest.raises(exc, match=msg):
        no_native.grouped_gemm_tn(*args)


def test_grouped_gemm_tn_rejects_an_unknown_activation(no_native):
    a, b = _ab()
    with pytest.raises(ValueError, match="act"):
        no_native.grouped_gemm_tn(a, b, None, act="relu")


@pytest.mark.parametrize("case", ["G_mismatch", "K_mismatch", "bias_N", "bias_1N", "bias_GN1", "bias_int", "2d"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_grouped_linear_applies_the_same_shape_rules_on_the_fallback(no_native, case, dtype):
    """On CPU tensors grouped_linear runs torch.bmm; it must refuse what the kernel path refuses (a [N] bias used to broadcast)."""
    _, (a, b, bias), exc, msg = next(c for c in _gemm_cases() if c[0] == case)
    a = a.to(dtype)
    b = b.to(dtype)
    with pytest.raises(exc, match=msg.replace("b must", "w must")):
        no_native.grouped_linear(a, b, bias)


def test_grouped_linear_fallback_bias_gradient_keeps_the_bias_dtype(no_native):
    x, w = torch.randn(2, 16, 8, dtype=torch.float64), torch.randn(2, 4, 8, dtype=torch.float64)
    bias = torch.randn(2, 4, dtype=torch.float64, requires_grad=True)
    no_native.grouped_linear(x, w, bias).sum().backward()
    assert bias.grad.dtype == torch.float64 and torch.equal(bias.grad, torch.full((2, 4), 16.0, dtype=torch.float64))
