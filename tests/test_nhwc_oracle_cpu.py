"""CPU checks of the NHWC epilogue oracle (tests/nhwc_oracle.py) and of the host-side guards in front of the kernels.

* The oracle's rules are torch's: ReLU, its gradient and max_pool2d's argmax on NaN, ±inf, ±0 and ties.
* The checks catch subtly wrong kernels, emulated here in fp32: a dropped or doubled row in the bias gradient, the last instead of
  the first maximum, one channel vector reading the wrong bias, NaN turned into 0.
* The raw bindings reject misaligned pointers by name before anything is launched, and ops/nhwc.py only hands the kernels
  16-byte aligned tensors.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import nhwc_oracle as oracle

DTYPES = [torch.bfloat16, torch.float16]
SPECIALS = [float("nan"), float("inf"), float("-inf"), -0.0, 0.0, 1.0, 1.0, -1.0]


def _special_tensor(shape, dtype, gen):
    vals = torch.tensor(SPECIALS, dtype=torch.float64)
    return oracle.cl(vals[torch.randint(0, len(SPECIALS), shape, generator=gen)].to(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
def test_oracle_pool_rule_is_torch_max_pool2d(dtype):
    """Argmax and value of the oracle's window scan equal torch.max_pool2d's (pre-bias x, bias 0) with NaN, ±inf, ±0 and ties."""
    gen = torch.Generator().manual_seed(0)
    x = _special_tensor((3, 8, 6, 10), dtype, gen)
    out, idx = oracle.pool_fwd(x, torch.zeros(8, dtype=dtype))
    m, flat = F.max_pool2d(x.double(), 2, 2, return_indices=True)
    W = x.shape[3]
    ho = torch.arange(m.shape[2]).view(1, 1, -1, 1)
    wo = torch.arange(m.shape[3]).view(1, 1, 1, -1)
    q = (flat // W - 2 * ho) * 2 + (flat % W - 2 * wo)
    assert torch.equal(idx.long(), q)
    oracle.assert_same(out, oracle.relu(m).to(dtype))
    assert torch.isnan(out).any() and (idx > 0).any()


@pytest.mark.parametrize("dtype", DTYPES)
def test_oracle_relu_rule_is_torch_relu_and_its_gradient(dtype):
    gen = torch.Generator().manual_seed(1)
    x = _special_tensor((2, 8, 4, 4), dtype, gen)
    b = torch.zeros(8, dtype=dtype)
    y = oracle.bias_relu_fwd(x, b)
    oracle.assert_same(y, torch.relu(x))
    xr = x.double().requires_grad_(True)
    g = oracle.make_grad(x.shape, dtype, "cpu", gen, exact=True)
    torch.relu(xr).backward(g.double())
    gout, _, _ = oracle.bias_relu_bwd(g, y)
    oracle.assert_same(gout, xr.grad.to(dtype))
    assert torch.isnan(y).any() and (gout[torch.isnan(y)] == g[torch.isnan(y)]).all()


def _emulated_kernel(x, b, g, pool, variant=None):
    """What the kernels compute, in fp32 on the host, optionally with one defect."""
    T = x.dtype
    bf = b.float().view(1, -1, 1, 1)
    if variant == "channel_vector":                   # the second channel vector reads the first one's bias
        bf = bf.clone()
        bf[:, 8:16] = bf[:, 0:8]
    if not pool:
        s = x.float() + bf
        y = (torch.where(s > 0, s, 0.0) if variant == "nan_to_zero" else oracle.relu(s)).to(T)
        gm = torch.where(y <= 0, torch.zeros_like(g), g)
        out, idx = y, None
    else:
        win = [x.float()[:, :, dy::2, dx::2] for dy, dx in oracle.WINDOW]
        m, idx = win[0], torch.zeros(win[0].shape, dtype=torch.uint8)
        for q in range(1, 4):
            take = win[q] >= m if variant == "last_max" else (win[q] > m) | torch.isnan(win[q])
            m, idx = torch.where(take, win[q], m), torch.where(take, torch.full_like(idx, q), idx)
        s = m + bf
        out = (torch.where(s > 0, s, 0.0) if variant == "nan_to_zero" else oracle.relu(s)).to(T)
        gm = torch.where(out <= 0, torch.zeros_like(g), g)
    rows = gm.float().permute(0, 2, 3, 1).reshape(-1, x.shape[1])
    if variant == "drop_row":
        rows = rows[:-1]
    if variant == "double_row":
        rows = torch.cat([rows, rows[-1:]])
    return out, idx, gm, rows.sum(0).to(T)


VARIANTS = ["drop_row", "double_row", "last_max", "channel_vector", "nan_to_zero"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pool", [False, True])
@pytest.mark.parametrize("variant", [None] + VARIANTS)
def test_checks_catch_wrong_kernels(dtype, pool, variant):
    """On exact data (plus NaNs for the NaN variant) the correct emulation passes every check and each defect fails one."""
    gen = torch.Generator().manual_seed(2)
    shape = (3, 16, 6, 10)
    x, b = oracle.make_exact(shape, dtype, "cpu", gen)
    if variant == "nan_to_zero":
        x = x.clone()
        x[0, :, 0, 0] = float("nan")
    gshape = (3, 16, 3, 5) if pool else shape
    g = oracle.make_grad(gshape, dtype, "cpu", gen, exact=True)
    out, idx, gm, bias_grad = _emulated_kernel(x, b, g, pool, variant)

    def check():
        if pool:
            want_out, want_idx = oracle.pool_fwd(x, b)
            oracle.assert_same(out, want_out, "out")
            assert torch.equal(idx, want_idx), "idx"
            _, exact, abs_sum = oracle.pool_bwd(g, want_out, want_idx, 6, 10)
        else:
            want_y = oracle.bias_relu_fwd(x, b)
            oracle.assert_same(out, want_y, "y")
            want_g, exact, abs_sum = oracle.bias_relu_bwd(g, want_y)
            oracle.assert_same(gm, want_g, "gout")
        oracle.check_bias_grad(bias_grad, exact, abs_sum, 1, True, "bias_grad")

    if variant is None or (variant == "last_max" and not pool):
        check()
    else:
        with pytest.raises(AssertionError):
            check()


def test_bias_grad_bound_holds_for_fp32_sums_and_catches_a_dropped_row():
    """Normal data: an fp32 sum in any order stays inside the bound; losing one row of a channel leaves it."""
    gen = torch.Generator().manual_seed(3)
    for dtype in DTYPES:
        g = torch.randn(4096, 8, generator=gen).to(dtype)
        exact = g.double().sum(0)
        abs_sum = g.double().abs().sum(0)
        for got in (g.float().sum(0), g.float().flip(0).cumsum(0)[-1], g.float().view(64, 64, 8).sum(1).sum(0)):
            oracle.check_bias_grad(got.to(dtype), exact, abs_sum, 4096, False)
        with pytest.raises(AssertionError):
            oracle.check_bias_grad(g[1:].float().sum(0).to(dtype), exact, abs_sum, 16, False)


def test_large_test_shapes_wrap_every_grid_stride_loop():
    """The large test shapes make every kernel's grid-stride loop wrap (grid capped at 132 * 8 blocks of 256 threads)."""
    assert oracle.bias_relu_fwd_passes(8 * 112 * 112, 64) > 1
    assert oracle.pool_fwd_passes(32, 224, 224, 64) > 1
    assert oracle.bias_relu_bwd_geometry(8 * 112 * 112, 64)[0] > 1
    assert oracle.pool_bwd_geometry(8, 112, 112, 64)[0] > 1
    assert oracle.bias_relu_fwd_passes(1, 8) == 1 and oracle.bias_relu_bwd_geometry(1, 2048) == (1, 3)


# ---- host-side guards ----------------------------------------------------------------------------------------------------------
BF16 = 4   # bagua DType code of bf16
A, M = 0x1000, 0x1008   # aligned / 8 bytes off 16-byte alignment


def _raw_calls(C):
    """(binding, its vector-accessed pointer arguments in check order, call(addresses)) for every raw NHWC binding."""
    ws, out, tk = A, A, A + 4 * 2048
    return [
        ("bias_relu_nhwc_fwd", ("y", "bias"), lambda p: C.bias_relu_nhwc_fwd(p["y"], p["bias"], 4, 8, BF16, 0)),
        ("bias_relu_nhwc_bwd", ("g", "y", "gout"), lambda p: C.bias_relu_nhwc_bwd(p["g"], p["y"], p["gout"], A, 4, 8, BF16, 0)),
        ("bias_relu_nhwc_bwd_fin", ("g", "y", "gout"), lambda p: C.bias_relu_nhwc_bwd_fin(p["g"], p["y"], p["gout"], ws, out, tk, 4, 8, BF16, 0)),
        ("bias_relu_pool_nhwc_fwd", ("x", "bias", "out", "idx"),
         lambda p: C.bias_relu_pool_nhwc_fwd(p["x"], p["bias"], p["out"], p["idx"], 1, 2, 2, 8, BF16, 0)),
        ("bias_relu_pool_nhwc_bwd", ("g", "out", "idx", "gin"),
         lambda p: C.bias_relu_pool_nhwc_bwd(p["g"], p["out"], p["idx"], p["gin"], A, 1, 2, 2, 8, BF16, 0)),
        ("bias_relu_pool_nhwc_bwd_fin", ("g", "out", "idx", "gin"),
         lambda p: C.bias_relu_pool_nhwc_bwd_fin(p["g"], p["out"], p["idx"], p["gin"], ws, out, tk, 1, 2, 2, 8, BF16, 0)),
    ]


def test_raw_bindings_reject_misaligned_pointers_by_name():
    """Every vector-accessed pointer of every binding, 8 bytes off (the argmax bytes 4 bytes off): RuntimeError naming it,
    nothing launched. Integer addresses: the check runs before any CUDA call, so no device is needed."""
    from bagua_b200.core import native

    C = native()
    n0 = C.launch_count()
    for name, args, call in _raw_calls(C):
        for bad in args:
            ptrs = {a: A for a in args}
            ptrs[bad] = A + 4 if bad == "idx" else M
            with pytest.raises(RuntimeError, match=rf"{name.replace('_fin', '')}: `{bad}` must be {8 if bad == 'idx' else 16}-byte aligned"):
                call(ptrs)
    assert C.launch_count() == n0


def test_pool_argmax_bytes_need_only_8_byte_alignment():
    """idx at an 8-byte boundary passes its check: the error names `gin`, which the backward checks after `idx`."""
    from bagua_b200.core import native

    C = native()
    n0 = C.launch_count()
    with pytest.raises(RuntimeError, match="`gin` must be 16-byte aligned"):
        C.bias_relu_pool_nhwc_bwd(A, A, A + 8, M, A, 1, 2, 2, 8, BF16, 0)
    assert C.launch_count() == n0


@pytest.mark.parametrize("offset", [2, 4, 6])
def test_views_off_16_byte_alignment_are_not_given_to_the_kernels(offset):
    """Channels_last views and bias views at 2, 4 and 6 elements (4, 8, 12 bytes) into a buffer: the alignment predicate of
    fused_supported rejects the activation, the bias is re-aligned by a copy whose gradient reaches the view."""
    from bagua_b200.ops import nhwc

    base = torch.zeros(8 + 2 * 16 * 4 * 4, dtype=torch.bfloat16)
    assert base.data_ptr() % 16 == 0
    x = base[offset:offset + 2 * 16 * 4 * 4].view(2, 4, 4, 16).permute(0, 3, 1, 2)
    assert x.is_contiguous(memory_format=torch.channels_last)
    assert not nhwc._aligned(x)
    assert nhwc._aligned(base[8:].view(2, 4, 4, 16).permute(0, 3, 1, 2))
    flat = torch.randn(10 + 16 + offset, dtype=torch.bfloat16).requires_grad_(True)
    bias = flat[offset:offset + 16]
    assert not nhwc._aligned(bias)
    kb = nhwc._kernel_bias(bias)
    assert nhwc._aligned(kb) and kb.is_contiguous() and torch.equal(kb, bias)
    kb.float().sum().backward()
    assert torch.equal(flat.grad[offset:offset + 16], torch.ones(16, dtype=torch.bfloat16))
    strided = torch.zeros(32, dtype=torch.bfloat16)[::2]
    assert nhwc._kernel_bias(strided).is_contiguous()
    aligned = torch.zeros(16, dtype=torch.bfloat16)
    assert nhwc._kernel_bias(aligned) is aligned
