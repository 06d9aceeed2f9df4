"""The fused NHWC conv epilogues (csrc/nhwc_fused.cu) against the float64 oracle of tests/nhwc_oracle.py, in bf16 and fp16.

Semantics (details and the summation bound in the oracle's docstring):
* ``y = relu(round_T(x + b))``; ``relu(NaN) = NaN``.
* pool: the window max is taken over the pre-bias x; the argmax is the first maximum in scan order (0,0), (0,1), (1,0),
  (1,1), or the last NaN of the window; ``out = relu(round_T(max + b))``.
* backward: ``g`` is kept where ``!(y <= 0)`` (NaN passes); the pool routes it to the argmax and writes 0 at the other three.
* Tie rule: rounding can make two different x equal after the bias is added. The kernel then routes the gradient to the
  larger x, eager torch (``max_pool2d`` after the bias add) to the first of the tied values.

Every case runs on two data families: *exact* data (small integers, gradients in multiples of 2^-4), where every result,
the bias gradient included, must match bit for bit, and *normal* data, where the bias gradient must stay within the bound that
follows from the kernel's summation tree. Every raw launch must raise ``launch_count()`` by exactly one.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import nhwc_oracle as oracle
from tests.nhwc_oracle import assert_bits, assert_same, cl

pytestmark = pytest.mark.gpu

DTYPES = [pytest.param(torch.bfloat16, id="bf16"), pytest.param(torch.float16, id="fp16")]
FAMILIES = ["exact", "normal"]
GUARD_C = [8, 16, 32, 64, 128, 256, 512, 1024, 2048]     # every C that fused_supported admits
ODD_C = [24, 136, 2040]                                   # C / 8 does not divide 256: raw bindings only
MAX_C = 2048


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def _native():
    from bagua_b200.core import native

    return native()


def _code(dtype):
    from bagua_b200.core import dtype_code

    return dtype_code(dtype)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class launches:
    """Asserts that the block raises the library's launch counter by exactly ``n``."""

    def __init__(self, n):
        self.n = n

    def __enter__(self):
        self.n0 = _native().launch_count()

    def __exit__(self, exc_type, *_):
        if exc_type is None:
            assert _native().launch_count() - self.n0 == self.n


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


# ---- the raw bindings ---------------------------------------------------------------------------------------------------------
def k_bias_relu_fwd(x, b):
    N, C, H, W = x.shape
    y = x.clone()
    with launches(1):
        _native().bias_relu_nhwc_fwd(y.data_ptr(), b.data_ptr(), N * H * W, C, _code(x.dtype), _stream())
    return y


def _new_workspace(dev):
    return torch.zeros(MAX_C + 4, dtype=torch.float32, device=dev)


def _check_workspace_zero(ws):
    torch.cuda.current_stream().synchronize()
    assert not ws.view(torch.int32).any(), "FIN workspace or ticket not handed back zeroed"


def k_bias_relu_bwd(g, y, fin=False, ws=None):
    N, C, H, W = y.shape
    gout = torch.empty_like(g, memory_format=torch.channels_last)
    if fin:
        ws = _new_workspace(y.device) if ws is None else ws
        bias_grad = torch.empty(C, dtype=y.dtype, device=y.device)
        with launches(1):
            _native().bias_relu_nhwc_bwd_fin(g.data_ptr(), y.data_ptr(), gout.data_ptr(), ws.data_ptr(), bias_grad.data_ptr(), ws.data_ptr() + 4 * MAX_C,
                                             N * H * W, C, _code(y.dtype), _stream())
        _check_workspace_zero(ws)
        return gout, bias_grad
    bg = torch.zeros(C, dtype=torch.float32, device=y.device)
    with launches(1):
        _native().bias_relu_nhwc_bwd(g.data_ptr(), y.data_ptr(), gout.data_ptr(), bg.data_ptr(), N * H * W, C, _code(y.dtype), _stream())
    return gout, bg.to(y.dtype)


def k_pool_fwd(x, b):
    N, C, H, W = x.shape
    out = torch.empty((N, C, H // 2, W // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    idx = torch.empty((N, C, H // 2, W // 2), dtype=torch.uint8, device=x.device, memory_format=torch.channels_last)
    with launches(1):
        _native().bias_relu_pool_nhwc_fwd(x.data_ptr(), b.data_ptr(), out.data_ptr(), idx.data_ptr(), N, H, W, C, _code(x.dtype), _stream())
    return out, idx


def k_pool_bwd(g, out, idx, H, W, fin=False, ws=None):
    N, C = out.shape[:2]
    gin = torch.empty((N, C, H, W), dtype=out.dtype, device=out.device, memory_format=torch.channels_last)
    if fin:
        ws = _new_workspace(out.device) if ws is None else ws
        bias_grad = torch.empty(C, dtype=out.dtype, device=out.device)
        with launches(1):
            _native().bias_relu_pool_nhwc_bwd_fin(g.data_ptr(), out.data_ptr(), idx.data_ptr(), gin.data_ptr(), ws.data_ptr(), bias_grad.data_ptr(),
                                                  ws.data_ptr() + 4 * MAX_C, N, H, W, C, _code(out.dtype), _stream())
        _check_workspace_zero(ws)
        return gin, bias_grad
    bg = torch.zeros(C, dtype=torch.float32, device=out.device)
    with launches(1):
        _native().bias_relu_pool_nhwc_bwd(g.data_ptr(), out.data_ptr(), idx.data_ptr(), gin.data_ptr(), bg.data_ptr(), N, H, W, C, _code(out.dtype),
                                          _stream())
    return gin, bg.to(out.dtype)


# ---- one case: kernels vs oracle ------------------------------------------------------------------------------------------------
def check_bias_relu(x, b, g, exact):
    """Forward, then backward plain and with the in-kernel finish, against the oracle."""
    N, C, H, W = x.shape
    y = k_bias_relu_fwd(x, b)
    want_y = oracle.bias_relu_fwd(x, b)
    assert_same(y, want_y, "y")
    want_g, exact_sum, abs_sum = oracle.bias_relu_bwd(g, want_y)
    _, depth = oracle.bias_relu_bwd_geometry(N * H * W, C)
    grads = []
    for fin in (False, True):
        gout, bg = k_bias_relu_bwd(g, y, fin)
        assert_bits(gout, want_g, f"gout (fin={fin})")
        oracle.check_bias_grad(bg, exact_sum, abs_sum, depth, exact, f"bias_grad (fin={fin})")
        grads.append(bg)
    if exact:
        assert_bits(grads[1], grads[0], "FIN vs plain bias_grad")


def check_pool(x, b, g, exact, backward=True):
    N, C, H, W = x.shape
    out, idx = k_pool_fwd(x, b)
    want_out, want_idx = oracle.pool_fwd(x, b)
    assert_same(out, want_out, "out")
    assert idx.is_contiguous(memory_format=torch.channels_last) and torch.equal(idx, want_idx), "idx"
    if not backward:
        return
    want_gin, exact_sum, abs_sum = oracle.pool_bwd(g, want_out, want_idx, H, W)
    _, depth = oracle.pool_bwd_geometry(N, H, W, C)
    grads = []
    for fin in (False, True):
        gin, bg = k_pool_bwd(g, out, idx, H, W, fin)
        assert_bits(gin, want_gin, f"gin (fin={fin})")
        oracle.check_bias_grad(bg, exact_sum, abs_sum, depth, exact, f"bias_grad (fin={fin})")
        grads.append(bg)
    if exact:
        assert_bits(grads[1], grads[0], "FIN vs plain bias_grad")


def _data(shape, dtype, family, dev, seed, gshape=None):
    gen = _gen(dev, seed)
    x, b = oracle.FAMILIES[family](shape, dtype, dev, gen)
    g = oracle.make_grad(gshape or shape, dtype, dev, gen, family == "exact")
    return x, b, g


def _pooled(shape):
    N, C, H, W = shape
    return (N, C, H // 2, W // 2)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("C", GUARD_C)
@pytest.mark.parametrize("NHW", [(1, 1, 1), (3, 5, 7)], ids=["one_row", "ragged_rows_odd_w"])
def test_bias_relu_kernels_match_oracle(dev, dtype, family, C, NHW):
    N, H, W = NHW
    shape = (N, C, H, W)
    check_bias_relu(*_data(shape, dtype, family, dev, C + H), family == "exact")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("C", GUARD_C)
@pytest.mark.parametrize("NHW", [(1, 2, 2), (3, 6, 10)], ids=["one_window", "h_ne_w"])
def test_pool_kernels_match_oracle(dev, dtype, family, C, NHW):
    N, H, W = NHW
    shape = (N, C, H, W)
    check_pool(*_data(shape, dtype, family, dev, C + H, _pooled(shape)), family == "exact")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("C", ODD_C)
def test_channel_counts_outside_the_python_guard(dev, dtype, family, C):
    """C / 8 does not divide 256: bias+ReLU forward / backward and the pool forward are still exact through the raw bindings;
    the pool backward (a thread keeps one channel vector across its grid stride) refuses without launching, and the Python
    front-end does not offer such tensors to the kernels."""
    from bagua_b200.ops.nhwc import fused_supported

    exact = family == "exact"
    shape = (3, C, 6, 10)
    x, b, g = _data(shape, dtype, family, dev, C)
    assert not fused_supported(x, C)
    check_bias_relu(x, b, g, exact)
    check_pool(x, b, None, exact, backward=False)
    out, idx = k_pool_fwd(x, b)
    gp = oracle.make_grad(_pooled(shape), dtype, dev, _gen(dev, 1), exact)
    for fin in (False, True):
        with launches(0), pytest.raises(RuntimeError, match="C/8 to divide 256"):
            k_pool_bwd(gp, out, idx, 6, 10, fin)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("shape", [(8, 64, 112, 112), (32, 64, 224, 224), (4, 2048, 28, 28)], ids=["8x64x112x112", "vgg16_block1", "8x2048x28x28"])
def test_grid_stride_loops_that_wrap(dev, dtype, family, shape):
    """Shapes whose grid-stride loops run several times (the grid is capped at 132 * 8 blocks); the bias gradient of exact data
    catches a row or block that is dropped or counted twice."""
    N, C, H, W = shape
    passes = [oracle.bias_relu_fwd_passes(N * H * W, C), oracle.bias_relu_bwd_geometry(N * H * W, C)[0], oracle.pool_bwd_geometry(N, H, W, C)[0]]
    assert min(passes) > 1 and (shape != (32, 64, 224, 224) or oracle.pool_fwd_passes(N, H, W, C) > 1)
    x, b, g = _data(shape, dtype, family, dev, 7)
    check_bias_relu(x, b, g, family == "exact")
    del g
    gp = oracle.make_grad(_pooled(shape), dtype, dev, _gen(dev, 8), family == "exact")
    check_pool(x, b, gp, family == "exact")


def _special_case(dtype, dev):
    """Exact data with NaN at each window position (two NaNs in one window), a NaN bias, ±inf, a window of -inf, x + b that
    overflows T, subnormals of T and -0."""
    shape = (2, 16, 4, 8)
    x, b, g = _data(shape, dtype, "exact", dev, 11)
    gp = oracle.make_grad(_pooled(shape), dtype, dev, _gen(dev, 12), True)
    nan, inf = float("nan"), float("inf")
    x = x.clone()
    b = b.clone()
    for q, (dy, dx) in enumerate(oracle.WINDOW):   # window (0, q) of channel 0: NaN at position q
        x[0, 0, dy, 2 * q + dx] = nan
    x[0, 0, 2, 1] = nan                             # window (1, 0): NaN at positions 1 and 3 -> argmax 3
    x[0, 0, 3, 1] = nan
    b[1] = nan
    x[1, 2, 0, 0], x[1, 2, 1, 1], x[1, 2, 2, 3] = inf, -inf, -inf
    x[1, 3, 0:2, 0:2] = -inf
    big = torch.finfo(dtype).max
    x[1, 4] = big
    b[4] = big                                      # x + b overflows to +inf in T
    tiny = torch.finfo(dtype).tiny                  # smallest normal: multiples of tiny / 8 are subnormal
    x[1, 5] = torch.randint(-6, 7, (4, 8), generator=_gen(dev, 13), device=dev).to(torch.float64).mul(tiny / 8).to(dtype)
    b[5] = tiny * 3 / 8
    x[1, 6] = -0.0
    b[6] = 0.0
    b[7] = -0.0
    assert (x[1, 5] != 0).any() and (x[1, 5].abs() < tiny).all()
    return cl(x), b, g, gp


@pytest.mark.parametrize("dtype", DTYPES)
def test_special_values(dev, dtype):
    """NaN propagates through both forwards and keeps its gradient in both backwards, with torch's argmax rule; ±inf,
    overflow, subnormals and -0 are exact."""
    x, b, g, gp = _special_case(dtype, dev)
    check_bias_relu(x, b, g, True)
    check_pool(x, b, gp, True)
    out, idx = k_pool_fwd(x, b)
    assert [idx[0, 0, 0, q].item() for q in range(4)] == [0, 1, 2, 3] and idx[0, 0, 1, 0].item() == 3
    assert torch.isnan(out[0, 0, 0]).all() and torch.isnan(out[:, 1]).all()
    assert torch.isinf(k_bias_relu_fwd(x, b)[1, 4]).all()
    # the fused front-ends agree with the unfused torch ops on the forward (NaN where torch has NaN)
    from bagua_b200.ops.nhwc import bias_relu, bias_relu_maxpool2

    assert_same(bias_relu(x.clone(), b), cl(F.relu(x + b.view(1, -1, 1, 1))), "bias_relu vs torch")
    assert_same(bias_relu_maxpool2(x, b), cl(F.max_pool2d(F.relu(x + b.view(1, -1, 1, 1)), 2, 2)), "bias_relu_maxpool2 vs torch")


# ---- the autograd Functions -------------------------------------------------------------------------------------------------
MODES = ["default", "fin", "deterministic", "native", "native_fin"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pool", [False, True], ids=["bias_relu", "bias_relu_maxpool2"])
@pytest.mark.parametrize("mode", MODES)
def test_autograd_functions_match_oracle(dev, dtype, pool, mode, monkeypatch):
    """bias_relu / bias_relu_maxpool2 through the Python autograd Functions (default, in-kernel finish, deterministic) and the
    C++ ones (BAGUA_NATIVE_NHWC, with and without the finish): output, input gradient and bias gradient bit for bit on exact
    data, one forward and one backward launch."""
    from bagua_b200.ops import nhwc

    monkeypatch.setenv("BAGUA_NHWC_FINALIZE", "1" if mode.endswith("fin") else "0")
    monkeypatch.setenv("BAGUA_NATIVE_NHWC", "1" if mode.startswith("native") else "0")
    monkeypatch.setattr(nhwc, "_native_fns", [False])
    if mode.startswith("native"):
        from bagua_b200 import _build

        _build.build_torch_hooks()
        assert nhwc._native_functions() is not None, "C++ autograd Functions unavailable"
    shape = (4, 64, 12, 16)
    x, b, g = _data(shape, dtype, "exact", dev, 21, _pooled(shape) if pool else None)
    xi, bi = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
    torch.use_deterministic_algorithms(mode == "deterministic", warn_only=True)
    try:
        with launches(2):
            out = (nhwc.bias_relu_maxpool2 if pool else nhwc.bias_relu)(xi * 1.0, bi)
            out.backward(g)
    finally:
        torch.use_deterministic_algorithms(False)
    if pool:
        want_out, want_idx = oracle.pool_fwd(x, b)
        want_gx, exact_sum, _ = oracle.pool_bwd(g, want_out, want_idx, shape[2], shape[3])
    else:
        want_out = oracle.bias_relu_fwd(x, b)
        want_gx, exact_sum, _ = oracle.bias_relu_bwd(g, want_out)
    assert_same(out.detach(), want_out, "out")
    assert_bits(xi.grad.contiguous(memory_format=torch.channels_last), want_gx, "x.grad")
    assert_bits(bi.grad, exact_sum.to(dtype), "bias.grad")


@pytest.mark.parametrize("dtype", DTYPES)
def test_fin_workspace_across_channel_counts_and_streams(dev, dtype):
    """One FIN workspace on one stream through launches whose C changes (2048, 8, 512, ...): every result equals the plain
    path's and the workspace and ticket read back zero after each launch. Then two streams, each with its own workspace."""
    ws = _new_workspace(dev)
    for i, C in enumerate([2048, 8, 512, 24, 64, 1024, 16, 2040, 256]):
        shape = (2, C, 6, 10)
        x, b, g = _data(shape, dtype, "exact", dev, 30 + i)
        y = k_bias_relu_fwd(x, b)
        assert_bits(k_bias_relu_bwd(g, y, True, ws)[1], k_bias_relu_bwd(g, y)[1], f"bias_relu C={C}")
        if 256 % (C // 8) == 0:
            out, idx = k_pool_fwd(x, b)
            gp = oracle.make_grad(_pooled(shape), dtype, dev, _gen(dev, 50 + i), True)
            a, want = k_pool_bwd(gp, out, idx, 6, 10, True, ws), k_pool_bwd(gp, out, idx, 6, 10)
            assert_bits(a[0], want[0], f"pool gin C={C}")
            assert_bits(a[1], want[1], f"pool C={C}")

    cases = []
    for i, C in enumerate([512, 64]):
        shape = (16, C, 28, 28)
        x, b, g = _data(shape, dtype, "exact", dev, 60 + i)
        y = k_bias_relu_fwd(x, b)
        cases.append((y, g, k_bias_relu_bwd(g, y)[1]))
    streams = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
    wss = [_new_workspace(dev) for _ in streams]
    results = [None, None]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    n0 = _native().launch_count()
    for rep in range(3):
        for k, (s, w, (y, g, _)) in enumerate(zip(streams, wss, cases)):
            with torch.cuda.stream(s):
                gout = torch.empty_like(g)
                bg = torch.empty(y.shape[1], dtype=dtype, device=dev)
                _native().bias_relu_nhwc_bwd_fin(g.data_ptr(), y.data_ptr(), gout.data_ptr(), w.data_ptr(), bg.data_ptr(), w.data_ptr() + 4 * MAX_C,
                                                 y.shape[0] * y.shape[2] * y.shape[3], y.shape[1], _code(dtype), s.cuda_stream)
                results[k] = bg
    torch.cuda.synchronize()
    assert _native().launch_count() - n0 == 6
    for (y, g, want), got, w in zip(cases, results, wss):
        assert_bits(got, want, "two streams")
        assert not w.view(torch.int32).any()


# ---- guards in front of the kernels ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_guard_rejections_launch_nothing(dev, dtype):
    """Tensors the kernels do not take go to torch without a launch: fp32, C / 8 not dividing 256, an activation at element
    offsets 2, 4 and 6 (not 16-byte aligned); the same activation at offset 8 is taken."""
    from bagua_b200.ops.nhwc import bias_relu, fused_supported

    shape = (2, 64, 6, 10)
    x, b, _ = _data(shape, dtype, "exact", dev, 70)
    with launches(0):
        out = bias_relu(x.float(), b.float())
    assert_same(out, F.relu(x.float() + b.float().view(1, -1, 1, 1)))
    x24, b24, _ = _data((2, 24, 6, 10), dtype, "exact", dev, 71)
    with launches(0):
        out = bias_relu(x24.clone(), b24)
    assert_same(out, F.relu(x24 + b24.view(1, -1, 1, 1)))
    n = x.numel()
    base = torch.zeros(8 + n, dtype=dtype, device=dev)
    for off in (2, 4, 6, 8):
        v = base[off:off + n].view(2, 6, 10, 64).permute(0, 3, 1, 2)
        v.copy_(x)
        assert v.is_contiguous(memory_format=torch.channels_last) and fused_supported(v, 64) == (off == 8)
        with launches(1 if off == 8 else 0):
            out = bias_relu(v, b)
        assert_same(out, cl(F.relu(x + b.view(1, -1, 1, 1))), f"offset {off}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pool", [False, True], ids=["bias_relu", "bias_relu_maxpool2"])
def test_misaligned_bias_view_is_realigned(dev, dtype, pool):
    """A bias that is a view at element offset 2 of a larger tensor (4 bytes off 16-byte alignment) is copied to an aligned
    buffer: still the fused kernels (one forward, one backward launch), results equal eager torch, gradient lands in the view."""
    from bagua_b200.ops.nhwc import bias_relu, bias_relu_maxpool2

    shape = (4, 64, 12, 16)
    x, b, g = _data(shape, dtype, "exact", dev, 80, _pooled(shape) if pool else None)
    grads, outs = [], []
    for fused in (True, False):
        flat = torch.zeros(2 + 64 + 6, dtype=dtype, device=dev)
        flat[2:66] = b
        flat.requires_grad_(True)
        bias = flat[2:66]
        assert bias.data_ptr() % 16 == 4
        xi = x.clone().requires_grad_(True)
        with launches(2 if fused else 0):
            if fused:
                out = (bias_relu_maxpool2 if pool else bias_relu)(xi * 1.0, bias)
            else:
                out = F.relu(xi + bias.view(1, -1, 1, 1))
                out = F.max_pool2d(out, 2, 2) if pool else out
            out.backward(g)
        outs.append(out.detach())
        grads.append((xi.grad, flat.grad))
    assert_same(outs[0], cl(outs[1]), "out")
    assert_bits(grads[0][0].contiguous(memory_format=torch.channels_last), grads[1][0].contiguous(memory_format=torch.channels_last), "x.grad")
    assert_bits(grads[0][1], grads[1][1], "bias grad in the flat tensor")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pool", [False, True], ids=["conv_relu", "conv_relu_pool"])
def test_conv_bias_packed_after_a_10_element_tensor(dev, dtype, pool):
    """A conv bias placed right after a 10-element tensor in one flat storage, as a bucket packs parameters back to back
    (20 bytes in: 4 bytes off 16-byte alignment). conv_bias_relu still takes the fused epilogue and equals the module path:
    integer inputs and weights keep the convolution exact, so the outputs match bit for bit and the fused bias gradient is the
    exact sum of the masked gradient."""
    import copy

    from bagua_b200.ops.nhwc import conv_bias_relu

    gen = _gen(dev, 90)
    conv = torch.nn.Conv2d(16, 64, 3, padding=1).to(dev)
    with torch.no_grad():
        conv.weight.copy_(torch.randint(-1, 2, conv.weight.shape, generator=gen, device=dev))
        conv.bias.copy_(torch.randint(-4, 5, (64,), generator=gen, device=dev))
    conv = conv.to(dtype).to(memory_format=torch.channels_last)
    ref = copy.deepcopy(conv)
    flat = torch.zeros(10 + 64, dtype=dtype, device=dev)
    flat[10:] = conv.bias.detach()
    conv.bias.data = torch.empty(0, dtype=dtype, device=dev).set_(flat.untyped_storage(), 10, (64,), (1,))
    assert conv.bias.data_ptr() % 16 == 4 and conv.bias.is_leaf
    x = cl(torch.randint(-1, 2, (4, 16, 12, 16), generator=gen, device=dev).to(dtype))
    g = oracle.make_grad((4, 64, 6, 8) if pool else (4, 64, 12, 16), dtype, dev, gen, True)
    res = []
    for m, fused in ((conv, True), (ref, False)):
        xi = x.clone().requires_grad_(True)
        with launches(2 if fused else 0):
            if fused:
                out = conv_bias_relu(xi, m, pool)
            else:
                out = F.relu(m(xi))
                out = F.max_pool2d(out, 2, 2) if pool else out
            out.backward(g)
        res.append((out.detach(), xi.grad, m.weight.grad, m.bias.grad))
    (o1, gx1, gw1, gb1), (o2, gx2, gw2, gb2) = res
    assert_same(o1, cl(o2), "out")
    assert_same(gb1, torch.where(o2 <= 0, torch.zeros_like(g), g).double().sum((0, 2, 3)).to(dtype), "bias grad")
    torch.testing.assert_close(gb2.float(), gb1.float(), rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(gx1.float(), gx2.float(), rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(gw1.float(), gw2.float(), rtol=1e-2, atol=1e-2)
