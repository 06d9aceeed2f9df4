"""Single-GPU numerics of the sm_90a kernels against plain PyTorch fp32 references."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n_chunks", [1, 8])
def test_minmax_uint8_roundtrip_matches_oracle(dev, dtype, n_chunks):
    from bagua_b200.ops import quant

    torch.manual_seed(0)
    x = (torch.randn(n_chunks * 4096 + 0, device=dev) * 3).to(dtype)
    buf = quant.compress(x, n_chunks)
    ref = quant.torch_compress(x, n_chunks)
    # identical wire bytes (header + payload); allow off-by-one levels from fp contraction differences
    diff = (buf.int() - ref.int()).abs()
    assert diff.max().item() <= 1
    assert (diff > 0).float().mean().item() < 1e-3
    out = torch.empty_like(x)
    quant.decompress(buf, out, n_chunks)
    ref_out = quant.torch_decompress(buf, x.numel(), n_chunks, dtype)
    # the kernel decodes with (q + lower) * (1/scale), the oracle with a division: at most one fp32 ulp apart, which can move a value
    # across a 16-bit rounding boundary for one level of one chunk in a few hundred (tests/test_quant_emulation.py) — allow one ulp of
    # the output dtype on a handful of elements, nothing beyond that
    diff = (out.float() - ref_out.float()).abs()
    ulp = {torch.float32: 2.0 ** -22, torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}[dtype]
    assert diff.max().item() <= ulp * ref_out.float().abs().max().item() + 1e-6
    assert (diff > 1e-3 + 1e-3 * ref_out.float().abs()).float().mean().item() < 5e-3
    # quantisation error bound: half a level of the chunk range
    for xc, oc in zip(x.float().chunk(n_chunks), out.float().chunk(n_chunks)):
        step = (xc.max() - xc.min()) / 255.0
        rounding = 0.0 if dtype == torch.float32 else xc.abs().max().item() * (2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11)
        assert (xc - oc).abs().max().item() <= step.item() * 0.51 + rounding


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("momentum,nesterov,wd", [(0.0, False, 0.0), (0.9, False, 1e-4), (0.9, True, 0.0)])
def test_flat_sgd_matches_torch(dev, gdtype, momentum, nesterov, wd):
    from bagua_b200.ops.optim import flat_sgd_

    torch.manual_seed(1)
    n = 100003  # odd size: exercises the scalar tail
    p_ref = torch.randn(n, device=dev)
    p = p_ref.clone()
    ref = torch.nn.Parameter(p_ref.clone())
    opt = torch.optim.SGD([ref], lr=0.1, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    mbuf = torch.zeros(n, device=dev) if momentum else None
    model = torch.empty(n, device=dev, dtype=torch.bfloat16)
    for step in range(3):
        g = torch.randn(n, device=dev).to(gdtype)
        ref.grad = g.float().clone()
        opt.step()
        gk = g.clone()
        flat_sgd_(p, gk, mbuf, lr=0.1, momentum=momentum, nesterov=nesterov, weight_decay=wd, first_step=(step == 0), zero_grad=True, model=model)
        assert gk.abs().max().item() == 0.0  # gradient cleared in the same pass
    torch.testing.assert_close(p, ref.data, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(model.float(), ref.data.to(torch.bfloat16).float(), rtol=0, atol=1e-2)


@pytest.mark.parametrize("adamw", [False, True])
def test_flat_adam_matches_torch(dev, adamw):
    from bagua_b200.ops.optim import flat_adam_

    torch.manual_seed(2)
    n = 65536 + 7
    p = torch.randn(n, device=dev)
    ref = torch.nn.Parameter(p.clone())
    cls = torch.optim.AdamW if adamw else torch.optim.Adam
    opt = cls([ref], lr=1e-2, weight_decay=0.01)
    m1, m2 = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    for step in range(1, 4):
        g = torch.randn(n, device=dev)
        ref.grad = g.clone()
        opt.step()
        flat_adam_(p, g.clone(), m1, m2, lr=1e-2, weight_decay=0.01, step=step, adamw=adamw)
    torch.testing.assert_close(p, ref.data, rtol=2e-5, atol=2e-5)


def test_fused_sgd_optimizer_on_bucketed_model(dev):
    """FusedSGD over a with_bagua model: one flat launch per step, same result as torch.optim.SGD."""
    import os

    import bagua_b200 as bagua
    from bagua_b200.env import find_free_network_port
    from bagua_b200.ops.optim import FusedSGD
    from bagua_b200.parallel.algorithms import gradient_allreduce

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
    if not bagua.is_initialized():
        bagua.init_process_group()
    torch.manual_seed(3)
    net = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 32)).to(dev)
    ref = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 32)).to(dev)
    ref.load_state_dict(net.state_dict())
    opt = FusedSGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    net = net.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    for _ in range(4):
        x = torch.randn(16, 64, device=dev)
        opt.zero_grad()
        ropt.zero_grad()
        net(x).square().mean().backward()
        ref(x).square().mean().backward()
        opt.step()
        ropt.step()
    assert len(opt.flat_segments()) == 1 and opt.kernel_launches == 4
    for a, b in zip(net.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    assert "momentum_buffer" in opt.state[next(iter(net.parameters()))]


def test_multi_tensor_kernels_via_fuse_optimizer(dev):
    from bagua_b200.contrib import fuse_optimizer

    torch.manual_seed(4)
    for cls, kw in [(torch.optim.SGD, dict(lr=0.1, momentum=0.9)), (torch.optim.Adam, dict(lr=1e-2)), (torch.optim.AdamW, dict(lr=1e-2, weight_decay=0.05))]:
        ps = [torch.nn.Parameter(torch.randn(s, device=dev)) for s in [(33, 7), (128,), (5, 5, 5)]]
        rs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
        opt, ropt = fuse_optimizer(cls(ps, **kw), do_flatten=True), cls(rs, **kw)
        for _ in range(3):
            for p, r in zip(ps, rs):
                g = torch.randn_like(p)
                p.grad, r.grad = g.clone(), g.clone()
            opt.fuse_step()
            ropt.step()
        for p, r in zip(ps, rs):
            torch.testing.assert_close(p, r, rtol=2e-5, atol=2e-5)
        assert opt._bagua_fused_count == 1  # one multi-tensor launch for the whole group


def test_async_apply_and_misc_elementwise(dev):
    from bagua_b200.core import dtype_code, native

    C = native()
    s = torch.cuda.current_stream().cuda_stream
    w, red, snap = torch.randn(10001, device=dev), torch.randn(10001, device=dev), torch.randn(10001, device=dev)
    ref = w + red / 4 - snap
    C.async_apply(w.data_ptr(), red.data_ptr(), snap.data_ptr(), w.numel(), dtype_code(w.dtype), 0.25, s)
    torch.testing.assert_close(w, ref)
    data = torch.randn(4, 1000, device=dev)
    ref = data.sum(0) / 4
    C.reduce_chunks(data.data_ptr(), 1000, 4, 2, dtype_code(data.dtype), True, s)
    torch.testing.assert_close(data[2], ref)
    a, b = torch.randn(999, device=dev, dtype=torch.bfloat16), torch.randn(999, device=dev, dtype=torch.bfloat16)
    ref = (0.5 * a.float() + 2.0 * b.float()).to(torch.bfloat16)
    C.axpby(a.data_ptr(), b.data_ptr(), 999, dtype_code(a.dtype), 0.5, 2.0, s)
    torch.testing.assert_close(a, ref)
    m, g = torch.randn(777, device=dev), torch.randn(777, device=dev, dtype=torch.bfloat16)
    ref = 0.9 * m + 0.1 * g.float()
    C.qadam_momentum(m.data_ptr(), g.data_ptr(), dtype_code(g.dtype), 777, 0.9, s)
    torch.testing.assert_close(m, ref)


def test_flagship_smoke(dev):
    import __graft_entry__ as ge

    ge.smoke()


@pytest.mark.parametrize("G,M,N,K", [(1, 128, 128, 64), (2, 256, 384, 192), (4, 1024, 512, 1024), (4, 2048, 1024, 256)])  # last: 256 tiles > 132 SMs
def test_tcgen05_grouped_gemm_matches_fp32_reference(dev, G, M, N, K):
    from bagua_b200.ops.gemm import grouped_gemm_tn, grouped_linear

    torch.manual_seed(5)
    a = (torch.randn(G, M, K, device=dev) * 0.5).to(torch.bfloat16)
    b = (torch.randn(G, N, K, device=dev) * 0.5).to(torch.bfloat16)
    bias = torch.randn(G, N, device=dev).to(torch.bfloat16)
    ref = torch.bmm(a.float(), b.float().transpose(1, 2)) + bias.float().unsqueeze(1)
    out = grouped_gemm_tn(a, b, bias)
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2 * ref.abs().max().item())
    out_gelu = grouped_gemm_tn(a, b, bias, act="gelu")
    torch.testing.assert_close(out_gelu.float(), torch.nn.functional.gelu(ref, approximate="tanh"), rtol=2e-2, atol=2e-2 * ref.abs().max().item())
    # autograd through the three TN GEMMs vs torch
    x = a.clone().requires_grad_(True)
    w = b.clone().requires_grad_(True)
    bb = bias.clone().requires_grad_(True)
    y = grouped_linear(x, w, bb)
    gy = torch.randn_like(y)
    y.backward(gy)
    x2, w2, b2 = a.float().requires_grad_(True), b.float().requires_grad_(True), bias.float().requires_grad_(True)
    (torch.bmm(x2, w2.transpose(1, 2)) + b2.unsqueeze(1)).backward(gy.float())
    for got, want in ((x.grad, x2.grad), (w.grad, w2.grad), (bb.grad, b2.grad)):
        torch.testing.assert_close(got.float(), want, rtol=3e-2, atol=3e-2 * want.abs().max().item())


@pytest.mark.parametrize("C,H,dtype", [pytest.param(C, H, dt, id=f"{C}-{H}" + ("" if dt == torch.bfloat16 else "-fp16"))
                                         for dt in (torch.bfloat16, torch.float16) for C, H in [(64, 16), (128, 12), (512, 8)]])
def test_fused_nhwc_conv_epilogues_match_torch(dev, C, H, dtype):
    from bagua_b200.ops.nhwc import bias_relu, bias_relu_maxpool2

    torch.manual_seed(6)
    for pool in (False, True):
        x = torch.randn(4, C, H, H, device=dev).to(dtype).contiguous(memory_format=torch.channels_last)
        b = torch.randn(C, device=dev).to(dtype)
        gy = None
        outs = []
        for fused in (True, False):
            xi = x.clone().requires_grad_(True)
            bi = b.clone().requires_grad_(True)
            if fused:
                y0 = xi * 1.0  # non-leaf input (the conv output in real use); in-place epilogue is allowed on it
                out = bias_relu_maxpool2(y0, bi) if pool else bias_relu(y0, bi)
            else:
                out = torch.nn.functional.relu(xi.float() + bi.float().view(1, -1, 1, 1))
                out = torch.nn.functional.max_pool2d(out, 2, 2) if pool else out
            if gy is None:
                gy = torch.randn_like(out.float())
            out.backward(gy.to(out.dtype))
            outs.append((out.detach().float(), xi.grad.float(), bi.grad.float()))
        (o1, gx1, gb1), (o2, gx2, gb2) = outs
        torch.testing.assert_close(o1, o2, rtol=1e-2, atol=1e-2)
        torch.testing.assert_close(gx1, gx2, rtol=1e-2, atol=1e-2)
        torch.testing.assert_close(gb1, gb2, rtol=2e-2, atol=2e-2 * max(1.0, gb2.abs().max().item()))


def test_vgg16_fused_path_matches_module_path(dev):
    from bagua_b200.models import vgg16

    for dtype in (torch.bfloat16, torch.float16):
        torch.manual_seed(8)
        m = vgg16(num_classes=10).to(dev).to(dtype).to(memory_format=torch.channels_last).eval()
        x = torch.randn(2, 3, 64, 64, device=dev).to(dtype).contiguous(memory_format=torch.channels_last)
        res = []
        for fuse in (True, False):
            m.fuse_epilogues = fuse
            m.zero_grad()
            out = m(x)
            out.float().sum().backward()
            res.append((out.detach().float(), m.features[0].bias.grad.float().clone(), m.features[28].weight.grad.float().clone()))
        for a, b in zip(*res):
            torch.testing.assert_close(a, b, rtol=5e-2, atol=5e-2 * max(1.0, b.abs().max().item()))


@pytest.mark.parametrize("pool", [False, True])
def test_nhwc_bias_grad_is_reproducible_in_deterministic_mode(dev, pool):
    """Under torch.use_deterministic_algorithms the bias gradient is the same bits on every call and agrees with the kernel's own
    (atomic, order-varying) reduction of the default mode."""
    from bagua_b200.ops.nhwc import bias_relu, bias_relu_maxpool2

    torch.manual_seed(8)
    C, H = 128, 32
    x = torch.randn(8, C, H, H, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    g = torch.randn(8, C, H // 2 if pool else H, H // 2 if pool else H, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    fn = bias_relu_maxpool2 if pool else bias_relu

    def bias_grad():
        b = torch.randn(C, device=dev, generator=torch.Generator(device=dev).manual_seed(3)).to(torch.bfloat16).requires_grad_(True)
        fn(x.clone(), b).backward(g)
        return b.grad.float()

    default = bias_grad()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        runs = [bias_grad() for _ in range(3)]
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(runs[0], r) for r in runs[1:])
    torch.testing.assert_close(runs[0], default, rtol=2e-2, atol=2e-2 * default.abs().max().item())
