"""GPU tests of kernels added after the last hardware session (they sort last on purpose: the round-end run uses ``-x``, and
a surprise here must not hide the results of the validated suites).  Same oracle rule as test_kernels_gpu.py: compare
against a plain fp32 PyTorch implementation of the same op."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def test_fused_adam_mixed_precision_multi_tensor(dev):
    """bf16 parameters that are not bucket-flattened: fp32 moments + fp32 master weights in the multi-tensor kernel."""
    from bagua_b200.ops.optim import FusedAdam

    torch.manual_seed(9)
    ps = [torch.nn.Parameter((torch.randn(s, device=dev) * 0.1).to(torch.bfloat16)) for s in [(65, 33), (1000,), (7, 9, 11)]]
    rs = [torch.nn.Parameter(p.detach().float().clone()) for p in ps]
    opt, ropt = FusedAdam(ps, lr=1e-3, adamw=True, weight_decay=0.01), torch.optim.AdamW(rs, lr=1e-3, weight_decay=0.01)
    for _ in range(20):
        for p, r in zip(ps, rs):
            g = torch.randn_like(r)
            p.grad, r.grad = g.to(torch.bfloat16), g.to(torch.bfloat16).float()
        opt.step()
        ropt.step()
    for p, r in zip(ps, rs):
        assert opt.state[p]["exp_avg"].dtype == torch.float32 and "master" in opt.state[p]
        torch.testing.assert_close(opt.state[p]["master"], r.data, rtol=1e-4, atol=1e-5)   # fp32 trajectory is preserved
        torch.testing.assert_close(p.data.float(), r.data, rtol=0, atol=8e-3)              # parameter = rounded master


@pytest.mark.skipif(__import__("os").environ.get("BAGUA_EXPERIMENTAL") != "1", reason="in-kernel bias-gradient finish: opt-in until validated on hardware")
def test_nhwc_backward_with_in_kernel_bias_grad_finish(dev, monkeypatch):
    """BAGUA_NHWC_FINALIZE=1 (last CTA converts the fp32 sums, workspace handed back zeroed) must equal the fill + kernel + cast path,
    repeatedly on the same stream (the workspace is reused without clearing)."""
    from bagua_b200.ops.nhwc import bias_relu, bias_relu_maxpool2

    torch.manual_seed(4)
    for C, H in [(64, 56), (512, 14), (2048, 4)]:
        x = torch.randn(8, C, H, H, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        b = torch.randn(C, device=dev).to(torch.bfloat16)
        for fn in (bias_relu, bias_relu_maxpool2):
            res = []
            for fin in ("0", "1", "1"):
                monkeypatch.setenv("BAGUA_NHWC_FINALIZE", fin)
                xi, bi = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
                out = fn(xi * 1.0, bi)
                out.float().pow(2).sum().backward()
                res.append((out.detach().float(), xi.grad.float(), bi.grad.float()))
            for other in res[1:]:
                for a, c in zip(res[0], other):
                    torch.testing.assert_close(a, c, rtol=2e-2, atol=2e-2 * max(1.0, a.abs().max().item()))


@pytest.mark.skipif(__import__("os").environ.get("BAGUA_EXPERIMENTAL") != "1", reason="C++ autograd Functions of the NHWC epilogues: opt-in until validated on hardware")
def test_native_nhwc_functions_match_python_functions(dev, monkeypatch):
    """BAGUA_NATIVE_NHWC=1 routes bias_relu / bias_relu_maxpool2 through the C++ autograd Functions of _C_torch.so (same kernels):
    outputs, input gradients and bias gradients must be identical to the Python Functions, with and without the in-kernel finish."""
    from bagua_b200 import _build
    from bagua_b200.models import vgg16
    from bagua_b200.ops import nhwc

    _build.build_torch_hooks()
    torch.manual_seed(6)
    x = torch.randn(4, 3, 64, 64, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    model = vgg16(num_classes=10).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    results = []
    for native, fin in (("0", "0"), ("1", "0"), ("1", "1")):
        monkeypatch.setenv("BAGUA_NATIVE_NHWC", native)
        monkeypatch.setenv("BAGUA_NHWC_FINALIZE", fin)
        nhwc._native_fns[0] = False                      # re-read the switches
        model.zero_grad(set_to_none=True)
        out = model(x)
        out.float().pow(2).sum().backward()
        assert (nhwc._native_functions() is not None) == (native == "1")
        results.append([out.detach().float()] + [p.grad.float().clone() for p in model.parameters()])
    for other in results[1:]:
        for a, b in zip(results[0], other):
            torch.testing.assert_close(a, b, rtol=2e-2, atol=2e-2 * max(1.0, a.abs().max().item()))
    nhwc._native_fns[0] = False


@pytest.mark.skipif(__import__("os").environ.get("BAGUA_EXPERIMENTAL") != "1", reason="CUDA-graph step capture: opt-in until validated on hardware")
def test_graphed_train_step_matches_eager_steps():
    """utils.graph.GraphedTrainStep (one-rank with_bagua model, FusedSGD with momentum, fused NHWC epilogues) — separate interpreter so
    a capture failure cannot poison this process's CUDA context."""
    import os
    import subprocess
    import sys

    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r'''
import os, sys, copy, torch
import torch.nn.functional as F
sys.path.insert(0, %r)
import bagua_b200 as bagua
from bagua_b200.env import find_free_network_port
from bagua_b200.models import vgg16
from bagua_b200.ops.optim import FusedSGD
from bagua_b200.parallel.algorithms import gradient_allreduce
from bagua_b200.utils.graph import GraphedTrainStep
os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", str(find_free_network_port()))
torch.cuda.set_device(0); dev = torch.device("cuda", 0)
bagua.init_process_group()
torch.backends.cudnn.benchmark = False
torch.manual_seed(0)
base = vgg16(num_classes=10, dropout=0.0).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
def make(tag):
    m = copy.deepcopy(base)
    opt = FusedSGD(m.parameters(), lr=0.01, momentum=0.9)
    m = m.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
    def step(x, y):
        opt.zero_grad()
        loss = F.cross_entropy(m(x).float(), y)
        loss.backward()
        opt.step()
        return loss
    return m, opt, step
batches = [(torch.randn(4, 3, 64, 64, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last), torch.randint(0, 10, (4,), device=dev)) for _ in range(6)]
m1, o1, eager = make("eager")
m2, o2, step2 = make("graphed")
g = GraphedTrainStep(m2, step2, batches[0], optimizers=[o2], warmup=3)
for _ in range(3):                      # the capture warms up with three real steps on batch 0: mirror them
    eager(*batches[0])
losses = []
for x, y in batches[:4]:
    le = eager(x, y)
    lg = g(x, y).clone()
    losses.append((float(le), float(lg)))
torch.cuda.synchronize()
for le, lg in losses:
    assert abs(le - lg) <= 2e-2 * max(1.0, abs(le)), losses
for p, q in zip(m1.parameters(), m2.parameters()):
    assert torch.allclose(p.float(), q.float(), rtol=2e-2, atol=2e-2)
assert g.captures == 1 and g.replays == 4
o2.param_groups[0]["lr"] = 0.005             # a schedule step → re-capture
g(*batches[4]); torch.cuda.synchronize()
assert g.captures == 2 and torch.isfinite(g.static_loss).item()
print("GRAPH_OK", losses)
''' % repo
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "GRAPH_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
