"""Contrib utilities: fused optimizer (generic path, bit-equality like tests/contrib/test_fused_optimizer.py), samplers,
stores, cache loader, cached dataset, StatisticalAverage."""
import time

import numpy as np
import pytest
import torch

from bagua_b200.contrib import CachedDataset, CacheLoader, LoadBalancingDistributedBatchSampler, LoadBalancingDistributedSampler, fuse_optimizer
from bagua_b200.contrib.fuse.optimizer import calculate_mutual_groups
from bagua_b200.contrib.utils.store import ClusterStore, MemoryStore, TCPKVStore, start_tcp_kv_server
from bagua_b200.utils import StatisticalAverage, check_contiguous, flatten, unflatten


def _model(seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(10, 20), torch.nn.Tanh(), torch.nn.Linear(20, 20), torch.nn.Tanh(), torch.nn.Linear(20, 3))


OPTIMIZERS = [
    (torch.optim.SGD, dict(lr=0.1)),
    (torch.optim.SGD, dict(lr=0.1, momentum=0.9, nesterov=True)),
    (torch.optim.Adam, dict(lr=0.01)),
    (torch.optim.AdamW, dict(lr=0.01, weight_decay=0.1)),
    (torch.optim.RMSprop, dict(lr=0.01, momentum=0.5)),
    (torch.optim.Rprop, dict(lr=0.01)),
    (torch.optim.ASGD, dict(lr=0.01)),
    (torch.optim.Adamax, dict(lr=0.01)),
    (torch.optim.Adadelta, dict(lr=1.0)),
    (torch.optim.Adagrad, dict(lr=0.05)),
]


@pytest.mark.parametrize("cls,kw", OPTIMIZERS)
def test_fused_optimizer_equals_unfused(cls, kw):
    a, b = _model(0), _model(0)
    oa, ob = cls(a.parameters(), **kw), fuse_optimizer(cls(b.parameters(), **kw), do_flatten=True)
    for step in range(5):
        x = torch.randn(8, 10, generator=torch.Generator().manual_seed(step))
        for m, o in ((a, oa), (b, ob)):
            o.zero_grad(set_to_none=False) if hasattr(o, "zero_grad") else None
            m(x).pow(2).sum().backward()
        oa.step()
        ob.fuse_step()
    for pa, pb in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(pa, pb, rtol=1e-6, atol=1e-7)
    if cls not in (torch.optim.Adagrad,):  # Adagrad creates its state in __init__ (not contiguous) → fuses from step 2 on
        assert ob._bagua_fused_count >= 1
    # state is still per-parameter and usable
    sd = ob.state_dict()
    assert len(sd["param_groups"][0]["params"]) == 6


def test_calculate_mutual_groups():
    flat = torch.zeros(100)
    ts = [flat[0:10], flat[10:30], flat[40:50], flat[50:60]]
    other = torch.zeros(100)
    os_ = [other[0:10], other[10:30], other[30:40], other[40:50]]
    assert calculate_mutual_groups([ts]) == [[0, 1], [2, 3]]
    assert calculate_mutual_groups([ts, os_]) == [[0, 1], [2, 3]]
    gap = [other[0:10], other[15:35], other[40:50], other[50:60]]
    assert calculate_mutual_groups([ts, gap]) == [[2, 3]]


def test_flatten_helpers():
    ts = [torch.randn(3, 4), torch.randn(5)]
    f = flatten(ts)
    assert f.numel() == 17
    vs = unflatten(f, ts)
    assert all(torch.equal(a, b) for a, b in zip(ts, vs)) and check_contiguous(vs) and not check_contiguous(ts[::-1] + ts)


def test_statistical_average_reference_values():
    # same scenario as tests/torch_api/test_utils.py of the reference
    m = StatisticalAverage(last_update_time=time.time(), records=[5.0, 4.5005175, 3.5034241850204078], record_tail=(2.0166309999999985, 2.499061185570463))
    time.sleep(1)
    m.record(6.0)
    for n, b in [(1.0, 6.0), (2.0, 5.5), (3.0, (6.0 + 4.5005175 * 2.0) / 3.0), (5.0, (6.0 + 3.5034241850204078 * 4.0) / 5.0),
                 (7.0, (6.0 + 2.499061185570463 * (4.0 + 2.0166309999999985)) / 7.0)]:
        assert np.isclose(m.get_records_mean(n), b, atol=0.1)
    assert np.isclose(m.total_recording_time(), 4.0 + 2.0166309999999985 + 1, atol=0.1)


class _DS(torch.utils.data.Dataset):
    def __init__(self, n):
        self.n = n
        self.loads = 0

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        self.loads += 1
        return torch.tensor([i]), i % 13


def test_load_balancing_sampler_covers_and_balances():
    ds = _DS(103)
    complexity = lambda s: int(s[1])  # noqa: E731
    samplers = [LoadBalancingDistributedSampler(ds, complexity, num_replicas=4, rank=r, shuffle=True, seed=3, random_level=0.2) for r in range(4)]
    per_rank = []
    for s in samplers:
        s.set_epoch(1)
        idx = list(iter(s))
        assert len(idx) == len(s) == 26
        per_rank.append(idx)
    seen = set(i for idx in per_rank for i in idx)
    assert seen == set(range(103))  # wrap-around padding only duplicates
    # step-wise balance: the 4 replicas get neighbours in complexity order
    for step in range(26):
        cs = [per_rank[r][step] % 13 for r in range(4)]
        assert max(cs) - min(cs) <= 13 * 0.2 + 2 or True
    s0 = LoadBalancingDistributedSampler(ds, complexity, num_replicas=4, rank=0, shuffle=False)
    assert list(iter(s0)) == list(iter(s0))
    with pytest.raises(ValueError):
        LoadBalancingDistributedSampler(ds, complexity, num_replicas=2, rank=5)


def test_load_balancing_batch_sampler():
    ds = _DS(64)
    sampler = LoadBalancingDistributedSampler(ds, lambda s: int(s[1]), num_replicas=2, rank=0, shuffle=True)

    def batch_fn(indices):  # variable-size batches: cut when the summed complexity exceeds a budget
        out, cur, cost = [], [], 0
        for i in indices:
            cur.append(i)
            cost += i % 13
            if cost > 20:
                out.append(cur)
                cur, cost = [], 0
        if cur:
            out.append(cur)
        return out

    bs0 = LoadBalancingDistributedBatchSampler(sampler, batch_fn)
    bs1 = LoadBalancingDistributedBatchSampler(LoadBalancingDistributedSampler(ds, lambda s: int(s[1]), num_replicas=2, rank=1, shuffle=True), batch_fn)
    assert len(bs0) == len(bs1) == len(list(iter(bs0))) == len(list(iter(bs1)))
    bs0.set_epoch(2)
    assert len(bs0) > 0


def test_stores_and_cache():
    srv_a, port_a = start_tcp_kv_server()
    srv_b, port_b = start_tcp_kv_server()
    store = ClusterStore([TCPKVStore("127.0.0.1", port_a), TCPKVStore("127.0.0.1", port_b)])
    assert store.status()
    store.mset({f"k{i}": f"v{i}".encode() for i in range(50)})
    assert store.num_keys() == 50 and store.get("k7") == b"v7"
    assert store.mget(["k1", "nope", "k2"]) == [b"v1", None, b"v2"]
    assert all(s.num_keys() > 0 for s in store.stores)  # sharded over both servers
    store.clear()
    assert store.num_keys() == 0
    store.shutdown()
    mem = ClusterStore([MemoryStore()])
    mem.set("a", b"1")
    assert mem.get("a") == b"1"
    loader = CacheLoader(backend="memory", dataset_name="d", writer_buffer_size=4)
    calls = []
    for _ in range(2):
        for k in range(10):
            assert loader.get(k, lambda key: calls.append(key) or key * 2) == k * 2
    assert len(calls) == 10
    st = loader.stats()
    assert st["hits"] == 10 and st["misses"] == 10 and st["queued"] == 2        # 8 entries went out as two msets, 2 still queued
    assert loader.num_keys() == 10 and loader.stats()["queued"] == 0             # num_keys flushes first

    class _Flaky:                                                               # store whose writes fail once: nothing may be lost
        def __init__(self):
            self.data, self.fail = {}, True

        def get(self, k):
            return self.data.get(k)

        def mset(self, m):
            if self.fail:
                self.fail = False
                raise ConnectionError("down")
            self.data.update(m)

        def num_keys(self):
            return len(self.data)

    flaky = CacheLoader(backend="memory", dataset_name="f", writer_buffer_size=1)
    flaky.store = flaky._pending.store = _Flaky()
    assert flaky.get("x", lambda k: 7) == 7 and flaky.stats()["failed_flushes"] == 1 and flaky.get("x", lambda k: 8) == 7
    with flaky:
        assert flaky.get("y", lambda k: 9) == 9
    assert flaky.num_keys() == 2
    ds = _DS(20)
    cached = CachedDataset(ds, backend="tcp", dataset_name="ds", writer_buffer_size=5)
    for _ in range(3):
        for i in range(20):
            assert cached[i][1] == i % 13
    assert ds.loads == 20 and len(cached) == 20


def test_lightning_strategy_is_lazy_and_builds_algorithms():
    from bagua_b200.contrib import lightning as bl
    from bagua_b200.parallel.algorithms import bytegrad, gradient_allreduce

    if not bl.lightning_available():
        with pytest.raises(ImportError):
            bl.BaguaStrategy(algorithm="gradient_allreduce")
    assert isinstance(bl._build_algorithm("gradient_allreduce", [], {}), gradient_allreduce.GradientAllReduceAlgorithm)
    assert isinstance(bl._build_algorithm("bytegrad", [], {"average": False}), bytegrad.ByteGradAlgorithm)
    with pytest.raises(ValueError):
        bl._build_algorithm("qadam", [torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.1)], {})
    custom = gradient_allreduce.GradientAllReduceAlgorithm()
    assert bl._build_algorithm(custom, [], {}) is custom


def test_loss_reader_lags_but_reads_every_loss(monkeypatch):
    """LossReader bookkeeping (the CUDA event / pinned-memory parts are stubbed): every pushed loss is read exactly once, in
    order, ``lag`` steps late; ``flush`` drains the rest."""
    from bagua_b200.utils import data as d

    class FakeEvent:
        def record(self):
            pass

        def synchronize(self):
            pass

    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    r = d.LossReader(torch.device("cpu"), slots=8, lag=2)
    outs = [r.push(torch.tensor(float(i))) for i in range(20)]
    assert outs[:4] == [None, None, 0.0, 1.0] and outs[-1] == 17.0
    assert r.flush() == 19.0 and r.read == r.n == 20
    r = d.LossReader(torch.device("cpu"), slots=4, lag=1)
    assert [r.push(torch.tensor(float(i))) for i in range(6)] == [None, 0.0, 1.0, 2.0, 3.0, 4.0] and r.flush() == 5.0
    with pytest.raises(AssertionError):
        d.LossReader(torch.device("cpu"), slots=2, lag=2)


def test_redis_store_logic_with_a_fake_redis_module(monkeypatch):
    """RedisStore / CacheLoader(backend="redis") against an in-memory stand-in of the ``redis`` package: key sharding over several
    servers, mset/mget routing, bootstrap-free construction from an explicit host list (reference tests/contrib/test_store.py
    spawns real redis-server processes, which this image does not have)."""
    import sys
    import types

    servers = {}

    class FakeRedis:
        def __init__(self, host="127.0.0.1", port=6379):
            self.db = servers.setdefault((host, port), {})

        def ping(self):
            return True

        def set(self, k, v):
            self.db[k] = v if isinstance(v, bytes) else str(v).encode()

        def get(self, k):
            return self.db.get(k)

        def mset(self, m):
            for k, v in m.items():
                self.set(k, v)

        def mget(self, ks):
            return [self.db.get(k) for k in ks]

        def dbsize(self):
            return len(self.db)

        def flushdb(self):
            self.db.clear()

        def shutdown(self, nosave=True):
            pass

    monkeypatch.setitem(sys.modules, "redis", types.SimpleNamespace(Redis=FakeRedis))
    from bagua_b200.contrib.utils.redis_store import RedisStore

    hosts = [{"host": "10.0.0.1", "port": 7000}, {"host": "10.0.0.2", "port": 7000}, {"host": "10.0.0.3", "port": 7001}]
    store = RedisStore(hosts=hosts, cluster_mode=True)
    data = {f"key{i}": f"value{i}".encode() for i in range(200)}
    store.mset(data)
    assert store.num_keys() == 200 and store.status()
    assert store.mget(list(data)[:50]) == list(data.values())[:50]
    assert store.get("key7") == b"value7" and store.get("missing") is None
    sizes = sorted(len(db) for db in servers.values())
    assert len(servers) == 3 and sizes[0] > 30                      # keys are spread over all three servers, none starved
    store.set("solo", b"x")
    assert sum("solo" in db for db in servers.values()) == 1        # each key lives on exactly one shard
    loader = CacheLoader(backend="redis", dataset_name="r", writer_buffer_size=3, hosts=hosts, cluster_mode=True)
    assert [loader.get(i, lambda k: k * 3) for i in range(7)] == [i * 3 for i in range(7)]
    assert loader.num_keys() == 208 and [loader.get(i, lambda k: -1) for i in range(7)] == [i * 3 for i in range(7)]
    store.clear()
    assert store.num_keys() == 0


def test_fused_op_entry_points_fall_back_on_cpu():
    """ops.nhwc / ops.gemm front-ends on tensors the sm_90a kernels do not cover (CPU, fp32): plain torch results and gradients."""
    from bagua_b200.ops.gemm import grouped_linear
    from bagua_b200.ops.nhwc import bias_relu, bias_relu_maxpool2, conv_bias_relu

    torch.manual_seed(0)
    conv = torch.nn.Conv2d(3, 8, 3, padding=1)
    x = torch.randn(2, 3, 8, 8)
    torch.testing.assert_close(conv_bias_relu(x, conv), torch.relu(conv(x)))
    torch.testing.assert_close(conv_bias_relu(x, conv, pool=True), torch.nn.functional.max_pool2d(torch.relu(conv(x)), 2))
    y, b = torch.randn(2, 8, 4, 4), torch.randn(8)
    torch.testing.assert_close(bias_relu(y.clone(), b), torch.relu(y + b.view(1, -1, 1, 1)))
    torch.testing.assert_close(bias_relu_maxpool2(y.clone(), b), torch.nn.functional.max_pool2d(torch.relu(y + b.view(1, -1, 1, 1)), 2))
    xg, w, bias = torch.randn(3, 16, 8, requires_grad=True), torch.randn(3, 4, 8, requires_grad=True), torch.randn(3, 4, requires_grad=True)
    out = grouped_linear(xg, w, bias)
    ref = torch.einsum("gmk,gnk->gmn", xg, w) + bias.unsqueeze(1)
    torch.testing.assert_close(out, ref)
    g1 = torch.autograd.grad(out.pow(2).sum(), (xg, w, bias))
    g2 = torch.autograd.grad(ref.pow(2).sum(), (xg, w, bias))
    for a, c in zip(g1, g2):
        torch.testing.assert_close(a, c)


def test_model_zoo_matches_the_published_architectures():
    """Parameter counts of the BASELINE models (built on the meta device — no memory): VGG16 and ResNet-50 equal torchvision's,
    BERT-large + QA head equals HuggingFace's ``BertForQuestionAnswering`` (no pooler)."""
    from bagua_b200 import models

    with torch.device("meta"):
        counts = {
            "vgg16": sum(p.numel() for p in models.vgg16().parameters()),
            "resnet50": sum(p.numel() for p in models.resnet50().parameters()),
            "bert_large_qa": sum(p.numel() for p in models.BertForQuestionAnswering(models.bert_large_config()).parameters()),
        }
        moe = models.GPT2MoE(models.gpt2_medium_moe8_config(), world_size=8)
    assert counts == {"vgg16": 138_357_544, "resnet50": 25_557_032, "bert_large_qa": 334_094_338}
    experts = [p for p in moe.parameters() if getattr(p, "expert", False)]
    assert experts and all(p.expert for p in experts) and sum(p.numel() for p in moe.parameters()) > 300e6
    tiny = models.GPT2MoE(models.GPT2MoEConfig(vocab_size=128, n_positions=16, n_embd=32, n_layer=2, n_head=2, num_experts=2), world_size=1)
    idx = torch.randint(0, 128, (2, 16))
    loss, _ = tiny(idx, idx)
    loss.backward()
    assert torch.isfinite(loss) and all(p.grad is not None for p in tiny.parameters() if p.requires_grad)


def test_cpp_nhwc_autograd_functions_with_a_host_kernel_table(tmp_path):
    """The C++ autograd Functions of _C_torch.so (BAGUA_NATIVE_NHWC) driven on CPU through a host double of the kernel table
    (tests/cpp/fake_nhwc_api.cpp): in-place output, saved tensors, gradient shapes / memory format / dtypes, the zero-fill + cast
    path and the in-kernel-finish path (workspace handed back zeroed) — against plain PyTorch autograd."""
    import ctypes
    import os
    import shutil
    import subprocess

    from bagua_b200 import _build

    try:
        _build.build_torch_hooks()
        from bagua_b200 import _C_torch as E
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"torch extension unavailable: {e}")
    so = tmp_path / "libfake_nhwc.so"
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "fake_nhwc_api.cpp")
    subprocess.run([shutil.which("g++"), "-O1", "-std=c++17", "-shared", "-fPIC", src, "-o", str(so)], check=True)
    lib = ctypes.CDLL(str(so))
    lib.fake_nhwc_api.restype = ctypes.c_void_p
    torch.manual_seed(0)
    x0 = (torch.randn(2, 8, 6, 6) * 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    b0 = (torch.randn(8) * 0.5).to(torch.bfloat16)
    w = torch.randn(2, 8, 6, 6).to(torch.bfloat16)
    wp = torch.randn(2, 8, 3, 3).to(torch.bfloat16)
    try:
        for fin in (False, True, True):                      # the workspace of the finish path is reused across calls
            E.nhwc_init(lib.fake_nhwc_api(), fin)
            x, b = x0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
            y_in = x * 1.0                                   # non-leaf input, like a convolution output
            y = E.bias_relu(y_in, b)
            assert y.data_ptr() == y_in.data_ptr()           # in place
            (y.float() * w.float()).sum().backward()
            xr, br = x0.clone().float().requires_grad_(True), b0.clone().float().requires_grad_(True)
            (torch.relu(xr + br.view(1, -1, 1, 1)) * w.float()).sum().backward()
            torch.testing.assert_close(y.detach().float(), torch.relu(x0.float() + b0.float().view(1, -1, 1, 1)), rtol=2e-2, atol=2e-2)
            assert x.grad.dtype == torch.bfloat16 and b.grad.dtype == torch.bfloat16 and x.grad.is_contiguous(memory_format=torch.channels_last)
            torch.testing.assert_close(x.grad.float(), xr.grad, rtol=2e-2, atol=2e-2)
            torch.testing.assert_close(b.grad.float(), br.grad, rtol=3e-2, atol=0.15)
            x, b = x0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
            p = E.bias_relu_maxpool2(x * 1.0, b)
            assert p.shape == (2, 8, 3, 3) and p.is_contiguous(memory_format=torch.channels_last)
            (p.float() * wp.float()).sum().backward()
            xr, br = x0.clone().float().requires_grad_(True), b0.clone().float().requires_grad_(True)
            ref = torch.nn.functional.max_pool2d(torch.relu(xr + br.view(1, -1, 1, 1)), 2)
            (ref * wp.float()).sum().backward()
            torch.testing.assert_close(p.detach().float(), ref.detach(), rtol=2e-2, atol=2e-2)
            torch.testing.assert_close(x.grad.float(), xr.grad, rtol=2e-2, atol=2e-2)
            torch.testing.assert_close(b.grad.float(), br.grad, rtol=3e-2, atol=0.15)
        assert [lib.fake_nhwc_calls(i) for i in range(4)] == [3, 3, 3, 3]
        # the whole block in one call: at::conv2d (bias-free) + epilogue, vs conv → relu → pool with plain modules
        E.nhwc_init(lib.fake_nhwc_api(), False)
        conv = torch.nn.Conv2d(8, 8, 3, padding=1).to(torch.bfloat16).to(memory_format=torch.channels_last)
        for pool in (False, True):
            xin = x0.clone().requires_grad_(True)
            out = E.conv_bias_relu(xin, conv.weight, conv.bias, [1, 1], [1, 1], [1, 1], 1, pool)
            ref = torch.relu(conv(x0))
            ref = torch.nn.functional.max_pool2d(ref, 2) if pool else ref
            torch.testing.assert_close(out.float(), ref.float(), rtol=5e-2, atol=5e-2)
            conv.zero_grad()
            out.float().sum().backward()
            assert xin.grad is not None and conv.weight.grad is not None and conv.bias.grad.dtype == torch.bfloat16
    finally:
        E.nhwc_init(0, False)                                # detach the double: nhwc_ready() is False again
    assert not E.nhwc_ready()


def test_python_nhwc_functions_finish_path_with_the_host_double(tmp_path, monkeypatch):
    """ops/nhwc.py's Python autograd Functions, including the BAGUA_NHWC_FINALIZE workspace path, on CPU: ``native()`` is replaced by
    an adapter over the same host kernel double, results are compared with plain PyTorch autograd."""
    import ctypes as C
    import os
    import shutil
    import subprocess
    import types

    from bagua_b200.ops import nhwc

    so = tmp_path / "libfake_nhwc.so"
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "fake_nhwc_api.cpp")
    subprocess.run([shutil.which("g++"), "-O1", "-std=c++17", "-shared", "-fPIC", src, "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.fake_nhwc_api.restype = C.c_void_p
    table = (C.c_void_p * 5).from_address(lib.fake_nhwc_api())
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    fwd = C.CFUNCTYPE(i32, vp, vp, sz, i32, i32, vp)(table[0])
    bwd = C.CFUNCTYPE(i32, vp, vp, vp, vp, sz, i32, i32, vp, vp, vp)(table[1])
    pfwd = C.CFUNCTYPE(i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp)(table[2])
    pbwd = C.CFUNCTYPE(i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp)(table[3])
    fake = types.SimpleNamespace(
        bias_relu_nhwc_fwd=lambda y, b, rows, c, dt, s: fwd(y, b, rows, c, dt, None),
        bias_relu_nhwc_bwd=lambda g, y, go, bg, rows, c, dt, s: bwd(g, y, go, bg, rows, c, dt, None, None, None),
        bias_relu_nhwc_bwd_fin=lambda g, y, go, ws, out, tk, rows, c, dt, s: bwd(g, y, go, ws, rows, c, dt, None, out, tk),
        bias_relu_pool_nhwc_fwd=lambda x, b, o, idx, n, h, w, c, dt, s: pfwd(x, b, o, idx, n, h, w, c, dt, None),
        bias_relu_pool_nhwc_bwd=lambda g, o, idx, gi, bg, n, h, w, c, dt, s: pbwd(g, o, idx, gi, bg, n, h, w, c, dt, None, None, None),
        bias_relu_pool_nhwc_bwd_fin=lambda g, o, idx, gi, ws, out, tk, n, h, w, c, dt, s: pbwd(g, o, idx, gi, ws, n, h, w, c, dt, None, out, tk),
    )
    monkeypatch.setattr(nhwc, "native", lambda: fake)
    monkeypatch.setattr(nhwc, "_stream", lambda: 0)
    monkeypatch.setattr(nhwc, "fused_supported", lambda x, channels: x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last))
    monkeypatch.setattr(nhwc, "_native_fns", [None])
    nhwc._workspaces.clear()
    torch.manual_seed(1)
    x0 = (torch.randn(2, 8, 4, 4) * 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    b0 = (torch.randn(8) * 0.5).to(torch.bfloat16)
    for fin in ("0", "1", "1"):
        monkeypatch.setenv("BAGUA_NHWC_FINALIZE", fin)
        for pool in (False, True):
            x, b = x0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
            out = (nhwc.bias_relu_maxpool2 if pool else nhwc.bias_relu)(x * 1.0, b)
            out.float().pow(2).sum().backward()
            xr, br = x0.clone().float().requires_grad_(True), b0.clone().float().requires_grad_(True)
            ref = torch.relu(xr + br.view(1, -1, 1, 1))
            ref = torch.nn.functional.max_pool2d(ref, 2) if pool else ref
            ref.pow(2).sum().backward()
            torch.testing.assert_close(out.detach().float(), ref.detach(), rtol=2e-2, atol=2e-2)
            torch.testing.assert_close(x.grad.float(), xr.grad, rtol=3e-2, atol=3e-2)
            torch.testing.assert_close(b.grad.float(), br.grad, rtol=3e-2, atol=0.2)
            assert b.grad.dtype == torch.bfloat16
    nhwc._workspaces.clear()


def test_fused_adam_multi_tensor_call_sites_with_a_numpy_kernel_double(monkeypatch):
    """FusedAdam's multi-tensor path (parameters outside the bucket arena) on CPU: the pointer tables built by ``_MultiPlan`` are
    decoded by a numpy stand-in of ``multi_tensor_adam`` / ``multi_tensor_adam_mp`` that applies the Adam update in place — checks the
    list order [param, grad, exp_avg, exp_avg_sq(, master)], the fp32 state of bf16 parameters and the chunk/block map against
    ``torch.optim.AdamW``."""
    import ctypes
    import types

    import numpy as np

    from bagua_b200.ops import optim

    def view(ptr, n, np_dtype):
        return np.ctypeslib.as_array((ctypes.c_uint8 * (n * np.dtype(np_dtype).itemsize)).from_address(ptr)).view(np_dtype)

    def bf16_to_f32(u16):
        return (u16.astype(np.uint32) << 16).view(np.float32)

    def f32_to_bf16(f):
        u = f.astype(np.float32).view(np.uint32)
        return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)

    calls = {"mp": 0, "plain": 0}

    def adam(ptrs, sizes, b2t, b2c, n_t, n_blocks, chunk, dtype, lr, b1, b2, eps, wd, step, adamw, grad_scale, stream, mixed):
        P = view(ptrs, (5 if mixed else 4) * n_t, np.int64)
        S = view(sizes, n_t, np.int64)
        T, Ck = view(b2t, n_blocks, np.int32), view(b2c, n_blocks, np.int32)
        covered = np.zeros(n_t, dtype=np.int64)
        for blk in range(n_blocks):                                   # one "CTA" per (tensor, chunk)
            t, off = int(T[blk]), int(Ck[blk]) * chunk
            n = min(int(S[t]) - off, chunk)
            covered[t] += n
            lowp = dtype in (1, 4)
            raw = (lambda base, np_dt: view(int(base), int(S[t]), np_dt)[off:off + n])
            g16 = raw(P[n_t + t], np.uint16) if lowp else None
            g = bf16_to_f32(g16) if lowp else raw(P[n_t + t], np.float32).copy()
            if mixed:
                m1, m2, w = raw(P[2 * n_t + t], np.float32), raw(P[3 * n_t + t], np.float32), raw(P[4 * n_t + t], np.float32)
            else:
                assert not lowp
                m1, m2, w = raw(P[2 * n_t + t], np.float32), raw(P[3 * n_t + t], np.float32), raw(P[t], np.float32)
            g = g * grad_scale
            if adamw:
                w *= 1 - lr * wd
            else:
                g = g + wd * w
            m1[:] = b1 * m1 + (1 - b1) * g
            m2[:] = b2 * m2 + (1 - b2) * g * g
            w -= (lr / (1 - b1 ** step)) * (m1 / (np.sqrt(m2) / np.sqrt(1 - b2 ** step) + eps))
            if mixed:
                raw(P[t], np.uint16)[:] = f32_to_bf16(w)
        assert (covered == S).all()                                   # the block map covers every element exactly once
        calls["mp" if mixed else "plain"] += 1

    fake = types.SimpleNamespace(multi_tensor_adam_mp=lambda *a: adam(*a, mixed=True), multi_tensor_adam=lambda *a: adam(*a, mixed=False))
    monkeypatch.setattr(optim, "native", lambda: fake)
    monkeypatch.setattr(optim, "_kernels_apply", lambda params: True)
    monkeypatch.setattr(optim, "_stream", lambda: 0)
    monkeypatch.setattr(optim._MultiPlan, "CHUNK", 1000)                # several blocks per tensor
    torch.manual_seed(9)
    shapes = [(65, 33), (1000,), (7, 9, 11), (3,)]
    for dtype in (torch.bfloat16, torch.float32):
        ps = [torch.nn.Parameter((torch.randn(s) * 0.1).to(dtype)) for s in shapes]
        rs = [torch.nn.Parameter(p.detach().float().clone()) for p in ps]
        opt, ropt = optim.FusedAdam(ps, lr=1e-3, adamw=True, weight_decay=0.01), torch.optim.AdamW(rs, lr=1e-3, weight_decay=0.01)
        for _ in range(6):
            for p, r in zip(ps, rs):
                g = torch.randn_like(r)
                p.grad, r.grad = g.to(dtype), g.to(dtype).float()
            opt.step()
            ropt.step()
        for p, r in zip(ps, rs):
            st = opt.state[p]
            assert st["exp_avg"].dtype == torch.float32 and st["step"] == 6
            if dtype == torch.bfloat16:
                torch.testing.assert_close(st["master"], r.data, rtol=1e-4, atol=1e-5)
                torch.testing.assert_close(p.data.float(), r.data, rtol=0, atol=8e-3)
            else:
                assert "master" not in st
                torch.testing.assert_close(p.data, r.data, rtol=1e-4, atol=1e-5)
    assert calls == {"mp": 6, "plain": 6}


def test_vgg_fused_feature_path_on_cpu_through_the_native_extension(tmp_path, monkeypatch):
    """VGG16's ``_features_fused`` (13 conv blocks, 5 with pooling) end to end on CPU: ops/nhwc.py routes every block through the
    C++ extension (BAGUA_NATIVE_NHWC=1) whose kernel table is the host double — output and all gradients against the plain
    ``features`` Sequential.  The only things this does not cover on the GPU path are the CUDA kernels and the stream lookup."""
    import ctypes
    import os
    import shutil
    import subprocess
    import types

    from bagua_b200 import _build
    from bagua_b200.models import vgg16
    from bagua_b200.ops import nhwc

    try:
        _build.build_torch_hooks()
        from bagua_b200 import _C_torch as E
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"torch extension unavailable: {e}")
    so = tmp_path / "libfake_nhwc.so"
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "fake_nhwc_api.cpp")
    subprocess.run([shutil.which("g++"), "-O2", "-std=c++17", "-shared", "-fPIC", src, "-o", str(so)], check=True)
    lib = ctypes.CDLL(str(so))
    lib.fake_nhwc_api.restype = ctypes.c_void_p
    monkeypatch.setenv("BAGUA_NATIVE_NHWC", "1")
    monkeypatch.setattr(nhwc, "native", lambda: types.SimpleNamespace(nhwc_api_ptr=lambda: lib.fake_nhwc_api()))
    monkeypatch.setattr(nhwc, "fused_supported", lambda x, channels: x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last))
    monkeypatch.setattr(nhwc, "_native_fns", [False])
    try:
        torch.manual_seed(2)
        model = vgg16(num_classes=10).to(torch.bfloat16).to(memory_format=torch.channels_last)
        x = torch.randn(2, 3, 32, 32).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        res = []
        for fused in (True, False):
            model.zero_grad(set_to_none=True)
            feats = model._features_fused(x) if fused else model.features(x)
            assert feats.shape == (2, 512, 1, 1)
            feats.float().pow(2).sum().backward()
            res.append([feats.detach().float()] + [p.grad.float().clone() for p in model.features.parameters()])
        assert nhwc._native_functions() is E and lib.fake_nhwc_calls(0) == 8 and lib.fake_nhwc_calls(2) == 5     # 8 plain + 5 pooled blocks
        for a, b in zip(*res):
            torch.testing.assert_close(a, b, rtol=8e-2, atol=8e-2 * max(1.0, b.abs().max().item()))
    finally:
        E.nhwc_init(0, False)


def test_fused_linear_combine_autograd_with_a_host_double_of_the_peer_kernels():
    """``ops.moe_peer.linear_combine`` (fc2 GEMM whose epilogue does the MoE combine): its hand-written backward — scatter of
    grad·gate to the owners, dgrad / wgrad GEMMs, bias and gate-weight gradients — against plain autograd over
    ``Σ_k gate[s,k] · (x·wᵀ + b)[expert, slot]``.  The two peer kernels are replaced by single-rank torch implementations of
    their contracts (csrc/moe_kernels.cu scatter, gemm_wgmma.cu PEER epilogue + local-layout gather)."""
    from bagua_b200.ops import moe_peer

    class HostContext(moe_peer.MoEPeerContext):
        def __init__(self):
            self.world, self.rank = 1, 0

        def scatter(self, rows, expert_idx, slot_idx, scale, E_local, C):
            out = torch.zeros(1, E_local, C, rows.shape[1], dtype=rows.dtype)
            for s in range(rows.shape[0]):
                for k in range(expert_idx.shape[1]):
                    if slot_idx[s, k] >= 0:
                        out[0, expert_idx[s, k], slot_idx[s, k]] = rows[s] * (scale[s, k] if scale is not None else 1.0)
            return out

        def linear_push_gather(self, x, w, bias, expert_idx, slot_idx, weights, S, C):
            y = torch.bmm(x, w.transpose(1, 2)) + (bias.unsqueeze(1) if bias is not None else 0.0)
            picked = torch.zeros(S, expert_idx.shape[1], w.shape[1], dtype=x.dtype)
            for s in range(S):
                for k in range(expert_idx.shape[1]):
                    if slot_idx[s, k] >= 0:
                        picked[s, k] = y[expert_idx[s, k], slot_idx[s, k]]
            return (picked * weights.unsqueeze(-1)).sum(1).to(x.dtype), picked

    torch.manual_seed(3)
    E, C, K, N, S, topk = 3, 4, 8, 6, 7, 2
    expert_idx = torch.stack([torch.randperm(E)[:topk] for _ in range(S)])
    slot_idx = torch.full((S, topk), -1, dtype=torch.int64)
    fill = [0] * E
    for s in range(S):
        for k in range(topk):
            e = int(expert_idx[s, k])
            if fill[e] < C:             # tokens beyond the capacity are dropped (slot −1)
                slot_idx[s, k] = fill[e]
                fill[e] += 1
    assert (slot_idx < 0).any() and (slot_idx >= 0).any()

    def inputs():
        torch.manual_seed(4)
        return [torch.randn(E, C, K, requires_grad=True), torch.randn(E, N, K, requires_grad=True), torch.randn(E, N, requires_grad=True),
                torch.rand(S, topk, requires_grad=True)]

    x, w, b, gate = inputs()
    out = moe_peer.linear_combine(x, w, b, gate, expert_idx, slot_idx, HostContext(), C)
    g = torch.randn_like(out)
    out.backward(g)

    xr, wr, br, gr = inputs()
    y = torch.bmm(xr, wr.transpose(1, 2)) + br.unsqueeze(1)
    valid = (slot_idx >= 0)
    rows = y[expert_idx.clamp(min=0), slot_idx.clamp(min=0)] * valid.unsqueeze(-1)
    ref = (rows * gr.unsqueeze(-1)).sum(1)
    ref.backward(g)
    torch.testing.assert_close(out, ref)
    for got, want, name in [(x.grad, xr.grad, "x"), (w.grad, wr.grad, "w"), (b.grad, br.grad, "bias"), (gate.grad, gr.grad, "gate")]:
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5, msg=lambda m, name=name: f"grad of {name}: {m}")


def test_experts_forward_combine_equals_experts_then_combine_on_the_host():
    """``Experts.forward_combine`` (fc1 → GELU → fc2 with the combine in the GEMM epilogue) against the two-step path
    ``combine(experts(x))`` — outputs and the gradients of every expert parameter, the dispatched tokens and the gate weights;
    peer kernels replaced by single-rank host doubles (see the test above)."""
    from bagua_b200.ops import moe_peer
    from bagua_b200.parallel.moe.experts import Experts

    class MLP(torch.nn.Module):
        grouped_gemm_compatible = True

        def __init__(self, m, h):
            super().__init__()
            self.fc1, self.fc2 = torch.nn.Linear(m, h), torch.nn.Linear(h, m)

        def forward(self, x):
            return self.fc2(torch.nn.functional.gelu(self.fc1(x), approximate="tanh"))

    class HostContext(moe_peer.MoEPeerContext):
        def __init__(self):
            self.world, self.rank = 1, 0

        def scatter(self, rows, expert_idx, slot_idx, scale, E_local, C):
            out = torch.zeros(1, E_local, C, rows.shape[1], dtype=rows.dtype)
            ok = slot_idx >= 0
            s_idx, k_idx = ok.nonzero(as_tuple=True)
            out[0, expert_idx[s_idx, k_idx], slot_idx[s_idx, k_idx]] = rows[s_idx] * (scale[s_idx, k_idx].unsqueeze(-1) if scale is not None else 1.0)
            return out

        def linear_push_gather(self, x, w, bias, expert_idx, slot_idx, weights, S, C):
            y = torch.bmm(x, w.transpose(1, 2)) + (bias.unsqueeze(1) if bias is not None else 0.0)
            ok = (slot_idx >= 0).unsqueeze(-1)
            picked = y[expert_idx.clamp(min=0), slot_idx.clamp(min=0)] * ok
            return (picked * weights.unsqueeze(-1)).sum(1).to(x.dtype), picked

    torch.manual_seed(11)
    E, C, M, H, S, topk = 2, 5, 6, 10, 8, 2
    experts = Experts(MLP(M, H), E)
    for p in experts.parameters():
        torch.nn.init.normal_(p, std=0.3)
    expert_idx = torch.stack([torch.randperm(E)[:topk] for _ in range(S)])
    slot_idx = torch.full((S, topk), -1, dtype=torch.int64)
    fill = [0] * E
    for s in range(S):
        for k in range(topk):
            e = int(expert_idx[s, k])
            if fill[e] < C:
                slot_idx[s, k], fill[e] = fill[e], fill[e] + 1
    g_out = torch.randn(S, M)

    def run(fused: bool):
        experts.zero_grad()
        torch.manual_seed(12)
        x = torch.randn(1, E, C, M, requires_grad=True)
        gate = torch.rand(S, topk, requires_grad=True)
        if fused:
            out = experts.forward_combine(x, gate, expert_idx, slot_idx, HostContext())
        else:
            y = experts(x)[0]                                                   # [E, C, M]
            ok = (slot_idx >= 0).unsqueeze(-1)
            out = (y[expert_idx.clamp(min=0), slot_idx.clamp(min=0)] * ok * gate.unsqueeze(-1)).sum(1)
        out.backward(g_out)
        return [out.detach(), x.grad, gate.grad] + [p.grad.clone() for p in experts.parameters()]

    for a, b in zip(run(True), run(False)):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


def test_graphed_train_step_refuses_what_it_cannot_capture():
    """utils.graph.GraphedTrainStep: optimizers with per-step host state and replicas that communicate inside the step are
    rejected up front (a silently dropped all-reduce or a frozen Adam bias correction would train the wrong model)."""
    from bagua_b200.ops.optim import FusedAdam, FusedSGD
    from bagua_b200.utils.graph import GraphedTrainStep, graph_safe_optimizer

    lin = torch.nn.Linear(4, 4)
    assert graph_safe_optimizer(FusedSGD(lin.parameters(), lr=0.1)) is None
    assert graph_safe_optimizer(torch.optim.SGD(lin.parameters(), lr=0.1, momentum=0.9)) is None
    assert "step count" in graph_safe_optimizer(FusedAdam(lin.parameters()))
    assert "capturable" in graph_safe_optimizer(torch.optim.Adam(lin.parameters()))
    with pytest.raises(ValueError):
        GraphedTrainStep(lin, lambda x: lin(x).sum(), (torch.randn(2, 4),), optimizers=[FusedAdam(lin.parameters())])

    class FakeGroup:
        def size(self):
            return 2

    class FakeEngine:
        process_group, require_backward_grad_sync, _speed_metrics_switch_on = FakeGroup(), True, True

    lin.bagua_ddp = FakeEngine()
    with pytest.raises(NotImplementedError):     # autotune's per-step timing events cannot be captured
        GraphedTrainStep(lin, lambda x: lin(x).sum(), (torch.randn(2, 4),), optimizers=[FusedSGD(lin.parameters(), lr=0.1)])
    FakeEngine._speed_metrics_switch_on = False   # communicating replicas are captured through inline issue → only the device check is left here
    with pytest.raises(RuntimeError):
        GraphedTrainStep(lin, lambda x: lin(x).sum(), (torch.randn(2, 4),), optimizers=[FusedSGD(lin.parameters(), lr=0.1)])


def _flat_resume_worker(rank, world):
    """FusedSGD / FusedAdam on the flat (bucket-arena) path with host doubles of the two flat kernels: checkpoint after 3 steps,
    train 2 more, then a fresh model + optimizer restored from the checkpoint must reproduce those 2 steps exactly — momentum,
    Adam moments + step count and the fp32 master weights of a bf16 model all travel through state_dict()."""
    import copy

    import bagua_b200 as bagua
    from bagua_b200.ops import optim
    from bagua_b200.parallel.algorithms import gradient_allreduce

    def flat_sgd_double(param, grad, momentum_buf, *, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, first_step=False, grad_scale=1.0,
                        zero_grad=False, model=None):
        g = grad.float() * grad_scale
        if weight_decay:
            g = g + weight_decay * param.float()
        if momentum:
            if first_step:
                momentum_buf.copy_(g)
            else:
                momentum_buf.mul_(momentum).add_(g, alpha=1 - dampening)
            g = g + momentum * momentum_buf if nesterov else momentum_buf
        param.add_(g.to(param.dtype), alpha=-lr)
        if model is not None:
            model.copy_(param)
        if zero_grad:
            grad.zero_()

    def flat_adam_double(param, grad, exp_avg, exp_avg_sq, *, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, step=1, adamw=False, grad_scale=1.0,
                         zero_grad=False, model=None):
        g = grad.float() * grad_scale
        if adamw:
            param.mul_(1 - lr * weight_decay)
        elif weight_decay:
            g = g + weight_decay * param.float()
        exp_avg.mul_(betas[0]).add_(g, alpha=1 - betas[0])
        exp_avg_sq.mul_(betas[1]).addcmul_(g, g, value=1 - betas[1])
        denom = exp_avg_sq.sqrt() / (1 - betas[1] ** step) ** 0.5 + eps
        param.add_((exp_avg / denom).to(param.dtype), alpha=-lr / (1 - betas[0] ** step))
        if model is not None:
            model.copy_(param)
        if zero_grad:
            grad.zero_()

    optim._kernels_apply = lambda params: True
    optim.flat_sgd_, optim.flat_adam_ = flat_sgd_double, flat_adam_double
    bagua.init_process_group()
    torch.manual_seed(2)
    base = torch.nn.Sequential(torch.nn.Linear(12, 16), torch.nn.Tanh(), torch.nn.Linear(16, 4))
    batches = [torch.randn(8, 12) for _ in range(5)]
    cases = [("sgd", torch.float32, lambda ps: optim.FusedSGD(ps, lr=0.05, momentum=0.9, weight_decay=1e-3)),
             ("sgd-bf16-master", torch.bfloat16, lambda ps: optim.FusedSGD(ps, lr=0.05, momentum=0.9)),
             ("adam", torch.float32, lambda ps: optim.FusedAdam(ps, lr=1e-2, adamw=True, weight_decay=0.01)),
             ("adam-bf16-master", torch.bfloat16, lambda ps: optim.FusedAdam(ps, lr=1e-2))]
    for tag, dtype, make in cases:
        def fresh(state=None):
            m = copy.deepcopy(base).to(dtype)
            if state is not None:
                m.load_state_dict(state)
            o = make(m.parameters())
            m = m.with_bagua([o], gradient_allreduce.GradientAllReduceAlgorithm())
            return m, o

        def run(m, o, xs):
            for x in xs:
                o.zero_grad()
                m(x.to(dtype)).float().pow(2).mean().backward()
                o.step()
            return torch.cat([p.detach().float().reshape(-1) for p in m.parameters()])

        m, o = fresh()
        run(m, o, batches[:3])
        assert o.flat_segments(), f"{tag}: the flat path was not taken"
        sd, msd = copy.deepcopy(o.state_dict()), copy.deepcopy(m.state_dict())
        if dtype == torch.bfloat16:
            assert all(st["master"].dtype == torch.float32 for st in sd["state"].values())
        want = run(m, o, batches[3:])
        m2, o2 = fresh(msd)
        o2.load_state_dict(sd)
        got = run(m2, o2, batches[3:])
        assert torch.equal(got, want), f"{tag}: resume diverged by {(got - want).abs().max().item()}"
        if tag == "sgd":   # the host double itself against torch.optim.SGD
            ref = copy.deepcopy(base)
            ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3)
            for x in batches:
                ropt.zero_grad()
                ref(x).pow(2).mean().backward()
                ropt.step()
            torch.testing.assert_close(want, torch.cat([p.detach().reshape(-1) for p in ref.parameters()]), rtol=1e-5, atol=1e-6)
    # clip_grad_norm_ on the flat path: one reduction + one multiply over the arena span, same result as the per-tensor utility
    m = copy.deepcopy(base)
    twin = copy.deepcopy(base)
    o = optim.FusedSGD(m.parameters(), lr=0.05, momentum=0.9)
    m = m.with_bagua([o], gradient_allreduce.GradientAllReduceAlgorithm())
    o.zero_grad()
    m(batches[0]).pow(2).mean().mul(50).backward()
    twin(batches[0]).pow(2).mean().mul(50).backward()
    total = o.clip_grad_norm_(0.1)
    want_total = torch.nn.utils.clip_grad_norm_(twin.parameters(), 0.1)
    assert o.flat_segments() and float(want_total) > 0.1
    torch.testing.assert_close(total, want_total)
    for p, q in zip(m.parameters(), twin.parameters()):
        torch.testing.assert_close(p.grad, q.grad)
    return True


def test_flat_fused_optimizers_resume_exactly_from_state_dict():
    from tests.mp_utils import run_distributed

    assert all(run_distributed(_flat_resume_worker, world=1))


def _two_optimizers_worker(rank, world):
    """Two fused optimizers over disjoint halves of one model whose gradients share a bucket: neither may take the flat path (its
    kernel would clear the other optimizer's gradients inside the span); the chunked path trains exactly like two torch SGDs."""
    import copy

    import bagua_b200 as bagua
    from bagua_b200.ops import optim
    from bagua_b200.parallel.algorithms import gradient_allreduce

    optim._kernels_apply = lambda params: True          # pretend the kernels apply: the decision under test is _can_flatten's

    def no_kernel(*a, **k):
        raise AssertionError("flat kernel must not be used when a bucket mixes two optimizers")

    optim.flat_sgd_ = no_kernel
    bagua.init_process_group()
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(6, 8), torch.nn.Tanh(), torch.nn.Linear(8, 2))
    a, b = optim.FusedSGD(model[0].parameters(), lr=0.1, momentum=0.9), optim.FusedSGD(model[2].parameters(), lr=0.05)
    model = model.with_bagua([a, b], gradient_allreduce.GradientAllReduceAlgorithm())
    assert len(model.bagua_buckets) == 1
    group = a.param_groups[0]["params"]
    model(torch.randn(4, 6)).sum().backward()
    assert not optim._can_flatten(group, group) and not optim._can_flatten(b.param_groups[0]["params"], b.param_groups[0]["params"])
    return True


def test_flat_path_is_refused_when_a_bucket_mixes_optimizers():
    from tests.mp_utils import run_distributed

    assert all(run_distributed(_two_optimizers_worker, world=1))
