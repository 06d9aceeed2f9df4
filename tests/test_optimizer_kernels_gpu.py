"""The optimizer kernels of csrc/multi_tensor.cu and their Python drivers against the float64 per-step oracle of
tests/optim_oracle.py: every dtype combination the flat launchers accept, vector and scalar paths, chunk edges of the multi-tensor
kernels, sentinel words around every buffer, and per-parameter state (first step, step count, fp32 master) in the drivers."""
import pytest
import torch

from tests import optim_oracle as oracle

pytestmark = pytest.mark.gpu

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
INT_OF = {F32: torch.int32, BF16: torch.int16, F16: torch.int16}
SENTINEL = 0x5A


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


class Arena:
    """Tensors carved out of one byte buffer, each 256-byte aligned plus ``misalign`` elements and surrounded by sentinel bytes;
    ``intact()`` tells whether a kernel wrote outside its tensors."""

    PAD = 64

    def __init__(self, dev, specs):
        offs, pos = [], 0
        for n, dt, mis in specs:
            pos = (pos + self.PAD + 255) // 256 * 256 + mis * dt.itemsize
            offs.append(pos)
            pos += n * dt.itemsize
        self.buf = torch.full((pos + self.PAD,), SENTINEL, dtype=torch.uint8, device=dev)
        owned = torch.zeros(self.buf.numel(), dtype=torch.bool)
        self.tensors = []
        for (n, dt, _), o in zip(specs, offs):
            owned[o:o + n * dt.itemsize] = True
            self.tensors.append(self.buf[o:o + n * dt.itemsize].view(dt))
        self.sentinel = (~owned).to(dev)

    def intact(self) -> bool:
        return bool((self.buf[self.sentinel] == SENTINEL).all())


def _fill(t, values):
    t.copy_(values.to(t.dtype))


def _grad_hi(*dtypes):
    return 2.0 if F16 in dtypes else 4.0  # fp16 keeps g*g / 1000 below its largest finite value


def _moments(n, gen, hi=2.0):
    """Adam state as training produces it: sqrt(exp_avg_sq) within a decade or two of |exp_avg|, both down to where eps dominates
    the denominator, and a share of elements that never saw a gradient (both zero: denominator = eps)."""
    m1 = oracle.wide(n, gen, -12, hi, zeros=0.0)
    m2 = m1.double() ** 2 * oracle.wide(n, gen, -2, 2, zeros=0.0, positive=True)
    fresh = torch.rand(n, generator=gen, device=gen.device) < 0.2
    return m1.masked_fill(fresh, 0.0), m2.float().masked_fill(fresh, 0.0)


SGD_CASES = [
    oracle.Sgd(lr=0.05),  # no momentum: no buffer is passed
    oracle.Sgd(lr=0.05, momentum=0.9, weight_decay=1e-4, first_step=True),
    oracle.Sgd(lr=0.05, momentum=0.9, dampening=0.1),
    oracle.Sgd(lr=0.05, momentum=0.9, nesterov=True, weight_decay=0.1, grad_scale=2.0 ** -16),
    oracle.Sgd(lr=0.05, momentum=0.9, weight_decay=1e-4, grad_scale=2.0 ** -16),
]
ADAM_CASES = [oracle.Adam(lr=1e-3, step=t, adamw=aw, weight_decay=0.01, grad_scale=1.0 if t % 2 else 2.0 ** -16)
              for t in (1, 2, 10, 10 ** 4) for aw in (False, True)]


def _run_flat(dev, kind, pt, gt, mt, n, misalign, cases, seed):
    """One arena per call; every case refills it, runs the flat kernel once and checks every output against the oracle."""
    from bagua_b200.ops.optim import flat_adam_, flat_sgd_

    names = ["param", "grad"] + (["m1", "m2"] if kind == "adam" else ["mom"]) + (["model"] if mt else [])
    dts = {"param": pt, "grad": gt, "model": mt}
    arena = Arena(dev, [(n, dts.get(k, F32), int(k == misalign)) for k in names])
    t = dict(zip(names, arena.tensors))
    gen = torch.Generator(device=dev).manual_seed(seed)
    for i, hp in enumerate(cases):
        zero_grad = i % 2 == 0
        _fill(t["param"], torch.randn(n, device=dev, generator=gen) * oracle.wide(n, gen, -3, 1, zeros=0.0, positive=True))
        _fill(t["grad"], oracle.wide(n, gen, hi=_grad_hi(pt, gt, mt)))
        if mt:
            t["model"].fill_(123.0)
        w0, g0 = t["param"].double(), t["grad"].clone()
        if kind == "sgd":
            has_mom = hp.momentum != 0
            # on a first step the kernel must not read the buffer: NaN there would show
            t["mom"].copy_(torch.full((n,), float("nan"), device=dev) if hp.first_step else oracle.wide(n, gen, -6, 2))
            m0 = t["mom"].double()
            ew, em, tw, tm = oracle.sgd(w0, g0, m0, hp)
            flat_sgd_(t["param"], t["grad"], t["mom"] if has_mom else None, lr=hp.lr, momentum=hp.momentum, dampening=hp.dampening,
                      weight_decay=hp.weight_decay, nesterov=hp.nesterov, first_step=hp.first_step, grad_scale=hp.grad_scale,
                      zero_grad=zero_grad, model=t.get("model"))
            if has_mom:
                oracle.check(t["mom"], em, tm, f"{hp} momentum")
            else:
                assert torch.equal(t["mom"].view(torch.int32), m0.float().view(torch.int32))  # untouched when no buffer is passed
        else:
            m1, m2 = _moments(n, gen)
            _fill(t["m1"], m1)
            _fill(t["m2"], m2)
            ew, em1, em2, tw, tm1, tm2 = oracle.adam(w0, g0, t["m1"], t["m2"], hp)
            flat_adam_(t["param"], t["grad"], t["m1"], t["m2"], lr=hp.lr, betas=hp.betas, eps=hp.eps, weight_decay=hp.weight_decay,
                       step=hp.step, adamw=hp.adamw, grad_scale=hp.grad_scale, zero_grad=zero_grad, model=t.get("model"))
            oracle.check(t["m1"], em1, tm1, f"{hp} exp_avg")
            oracle.check(t["m2"], em2, tm2, f"{hp} exp_avg_sq")
        oracle.check(t["param"], ew, tw, f"{hp} param")
        if mt and pt == F32:  # both stores come from one fp32 register: the model copy is the master rounded once
            assert torch.equal(t["model"], t["param"].to(mt)), hp
        elif mt:
            oracle.check(t["model"], ew, tw, f"{hp} model copy")
        if zero_grad:
            assert bool((t["grad"].view(INT_OF[gt]) == 0).all()), hp
        else:
            assert torch.equal(t["grad"].view(INT_OF[gt]), g0.view(INT_OF[gt])), hp
        assert arena.intact(), (hp, "a sentinel byte changed")


DTYPE_MATRIX = [(p, g, m) for p in (F32, BF16, F16) for g in (F32, BF16, F16) for m in (None, BF16, F16)]


@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("pt,gt,mt", DTYPE_MATRIX, ids=lambda d: str(d).replace("torch.", "") if d else "none")
def test_flat_kernels_every_dtype_combination(dev, kind, pt, gt, mt):
    cases = [SGD_CASES[2], SGD_CASES[3]] if kind == "sgd" else [ADAM_CASES[4], ADAM_CASES[5]]
    _run_flat(dev, kind, pt, gt, mt, 4099, None, cases, seed=11)


BENCH_SIZES = [1, 7, 8, 9, 5 * 2 ** 20 + 13]  # the last is more than one sweep of the grid: 528 CTAs x 512 threads x 8


@pytest.mark.parametrize("n", BENCH_SIZES)
@pytest.mark.parametrize("pt,gt,mt", [(F32, BF16, BF16), (F32, F32, None)], ids=["f32-bf16-bf16", "f32-f32-none"])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_flat_kernels_at_the_benchmark_dtypes_on_vector_and_scalar_paths(dev, kind, pt, gt, mt, n):
    names = ["param", "grad"] + (["m1", "m2"] if kind == "adam" else ["mom"]) + (["model"] if mt else [])
    for misalign in [None] + names:  # all 32-byte aligned (vector path), then each buffer in turn off by one element
        _run_flat(dev, kind, pt, gt, mt, n, misalign, SGD_CASES if kind == "sgd" else ADAM_CASES, seed=n)


CHUNK_SIZES = [0, 1, 65535, 65536, 65537, 2 * 65536 + 3]
CL_SHAPE = (3, 8, 5, 7)  # a channels_last 4-D parameter: the kernels walk its raw memory


def _multi(dev, kernel, dt, has_mom, hp, seed):
    from bagua_b200.core import dtype_code, native
    from bagua_b200.ops.optim import multi_tensor_plan

    C = native()
    sizes = CHUNK_SIZES + [torch.Size(CL_SHAPE).numel()]
    if kernel.startswith("sgd"):
        mp = kernel == "sgd_mp"
        state = ([F32] if mp else []) + ([F32 if mp else dt] if has_mom else [])
    else:
        mp = kernel == "adam_mp"
        state = [F32, F32, F32] if mp else [dt, dt]
    dtypes = [dt, dt] + state
    arena = Arena(dev, [(n, d, 0) for d in dtypes for n in sizes])
    flat = [arena.tensors[i * len(sizes):(i + 1) * len(sizes)] for i in range(len(dtypes))]  # raw memory, filled and checked
    cl = torch.empty(CL_SHAPE).to(memory_format=torch.channels_last).stride()
    lists = [lst[:-1] + [lst[-1].as_strided(CL_SHAPE, cl)] for lst in flat]  # what the kernel is given
    gen = torch.Generator(device=dev).manual_seed(seed)
    for f in flat[0]:
        _fill(f, torch.randn(f.numel(), device=dev, generator=gen) * oracle.wide(f.numel(), gen, -3, 1, zeros=0.0, positive=True))
    for f in flat[1]:
        _fill(f, oracle.wide(f.numel(), gen, hi=_grad_hi(dt)))
    if mp:  # master weights: the parameter's values, kept in fp32
        for f, p in zip(flat[2 if kernel == "sgd_mp" else 4], flat[0]):
            _fill(f, p.float() + oracle.wide(p.numel(), gen, -9, -6))
    if kernel.startswith("adam"):
        for f1, f2 in zip(flat[2], flat[3]):
            m1, m2 = _moments(f1.numel(), gen, hi=0.0 if state[0] == F16 else 2.0)  # fp16 moments stay finite
            _fill(f1, m1)
            _fill(f2, m2)
    elif has_mom:
        for f in flat[-1]:
            _fill(f, oracle.wide(f.numel(), gen, -6, 2))
    before = [[f.double() for f in lst] for lst in flat]
    grads_bits = [f.clone() for f in flat[1]]
    plan = multi_tensor_plan(lists)
    s = torch.cuda.current_stream().cuda_stream
    if kernel.startswith("sgd"):
        fn = C.multi_tensor_sgd_mp if mp else C.multi_tensor_sgd
        fn(*plan.args(), dtype_code(dt), has_mom, hp.lr, hp.momentum, hp.dampening, hp.weight_decay, hp.nesterov, hp.first_step, hp.grad_scale, s)
    else:
        fn = C.multi_tensor_adam_mp if mp else C.multi_tensor_adam
        fn(*plan.args(), dtype_code(dt), hp.lr, hp.betas[0], hp.betas[1], hp.eps, hp.weight_decay, hp.step, hp.adamw, hp.grad_scale, s)
    for i in range(len(sizes)):
        b = [lst[i] for lst in before]
        out = [lst[i] for lst in flat]
        what = f"{kernel} {dt} tensor of {sizes[i]} {hp}"
        assert torch.equal(out[1].view(INT_OF[dt]), grads_bits[i].view(INT_OF[dt])), what
        if kernel.startswith("sgd"):
            w = b[2] if mp else b[0]
            ew, em, tw, tm = oracle.sgd(w, b[1], b[-1], hp)
            if has_mom:
                oracle.check(out[-1], em, tm, what + " momentum")
            master = out[2] if mp else None
        else:
            w = b[4] if mp else b[0]
            ew, em1, em2, tw, tm1, tm2 = oracle.adam(w, b[1], b[2], b[3], hp)
            oracle.check(out[2], em1, tm1, what + " exp_avg")
            oracle.check(out[3], em2, tm2, what + " exp_avg_sq")
            master = out[4] if mp else None
        if master is not None:
            oracle.check(master, ew, tw, what + " master")
            assert torch.equal(out[0], master.to(dt)), what  # the parameter is the new master rounded once
        else:
            oracle.check(out[0], ew, tw, what + " param")
    assert arena.intact(), "a sentinel byte changed"


@pytest.mark.parametrize("dt", [F32, BF16, F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("kernel", ["sgd", "sgd_mp"])
def test_multi_tensor_sgd_kernels_across_chunk_edges(dev, kernel, dt):
    for i, hp in enumerate(SGD_CASES):
        _multi(dev, kernel, dt, hp.momentum != 0, hp, seed=i)


@pytest.mark.parametrize("dt", [F32, BF16, F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("kernel", ["adam", "adam_mp"])
def test_multi_tensor_adam_kernels_across_chunk_edges(dev, kernel, dt):
    for i, hp in enumerate([ADAM_CASES[0], ADAM_CASES[3], ADAM_CASES[7]]):
        _multi(dev, kernel, dt, False, hp, seed=i)


# ---- drivers: torch.optim semantics, state tracked per parameter -------------------------------------------------------
# hyperparameters exactly representable in fp32, so that torch's double-precision scalars and the kernels' fp32 ones agree
LR, MOM, DAMP, WD, BETAS = 2.0 ** -5, 0.875, 0.125, 2.0 ** -10, (0.875, 1 - 2.0 ** -9)


def _make(driver, params, lr=LR):
    from bagua_b200.contrib import fuse_optimizer
    from bagua_b200.ops.optim import FusedAdam, FusedSGD

    if driver == "FusedSGD":
        return FusedSGD(params, lr=lr, momentum=MOM, dampening=DAMP, weight_decay=WD)
    if driver == "FusedAdam":
        return FusedAdam(params, lr=lr, betas=BETAS, weight_decay=WD, adamw=True)
    if driver == "fuse_optimizer(SGD)":
        return fuse_optimizer(torch.optim.SGD(params, lr=lr, momentum=MOM, dampening=DAMP, weight_decay=WD), do_flatten=False)
    return fuse_optimizer(torch.optim.Adam(params, lr=lr, betas=BETAS, weight_decay=WD), do_flatten=False)


class Tracker:
    """Runs ``opt`` step by step and checks each parameter against the oracle from its own state before the step, with the first
    step and the step count that ``torch.optim`` would use for that parameter."""

    def __init__(self, driver, opt, params, lr=LR):
        self.sgd = "SGD" in driver
        self.adamw = driver == "FusedAdam"
        self.opt, self.params, self.lr = opt, params, lr
        self.count = [0] * len(params)

    def step(self):
        expect = []
        for i, p in enumerate(self.params):
            if p.grad is None:
                expect.append(p.detach().clone())
                continue
            st = self.opt.state.get(p, {})
            w = st["master"] if "master" in st else p.detach()
            zeros = torch.zeros_like(w, dtype=torch.float64)
            if self.sgd:
                hp = oracle.Sgd(lr=self.lr, momentum=MOM, dampening=DAMP, weight_decay=WD, first_step=self.count[i] == 0)
                expect.append(oracle.sgd(w, p.grad, st.get("momentum_buffer", zeros), hp))
            else:
                hp = oracle.Adam(lr=self.lr, step=self.count[i] + 1, betas=BETAS, weight_decay=WD, adamw=self.adamw)
                expect.append(oracle.adam(w, p.grad, st.get("exp_avg", zeros), st.get("exp_avg_sq", zeros), hp))
        self.opt.fuse_step() if hasattr(self.opt, "fuse_step") else self.opt.step()
        for i, (p, e) in enumerate(zip(self.params, expect)):
            what = f"parameter {i} after its step {self.count[i] + 1}"
            if p.grad is None:
                assert torch.equal(p, e), what
                continue
            self.count[i] += 1
            st = self.opt.state[p]
            if self.sgd:
                ew, em, tw, tm = e
                oracle.check(st["momentum_buffer"], em, tm, what + " momentum")
            else:
                ew, em1, em2, tw, tm1, tm2 = e
                oracle.check(st["exp_avg"], em1, tm1, what + " exp_avg")
                oracle.check(st["exp_avg_sq"], em2, tm2, what + " exp_avg_sq")
            if "master" in st:
                oracle.check(st["master"], ew, tw, what + " master")
                assert torch.equal(p.detach(), st["master"].to(p.dtype)), what
            else:
                oracle.check(p, ew, tw, what)


DRIVERS = ["FusedSGD", "FusedAdam", "fuse_optimizer(SGD)", "fuse_optimizer(Adam)"]


@pytest.mark.parametrize("late", [0, 2], ids=["first", "last"])
@pytest.mark.parametrize("driver", DRIVERS)
def test_a_parameter_that_joins_late_keeps_the_others_state(dev, driver, late):
    """The late parameter's gradient is None for two steps (a frozen layer, an unused branch): its first step must be a first
    step, and the others must keep their momentum and step counts."""
    torch.manual_seed(5)
    params = [torch.nn.Parameter(torch.randn(s, device=dev)) for s in [(70000,), (33, 3), (129,)]]
    tr = Tracker(driver, _make(driver, params), params)
    for step in range(5):
        for i, p in enumerate(params):
            p.grad = None if (i == late and step < 2) else torch.randn_like(p)
        tr.step()
    assert tr.count == [5 if i != late else 3 for i in range(3)]


@pytest.mark.parametrize("driver", ["FusedSGD", "FusedAdam"])
def test_bf16_parameters_move_through_their_fp32_master(dev, driver):
    """lr * update stays below half a bf16 ulp of the weights for 100 steps: only an fp32 master accumulates it."""
    torch.manual_seed(6)
    params = [torch.nn.Parameter((1.0 + 0.01 * torch.rand(s, device=dev)).to(BF16)) for s in [(1000,), (70000,)]]
    start = [p.detach().clone() for p in params]
    lr = 2.0 ** -13
    tr = Tracker(driver, _make(driver, params, lr=lr), params, lr=lr)
    for _ in range(100):
        for p in params:
            p.grad = (torch.rand_like(p, dtype=F32) * 0.5 + 0.5).to(BF16)
        tr.step()
    for p, p0 in zip(params, start):
        st = tr.opt.state[p]
        assert st["master"].dtype == F32
        assert (st["momentum_buffer"] if driver == "FusedSGD" else st["exp_avg"]).dtype == F32
        assert bool((p != p0).float().mean() > 0.9), "the bf16 parameters did not move"


@pytest.mark.parametrize("driver", DRIVERS)
def test_channels_last_parameter_with_a_contiguous_gradient(dev, driver):
    torch.manual_seed(7)
    params = [torch.nn.Parameter(torch.randn(4, 6, 5, 3, device=dev).to(memory_format=torch.channels_last)),
              torch.nn.Parameter(torch.randn(17, device=dev))]
    tr = Tracker(driver, _make(driver, params), params)
    for _ in range(3):
        for p in params:
            p.grad = torch.randn(p.shape, device=dev)  # contiguous, whatever the parameter's layout
        tr.step()
