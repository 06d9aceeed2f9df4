"""Every NVSwitch peer kernel against fp32 oracles on ONE GPU.

``bagua_b200.parallel.virtual.VirtualPeerWorld`` gives P virtual ranks their own signal pads, buffers and streams on the same
device; the P kernels of a collective are launched back to back, become co-resident and exchange data exactly as they would
over NVLink (same slice arithmetic, peer rotation, barrier protocol, parity double-buffering, in/out boxes).  The reference can
only exercise its collectives with >= 2 real GPUs (tests/comm/test_communicator.py, tests/torch_api/test_decentralized.py);
its python oracles are mirrored here (tests/internal/compressor.py:4-33 for MinMaxUInt8).

Not covered here: ``multimem`` (NVLS) flavours — they need a multicast object; see test_self_peer_engine_* for world = 1 and
tests/test_peer_gpu.py for >= 2 GPUs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 3, 4, 8]


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


def _world(P):
    from bagua_b200.parallel.virtual import VirtualPeerWorld

    return VirtualPeerWorld(P, torch.device("cuda", 0), timeout_s=20.0)


def _code(dtype):
    from bagua_b200.core import dtype_code

    return dtype_code(dtype)


def _f32(x):
    return torch.tensor(x, dtype=torch.float32)


def _owned_slice_sum(xs, scale):
    """Bit-exact oracle of the owned-slice reduction (fp32, on the CPU): the vectors of slice s start from rank s's copy, add rank
    (s + i) % P for i = 1 .. P-1 in that order, and are multiplied by the fp32 ``scale``.  Rounding to the dtype is the caller's."""
    P, numel = len(xs), xs[0].numel()
    per = 16 // xs[0].element_size()
    vpr = (numel // per + P - 1) // P
    xs = [x.cpu().float() for x in xs]
    out = torch.empty(numel, dtype=torch.float32)
    for s in range(P):
        lo, hi = s * vpr * per, min((s + 1) * vpr * per, numel)
        if lo >= hi:
            continue
        acc = xs[s][lo:hi].clone()
        for i in range(1, P):
            acc += xs[(s + i) % P][lo:hi]
        out[lo:hi] = acc * scale
    return out


# ---------------------------------------------------------------------------------------------------------------------
# allreduce: two-shot, one-shot, reduce-scatter + all-gather
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_twoshot_allreduce_matches_fp32_sum(C, P, dtype):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    for numel in (8 * 16 // es, 4096 + 16 // es * 3, (1 << 20) + 16 // es * 5):   # tiny, ragged slices, multi-iteration
        nbytes = numel * es
        torch.manual_seed(numel + P)
        xs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        src = w.alloc(nbytes)
        dst = w.alloc(nbytes)
        for r in range(P):
            src.view(r, dtype, numel).copy_(xs[r])
        ref = _owned_slice_sum(xs, _f32(1.0 / P)).to(dtype)
        # out of place, then in place (twice: epochs advance, no reset)
        w.run(lambda r: C.AllReduceOp(w.comms[r], src.buf, dst.buf, 0, 0, nbytes, _code(dtype), 1.0 / P, C.AR_TWO_SHOT, w.cfg(4)))
        for r in range(P):
            assert torch.equal(dst.view(r, dtype, numel).cpu(), ref), (P, dtype, numel, r)
            assert torch.equal(src.view(r, dtype, numel), xs[r])   # source untouched
        w.run(lambda r: C.AllReduceOp(w.comms[r], src.buf, src.buf, 0, 0, nbytes, _code(dtype), 1.0, C.AR_TWO_SHOT, w.cfg(7)))
        ref_sum = _owned_slice_sum(xs, _f32(1.0)).to(dtype)
        for r in range(P):
            assert torch.equal(src.view(r, dtype, numel).cpu(), ref_sum), (P, dtype, numel, r)


@pytest.mark.parametrize("P", WORLDS)
def test_oneshot_allreduce_parity_survives_mixed_grids(C, P):
    """The double-buffered staging half is chosen by the communicator's CALL counter, so calls with different grids (1 CTA for a
    small message, 8 for a larger one) stay in step — the round-1 kernel derived it from per-CTA epochs and did not."""
    from bagua_b200.parallel.symm import ONE_SHOT_SLOT

    w = _world(P)
    dtype = torch.float32
    staging = w.alloc(2 * P * ONE_SHOT_SLOT)
    for i, (numel, blocks) in enumerate([(256, 1), (65536, 8), (4096, 2), (131072, 8), (512, 1), (131072, 5)]):
        nbytes = numel * 4
        torch.manual_seed(i)
        xs = [torch.randn(numel, device=w.device) for _ in range(P)]
        outs = [torch.empty(numel, device=w.device) for _ in range(P)]
        ops = [C.AllReduceOneShotOp(w.comms[r], staging.buf, 0, ONE_SHOT_SLOT, xs[r].data_ptr(), outs[r].data_ptr(), nbytes, _code(dtype), 1.0 / P, w.cfg(blocks))
               for r in range(P)]
        w.run(None, ops=ops)
        ref = xs[0].cpu().clone()   # every rank sums the staging slots in slot order 0 .. P-1
        for p in range(1, P):
            ref += xs[p].cpu()
        ref = ref * _f32(1.0 / P)
        for r in range(P):
            assert torch.equal(outs[r].cpu(), ref), (P, i, r)


@pytest.mark.parametrize("P", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_reduce_scatter_then_all_gather(C, P, dtype):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 18) + 16 // es * 3
    nbytes = numel * es
    torch.manual_seed(5)
    xs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
    buf = w.alloc(nbytes)
    for r in range(P):
        buf.view(r, dtype, numel).copy_(xs[r])
    w.run(lambda r: C.ReduceScatterOp(w.comms[r], buf.buf, 0, nbytes, _code(dtype), 1.0 / P, False, w.cfg(4)))
    ref = _owned_slice_sum(xs, _f32(1.0 / P)).to(dtype)
    per = 16 // es
    vecs = nbytes // 16
    vpr = (vecs + P - 1) // P
    for r in range(P):
        lo, hi = r * vpr * per, min((r + 1) * vpr * per, numel)
        assert torch.equal(buf.view(r, dtype, numel)[lo:hi].cpu(), ref[lo:hi]), (P, dtype, r)
    w.run(lambda r: C.AllGatherOp(w.comms[r], buf.buf, 0, nbytes, _code(dtype), False, w.cfg(4)))
    for r in range(P):
        assert torch.equal(buf.view(r, dtype, numel).cpu(), ref), (P, dtype, r)
    for r in range(1, P):
        assert torch.equal(buf.view(r, dtype, numel), buf.view(0, dtype, numel))   # bit-identical replicas


# ---------------------------------------------------------------------------------------------------------------------
# reduce-scatter -> optimizer -> all-gather (the kernel behind the N > 1 headline)
# ---------------------------------------------------------------------------------------------------------------------
def _shard(numel, es, P, r):
    per = 16 // es
    vecs = numel * es // 16
    vpr = (vecs + P - 1) // P
    return r * vpr * per, min((r + 1) * vpr * per, numel), vpr * per


@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("momentum,nesterov,wd", [(0.0, False, 0.0), (0.9, False, 1e-4), (0.9, True, 5e-4)])
def test_allreduce_sgd_matches_torch_sgd_on_averaged_gradients(C, P, dtype, momentum, nesterov, wd):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 16) + 16 // es * 3       # slices of unequal length
    nbytes = numel * es
    torch.manual_seed(11)
    w0 = torch.randn(numel, device=w.device).to(dtype)
    grads, weights = w.alloc(nbytes), w.alloc(nbytes)
    masters, moms, ops = [], [], []
    for r in range(P):
        weights.view(r, dtype, numel).copy_(w0)
        lo, hi, length = _shard(numel, es, P, r)
        m = torch.zeros(length, device=w.device)
        if hi > lo:
            m[: hi - lo].copy_(w0[lo:hi].float())
        masters.append(m)
        moms.append(torch.zeros(length, device=w.device))
        op = C.AllReduceSgdOp(w.comms[r], grads.buf, weights.buf, 0, 0, nbytes, _code(dtype), m.data_ptr(), moms[r].data_ptr(), 1.0 / P, True, False, w.cfg(6))
        op.set_hyper(0.1, momentum, 0.0, wd, nesterov)
        ops.append(op)
    ref = torch.nn.Parameter(w0.float().clone())
    opt = torch.optim.SGD([ref], lr=0.1, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    for step in range(3):
        gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
        ref.grad = sum(g.float() for g in gs) / P
        opt.step()
        w.run(None, ops=ops)
        for r in range(P):
            assert grads.view(r, dtype, numel).abs().max().item() == 0.0, "gradient bucket must be cleared on the way out"
    # fp32 master shards follow torch exactly; the model copy is the master rounded to the model dtype
    for r in range(P):
        lo, hi, _ = _shard(numel, es, P, r)
        if hi > lo:
            torch.testing.assert_close(masters[r][: hi - lo], ref.data[lo:hi], rtol=2e-5, atol=2e-5)
        got = weights.view(r, dtype, numel).float()
        torch.testing.assert_close(got, ref.data.to(dtype).float(), rtol=0, atol=4e-2 if dtype == torch.bfloat16 else 1e-4)  # one bf16 ulp at |w| ~ 4
        assert torch.equal(weights.view(r, dtype, numel), weights.view(0, dtype, numel))


@pytest.mark.parametrize("P", [1, 2, 4, 8])
@pytest.mark.parametrize("adamw", [False, True])
def test_allreduce_adam_matches_torch(C, P, adamw):
    w = _world(P)
    dtype = torch.bfloat16
    numel = (1 << 15) + 24
    nbytes = numel * 2
    torch.manual_seed(12)
    w0 = torch.randn(numel, device=w.device).to(dtype)
    grads, weights = w.alloc(nbytes), w.alloc(nbytes)
    state, ops = [], []
    for r in range(P):
        weights.view(r, dtype, numel).copy_(w0)
        lo, hi, length = _shard(numel, 2, P, r)
        m = torch.zeros(length, device=w.device)
        if hi > lo:
            m[: hi - lo].copy_(w0[lo:hi].float())
        a, b = torch.zeros(length, device=w.device), torch.zeros(length, device=w.device)
        state.append((m, a, b))
        op = C.AllReduceAdamOp(w.comms[r], grads.buf, weights.buf, 0, 0, nbytes, _code(dtype), m.data_ptr(), a.data_ptr(), b.data_ptr(), 1.0 / P, True, False, w.cfg(4))
        op.set_hyper(1e-2, 0.9, 0.999, 1e-8, 0.01, adamw)
        ops.append(op)
    ref = torch.nn.Parameter(w0.float().clone())
    opt = (torch.optim.AdamW if adamw else torch.optim.Adam)([ref], lr=1e-2, weight_decay=0.01)
    for step in range(3):
        gs = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
        for r in range(P):
            grads.view(r, dtype, numel).copy_(gs[r])
        ref.grad = sum(g.float() for g in gs) / P
        opt.step()
        w.run(None, ops=ops)
    for r in range(P):
        lo, hi, _ = _shard(numel, 2, P, r)
        if hi > lo:
            torch.testing.assert_close(state[r][0][: hi - lo], ref.data[lo:hi], rtol=5e-4, atol=5e-4)  # 1/(sqrt(v)+eps) amplifies summation-order noise where v is tiny
        torch.testing.assert_close(weights.view(r, dtype, numel).float(), ref.data.to(dtype).float(), rtol=0, atol=4e-2)


# ---------------------------------------------------------------------------------------------------------------------
# decentralized: shift_one peer average
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [2, 4, 8])
def test_peer_average_shift_one_pairs_and_values(C, P):
    w = _world(P)
    dtype = torch.float32
    numel = 100000 // 4 * 4
    nbytes = numel * 4
    weights = w.alloc(nbytes)
    outs = [torch.empty(numel, device=w.device) for _ in range(P)]
    ops = [C.PeerAverageOp(w.comms[r], weights.buf, 0, outs[r].data_ptr(), nbytes, _code(dtype), w.cfg(4)) for r in range(P)]
    for step in range(3):
        xs = [torch.randn(numel, device=w.device) + 10 * r for r in range(P)]
        for r in range(P):
            weights.view(r, dtype, numel).copy_(xs[r])
        w.run(None, ops=ops)
        for r in range(P):
            peer = C.PeerAverageOp.shift_one_peer(r, P, step)
            assert C.PeerAverageOp.shift_one_peer(peer, P, step) == r, "pairing must be symmetric"
            assert torch.equal(outs[r].cpu(), (xs[r].cpu() + xs[peer].cpu()) * _f32(0.5)), (P, step, r)


# ---------------------------------------------------------------------------------------------------------------------
# ByteGrad and the low-precision ring against the reference pipeline re-implemented in torch
# ---------------------------------------------------------------------------------------------------------------------
def _bytegrad_oracle(xs, average):
    """compress → alltoall → decompress → reduce (in T) → compress → allgather → decompress, for P virtual ranks."""
    from bagua_b200.ops import quant

    P = len(xs)
    dtype = xs[0].dtype
    numel = xs[0].numel()
    chunk = numel // P
    reduced = []
    for j in range(P):           # owner j
        acc = torch.zeros(chunk, device=xs[0].device)
        for s in range(P):       # contribution of rank s to chunk j, as rank j decodes it
            mm, q = quant.torch_compress_chunk(xs[s][j * chunk:(j + 1) * chunk])
            acc += quant.torch_decompress_chunk(mm, q, dtype).float()
        if average:
            acc = acc / P
        reduced.append(acc.to(dtype))
    out = []
    for j in range(P):
        mm, q = quant.torch_compress_chunk(reduced[j])
        out.append(quant.torch_decompress_chunk(mm, q, dtype))
    return torch.cat(out)


@pytest.mark.parametrize("P", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bytegrad_fused_kernel_matches_pipeline_oracle(C, P, dtype):
    w = _world(P)
    numel = 32 * P * 517
    torch.manual_seed(21)
    box = C.ByteGradOp.box_bytes(numel, P)
    inbox, outbox = w.alloc(box), w.alloc(box)
    datas = [torch.empty(numel, device=w.device, dtype=dtype) for _ in range(P)]
    ops = [C.ByteGradOp(w.comms[r], datas[r].data_ptr(), numel, _code(dtype), inbox.buf, 0, outbox.buf, 0, True, w.cfg(2 * P, 256)) for r in range(P)]
    for it in range(3):          # parity double-buffering of the min/max scratch, monotone grid-barrier counters
        xs = [(torch.randn(numel, device=w.device) * (1 + r)).to(dtype) for r in range(P)]
        for r in range(P):
            datas[r].copy_(xs[r])
        w.run(None, ops=ops)
        ref = _bytegrad_oracle(xs, True).float()
        step = max((x.float().max() - x.float().min()).item() for x in xs) / 255
        for r in range(P):
            err = (datas[r].float() - ref).abs().max().item()
            assert err <= 1.01 * step + (0.02 * ref.abs().max().item() if dtype == torch.bfloat16 else 0.0), (P, dtype, it, r, err, step)
            assert torch.equal(datas[r], datas[0]), "every rank must decode the same bytes"


@pytest.mark.parametrize("P", [1, 4])
def test_bytegrad_with_qadam_momentum_folded_in(C, P):
    """QAdam's compressed stage: m = beta1*m + (1-beta1)*g applied in the kernel's first pass, then the moments are averaged."""
    w = _world(P)
    dtype = torch.float32
    numel = 32 * P * 300
    beta1 = 0.9
    torch.manual_seed(22)
    box = C.ByteGradOp.box_bytes(numel, P)
    inbox, outbox = w.alloc(box), w.alloc(box)
    ms = [torch.randn(numel, device=w.device) for _ in range(P)]
    gs = [torch.randn(numel, device=w.device) for _ in range(P)]
    local = [m.clone().mul_(beta1).add_(g, alpha=1 - beta1) for m, g in zip(ms, gs)]
    ops = []
    for r in range(P):
        op = C.ByteGradOp(w.comms[r], ms[r].data_ptr(), numel, _code(dtype), inbox.buf, 0, outbox.buf, 0, True, w.cfg(2 * P, 256))
        op.set_momentum_source(gs[r].data_ptr(), beta1)
        assert op.kind() == "qadam_momentum_bytegrad_fused"
        ops.append(op)
    w.run(None, ops=ops)
    ref = _bytegrad_oracle(local, True)
    step = max((x.max() - x.min()).item() for x in local) / 255
    for r in range(P):
        assert (ms[r] - ref).abs().max().item() <= 1.01 * step


def _lpdec_oracle(xs, ws, ls, rs):
    from bagua_b200.ops import quant

    P = len(xs)
    dtype = xs[0].dtype
    diffs, qs = [], []
    for r in range(P):
        d = xs[r].clone()
        d.add_(ls[r], alpha=1.0 / 3.0).add_(rs[r], alpha=1.0 / 3.0).sub_(ws[r], alpha=5.0 / 3.0)
        diffs.append(d)
        qs.append(quant.torch_compress_chunk(d))
    out = []
    for r in range(P):
        left, right = (r + P - 1) % P, (r + 1) % P
        nl = ls[r] + quant.torch_decompress_chunk(*qs[left], dtype)
        nr = rs[r] + quant.torch_decompress_chunk(*qs[right], dtype)
        nx = quant.torch_decompress_chunk(*qs[r], dtype) + ws[r]
        out.append((nx, nx.clone(), nl, nr))
    return out


@pytest.mark.parametrize("P", [1, 2, 4, 8])
def test_low_precision_ring_kernel_matches_oracle(C, P):
    w = _world(P)
    dtype = torch.float32
    numel = 32 * 1000
    torch.manual_seed(31)
    box = w.alloc(C.LowPrecRingOp.box_bytes(numel))
    xs = [torch.randn(numel, device=w.device) for _ in range(P)]
    ws = [x + 0.01 * torch.randn_like(x) for x in xs]
    ls = [torch.randn(numel, device=w.device) for _ in range(P)]
    rs = [torch.randn(numel, device=w.device) for _ in range(P)]
    ops = [C.LowPrecRingOp(w.comms[r], xs[r].data_ptr(), ws[r].data_ptr(), ls[r].data_ptr(), rs[r].data_ptr(), numel, _code(dtype), box.buf, 0, w.cfg(4))
           for r in range(P)]
    for it in range(2):
        ref = _lpdec_oracle([x.clone() for x in xs], [x.clone() for x in ws], [x.clone() for x in ls], [x.clone() for x in rs])
        w.run(None, ops=ops)
        for r in range(P):
            for got, want, name in zip((xs[r], ws[r], ls[r], rs[r]), ref[r], ("x", "weight", "left", "right")):
                # identical quantisation levels up to fp contraction: allow one level of the diff's range on rare elements
                tol = 2 * (want.max() - want.min()).item() / 255
                assert (got - want).abs().max().item() <= tol, (P, it, r, name)
                assert ((got - want).abs() > 1e-4).float().mean().item() < 2e-3, (P, it, r, name)


# ---------------------------------------------------------------------------------------------------------------------
# asynchronous model average: one kernel per round, vote-based abort, device-side weight gate
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", WORLDS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_async_average_kernel_round_and_abort_vote(C, P, dtype):
    w = _world(P)
    es = torch.empty(0, dtype=dtype).element_size()
    numel = (1 << 16) + 16 // es * 5
    nbytes = numel * es
    snap, avg = w.alloc(nbytes), w.alloc(nbytes)
    torch.manual_seed(41)
    weights = [torch.randn(numel, device=w.device).to(dtype) for _ in range(P)]
    gates = [C.WeightGate(0) for _ in range(P)]
    ops = [C.AsyncAverageOp(w.comms[r], weights[r].data_ptr(), snap.buf, 0, avg.buf, 0, nbytes, _code(dtype), gates[r], 2.0, False, w.cfg(5)) for r in range(P)]
    x0 = [x.clone() for x in weights]
    w.run(None, ops=ops)
    # the mean is rounded to the dtype when it is published; then w += mean - snapshot in fp32, with snapshot == w here
    mean = _owned_slice_sum(x0, _f32(1.0) / P).to(dtype).float()
    want = [(x.cpu().float() + (mean - x.cpu().float())).to(dtype) for x in x0]
    for r in range(P):
        assert ops[r].status() == 1
        assert gates[r].state() == 0, "the gate must be handed back"
        assert torch.equal(weights[r].cpu(), want[r]), (P, dtype, r)
    # second round with the trainer holding the gate on rank 0: that rank skips the apply after the bounded wait, the others average
    if P > 1:
        ops2 = [C.AsyncAverageOp(w.comms[r], weights[r].data_ptr(), snap.buf, 0, avg.buf, 0, nbytes, _code(dtype), gates[r], 0.2, False, w.cfg(5)) for r in range(P)]
        for r in range(P):
            weights[r].copy_(x0[r])
        gates[0].acquire(torch.cuda.current_stream().cuda_stream, 1.0)
        torch.cuda.synchronize()
        assert gates[0].state() == 1
        w.run(None, ops=ops2)
        assert torch.equal(weights[0], x0[0]), "weights must not change while the trainer holds the gate"
        assert torch.equal(weights[1].cpu(), want[1])
        gates[0].release(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert gates[0].state() == 0
        ops = ops2
    # abort negotiation: ONE rank votes stop -> nobody averages this round and every rank learns it
    for r in range(P):
        weights[r].copy_(x0[r])
    ops[P - 1].abort()
    w.run(None, ops=ops)
    for r in range(P):
        assert ops[r].status() == 0
        assert torch.equal(weights[r], x0[r])
    # resume
    ops[P - 1].reset()
    w.run(None, ops=ops)
    for r in range(P):
        assert ops[r].status() == 1
        assert torch.equal(weights[r].cpu(), want[r]), (P, dtype, r)


def test_weight_gate_orders_apply_after_the_trainer_release(C):
    """The averaging kernel's apply phase waits (on the device) until the trainer's stream releases the gate."""
    P = 2
    w = _world(P)
    numel = 1 << 14
    nbytes = numel * 4
    snap, avg = w.alloc(nbytes), w.alloc(nbytes)
    weights = [torch.full((numel,), float(r), device=w.device) for r in range(P)]
    gates = [C.WeightGate(0) for _ in range(P)]
    ops = [C.AsyncAverageOp(w.comms[r], weights[r].data_ptr(), snap.buf, 0, avg.buf, 0, nbytes, _code(torch.float32), gates[r], 10.0, False, w.cfg(2)) for r in range(P)]
    trainer = torch.cuda.Stream()
    with torch.cuda.stream(trainer):
        # CUDA loads kernels lazily and may not load one while another kernel is running: everything the "trainer" launches while
        # the averaging kernel is parked at the gate must have run once before (true of any training loop after its first step)
        torch.cuda._sleep(1000)
        weights[0].add_(0.0)
    gates[0].acquire(trainer.cuda_stream, 1.0)
    torch.cuda.synchronize()
    for r in range(P):
        C.run_op(ops[r], w.streams[r].cuda_stream, 0)
    # rank 0's kernel is now parked in front of the gate; the "optimizer step" of the trainer lands first, then the release
    with torch.cuda.stream(trainer):
        torch.cuda._sleep(20_000_000)
        weights[0].add_(100.0)
        gates[0].release(trainer.cuda_stream)
    torch.cuda.synchronize()
    w.check()
    # snapshot was taken before the +100 (value 0), mean = 0.5, so rank 0 ends at 100 + (0.5 - 0) and rank 1 at 1 + (0.5 - 1)
    torch.testing.assert_close(weights[0], torch.full_like(weights[0], 100.5))
    torch.testing.assert_close(weights[1], torch.full_like(weights[1], 0.5))


# ---------------------------------------------------------------------------------------------------------------------
# a failed collective is fatal
# ---------------------------------------------------------------------------------------------------------------------
def test_a_lonely_collective_times_out_and_poisons_the_communicator(C):
    from bagua_b200.parallel.virtual import VirtualPeerWorld

    w = VirtualPeerWorld(2, torch.device("cuda", 0), timeout_s=0.3)
    buf = w.alloc(1 << 16)
    op0 = C.AllReduceOp(w.comms[0], buf.buf, buf.buf, 0, 0, 1 << 16, _code(torch.float32), 1.0, C.AR_TWO_SHOT, w.cfg(2))
    C.run_op(op0, w.streams[0].cuda_stream, 0)           # rank 1 never shows up
    torch.cuda.synchronize()
    assert w.comms[0].error_code() == 1
    assert w.comms[0].host_error() == 1                  # mirrored into host-mapped memory: readable without a sync
    with pytest.raises(RuntimeError, match="timed out waiting for another rank"):
        C.run_op(op0, w.streams[0].cuda_stream, 0)       # every later op of the communicator refuses to run
    # abort flag: a spinning kernel gives up immediately and reports "aborted"
    w2 = VirtualPeerWorld(2, torch.device("cuda", 0), timeout_s=30.0)
    buf2 = w2.alloc(1 << 16)
    op = C.AllReduceOp(w2.comms[0], buf2.buf, buf2.buf, 0, 0, 1 << 16, _code(torch.float32), 1.0, C.AR_TWO_SHOT, w2.cfg(2))
    C.run_op(op, w2.streams[0].cuda_stream, 0)
    w2.comms[0].abort()
    torch.cuda.synchronize()
    assert w2.comms[0].error_code() == 2
