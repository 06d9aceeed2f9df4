"""One launch of every hand-written kernel at a production-sized problem, world = 1 (this GPU is its own peer), for ``ncu``:

    ncu --set full --clock-control none --import-source on -k 'regex:allreduce_|all_gather_k|reduce_scatter_k|peer_average|bytegrad|lpdec|async_average|flat_sgd|flat_adam|minmax_uint8|bias_relu|moe_|grouped_gemm' -o gpurun_out/ncu_zoo python scripts/kernel_zoo.py

ncu serialises and replays kernels, so it can never wrap a multi-rank job; the self-peer launches exercise the same code (slice
arithmetic, barrier, optimizer epilogue, quantisation passes) with the peer loads/stores landing in local HBM — which is what the
DRAM-side roofline of these kernels is about.  NVLink-side numbers come from the event-timed multi-GPU benches
(benchmarks/collective_bench.py).  Without ncu the script prints CUDA-event times per kernel (L2 flushed in between) with the
clock record, as JSON lines.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bagua_b200.core import dtype_code, native  # noqa: E402
from bagua_b200.ops import gemm, quant  # noqa: E402
from bagua_b200.ops.optim import flat_adam_, flat_sgd_, multi_tensor_plan  # noqa: E402
from bagua_b200.parallel.virtual import VirtualPeerWorld  # noqa: E402

from bench import ClockSampler  # noqa: E402

dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
sampler = ClockSampler(0).start()
C = native()
w = VirtualPeerWorld(1, dev, timeout_s=10.0)
comm = w.comms[0]
bf, f32 = torch.bfloat16, torch.float32
stream = torch.cuda.current_stream().cuda_stream
flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device=dev)
rows = []


UNDER_NCU = os.environ.get("ZOO_NCU", "0") == "1"   # one launch per kernel, no warm-up: every launch is replayed ~40x by ncu


def timed(name, fn, nbytes_alg, iters=5, flops=0.0):
    """``nbytes_alg``: algorithmic HBM bytes of one launch (what an ideal implementation must move)."""
    if UNDER_NCU:
        iters = 1
    else:
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ms = sorted(ts)[len(ts) // 2]
    row = {"kernel": name, "ms": ms, "alg_bytes": nbytes_alg, "GBps": nbytes_alg / ms / 1e6}
    if flops:
        row["TFLOPs"] = flops / ms / 1e9
    rows.append(row)


def run(op):
    C.run_op(op, stream, 0)


NB = 64 * 1024 * 1024          # one bucket
n = NB // 2
a, b = w.alloc(NB), w.alloc(NB)
a.view(0, bf, n).normal_()
b.view(0, bf, n).normal_()
code = dtype_code(bf)

op = C.AllReduceOp(comm, a.buf, b.buf, 0, 0, NB, code, 1.0, C.AR_TWO_SHOT, w.cfg(32))
timed("allreduce_twoshot_kernel<bf16,P=1> 64MiB out-of-place", lambda: run(op), 2 * NB)
master, mom = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
sgd = C.AllReduceSgdOp(comm, a.buf, b.buf, 0, 0, NB, code, master.data_ptr(), mom.data_ptr(), 1.0, True, False, w.cfg(32))
sgd.set_hyper(0.01, 0.9, 0.0, 1e-4, False)
run(sgd)  # first step initialises the momentum
# reads grads (2B) + master, momentum (8B); writes master, momentum (8B) + weights (2B) + zeroed grads (2B) per element
timed("allreduce_update_kernel<bf16,P=1,peer,SgdRule> 64MiB bucket, momentum", lambda: run(sgd), n * 22)
m2 = torch.zeros(n, device=dev)
adam = C.AllReduceAdamOp(comm, a.buf, b.buf, 0, 0, NB, code, master.data_ptr(), mom.data_ptr(), m2.data_ptr(), 1.0, True, False, w.cfg(32))
adam.set_hyper(1e-3, 0.9, 0.999, 1e-8, 0.01, True)
timed("allreduce_update_kernel<bf16,P=1,peer,AdamRule> 64MiB bucket", lambda: run(adam), n * 30)
rs = C.ReduceScatterOp(comm, a.buf, 0, NB, code, 1.0, False, w.cfg(32))
timed("reduce_scatter_kernel<bf16,P=1> 64MiB", lambda: run(rs), 2 * NB)
ag = C.AllGatherOp(comm, a.buf, 0, NB, code, False, w.cfg(32))
timed("all_gather_kernel<bf16,P=1> 64MiB", lambda: run(ag), NB)
out = torch.empty(n, device=dev, dtype=bf)
pa = C.PeerAverageOp(comm, b.buf, 0, out.data_ptr(), NB, code, w.cfg(32))
timed("peer_average_kernel<bf16> 64MiB", lambda: run(pa), 3 * NB)

numel = 32 * 1024 * 1024
data = torch.randn(numel, device=dev).to(bf)
box = C.ByteGradOp.box_bytes(numel, 1)
inbox, outbox = w.alloc(box), w.alloc(box)
bg = C.ByteGradOp(comm, data.data_ptr(), numel, code, inbox.buf, 0, outbox.buf, 0, True, w.cfg(128, 512))
# A: read 2B; B: read 2B write 1B; C: read 1B write 4B(fp32 scratch); D: read 4B write 1B; E: read 1B write 2B  = 18 B / element
timed("bytegrad_kernel<bf16,P=1> 32M elements", lambda: run(bg), numel * 18)
g = torch.randn(numel, device=dev).to(bf)
bg2 = C.ByteGradOp(comm, data.data_ptr(), numel, code, inbox.buf, 0, outbox.buf, 0, True, w.cfg(128, 512))
bg2.set_momentum_source(g.data_ptr(), 0.9)
timed("bytegrad_kernel<bf16,P=1>+qadam momentum 32M elements", lambda: run(bg2), numel * 22)
x32, w32, l32, r32 = (torch.randn(16 * 1024 * 1024, device=dev) for _ in range(4))
ring_box = w.alloc(C.LowPrecRingOp.box_bytes(x32.numel()))
ring = C.LowPrecRingOp(comm, x32.data_ptr(), w32.data_ptr(), l32.data_ptr(), r32.data_ptr(), x32.numel(), dtype_code(f32), ring_box.buf, 0, w.cfg(128))
timed("lpdec_ring_kernel<f32> 16M elements", lambda: run(ring), x32.numel() * (20 + 7 + 4 * 9))
gate = C.WeightGate(0)
snap, avg = w.alloc(NB), w.alloc(NB)
aa = C.AsyncAverageOp(comm, out.data_ptr(), snap.buf, 0, avg.buf, 0, NB, code, gate, 1.0, False, w.cfg(16))
timed("async_average_kernel<bf16,P=1,peer> 64MiB", lambda: run(aa), 8 * NB)
# in-bucket LAMB on the 64 MiB bucket as ONE parameter (shard, master, moments fp32)
shard = torch.randn(n, device=dev)
lplan = multi_tensor_plan([[master], [shard], [mom], [m2]])
lpart = torch.zeros(lplan.n_blocks, 2, dtype=torch.float64, device=dev)
lmom = C.LambMomentsOp(*lplan.args(), 0, lpart.data_ptr())
lmom.set_hyper(1e-3, 0.9, 0.999, 1e-6, 0.01)
# reads master, shard, both moments (16B); writes both moments (8B) per element
timed("multi_tensor_lamb_stage1_kernel<f32> 32M-element shard (in-bucket moments)", lambda: run(lmom), n * 24)
lptr = torch.tensor([lpart.data_ptr()], dtype=torch.int64, device=dev)
lnb = torch.tensor([lplan.n_blocks], dtype=torch.int32, device=dev)
lratio, lsums = torch.ones(1, device=dev), torch.zeros(1, 2, dtype=torch.float64, device=dev)
rbox = w.alloc(C.LambRatioOp.box_bytes(1))
lrop = C.LambRatioOp(comm, rbox.buf, 0, lptr.data_ptr(), lnb.data_ptr(), 1, lratio.data_ptr(), lsums.data_ptr())
timed("lamb_ratio_kernel 1 parameter", lambda: run(lrop), lplan.n_blocks * 16)
lsegs = torch.tensor([0, n, 0], dtype=torch.int32, device=dev)
lapply = C.ShardLambOp(comm, b.buf, 0, NB, code, master.data_ptr(), mom.data_ptr(), m2.data_ptr(), lsegs.data_ptr(), 1, lratio.data_ptr(), False, w.cfg(32))
lapply.set_hyper(1e-3, 0.9, 0.999, 1e-6, 0.01)
# reads master and both moments (12B); writes master (4B) + weights (2B) per element
timed("shard_update_kernel<bf16,P=1,peer,LambRule> 64MiB bucket", lambda: run(lapply), n * 18)
# in-bucket LARS on the same bucket as ONE parameter: stage-1 norms over [master, shard], apply from the exchanged sums
nplan = multi_tensor_plan([[master], [shard]])
npart = torch.zeros(nplan.n_blocks, 2, dtype=torch.float64, device=dev)
lnorms = C.LarsNormsOp(*nplan.args(), 0, npart.data_ptr())
# reads master and shard (8B) per element
timed("multi_tensor_lars_stage1_kernel<f32> 32M-element shard (in-bucket norms)", lambda: run(lnorms), n * 8)
lsums.copy_(torch.tensor([[float(n), float(n)]], dtype=torch.float64))
lars = C.ShardLarsOp(comm, b.buf, 0, NB, code, shard.data_ptr(), 0, master.data_ptr(), mom.data_ptr(), lsegs.data_ptr(), 1, lsums.data_ptr(), False, w.cfg(32))
lars.set_hyper(1e-3, 0.9, 5e-4, 1e-3)
# reads shard, master, momentum (12B); writes master, momentum (8B) + weights (2B) per element
timed("shard_update_kernel<bf16,P=1,peer,LarsRule> 64MiB bucket", lambda: run(lars), n * 22)
# phase A into the same shard: overwrite (reads the bucket 2B, writes the shard 4B) and accumulate (+ reads the shard 4B) per element
gpart = torch.zeros(C.MAX_COMM_BLOCKS, dtype=torch.float64, device=dev)
for acc, nb in ((False, 6), (True, 10)):
    sg = C.ShardGradOp(comm, a.buf, 0, NB, code, shard.data_ptr(), gpart.data_ptr(), 1.0, True, False, w.cfg(64), acc)
    run(sg)   # an accumulating op overwrites on its first run
    timed(f"shard_grad_kernel<bf16,P=1,peer,ACCUM={str(acc).lower()}> 64MiB bucket", lambda sg=sg: run(sg), n * nb)
# weight EMA of the same shard: the local update (reads master and EMA 8B, writes the EMA 4B per element), and the EMA published as the
# bucket's weights (reads the shard 4B, writes the weights 2B per element)
eshard = master.clone()
eplan = multi_tensor_plan([[master], [eshard]])
ema_op = C.EmaOp(*eplan.args(), 1e-4, 0)
timed("multi_tensor_ema_kernel 32M-element shard", lambda: run(ema_op), n * 12)
pub = C.ShardPublishOp(comm, b.buf, 0, NB, code, eshard.data_ptr(), False, w.cfg(64))
timed("shard_publish_kernel<bf16,P=1,peer> 64MiB bucket", lambda: run(pub), n * 6)
# in-bucket Lion on the same bucket: the fused kernel (reads the bucket 2B, master and exp_avg 8B; writes master and exp_avg 8B, the
# weights 2B and the cleared bucket 2B per element) and phase B (reads shard, master, exp_avg 12B; writes 8B + the weights 2B)
lion = C.AllReduceLionOp(comm, a.buf, b.buf, 0, 0, NB, code, master.data_ptr(), mom.data_ptr(), 1.0, True, False, w.cfg(32))
lion.set_hyper(1e-4, 0.9, 0.99, 0.1)
timed("allreduce_update_kernel<bf16,P=1,peer,LionRule> 64MiB bucket", lambda: run(lion), n * 22)
unit = torch.ones(1, device=dev)
slion = C.ShardLionOp(comm, b.buf, 0, NB, code, shard.data_ptr(), unit.data_ptr(), master.data_ptr(), mom.data_ptr(), False, w.cfg(64))
slion.set_hyper(1e-4, 0.9, 0.99, 0.1)
timed("shard_update_kernel<bf16,P=1,peer,LionRule> 64MiB bucket", lambda: run(slion), n * 22)
del shard, lpart, npart, gpart, eshard

# single-GPU kernels ------------------------------------------------------------------------------------------------------
P = 138 * 1000 * 1000 // 8 * 8   # VGG16-sized arena
p32 = torch.randn(P, device=dev)
g16 = torch.randn(P, device=dev).to(bf)
mb = torch.zeros(P, device=dev)
model = torch.empty(P, device=dev, dtype=bf)
timed("flat_sgd_kernel 138M params (bf16 grads, fp32 master, momentum)", lambda: flat_sgd_(p32, g16, mb, lr=0.01, momentum=0.9, zero_grad=True, model=model, first_step=False), P * 22, iters=3)
e1, e2 = torch.zeros(P, device=dev), torch.zeros(P, device=dev)
timed("flat_adam_kernel 138M params", lambda: flat_adam_(p32, g16, e1, e2, lr=1e-3, step=2, adamw=True, weight_decay=0.01, zero_grad=True, model=model), P * 30, iters=3)
# multi-tensor Lion over the same arena as one bf16 parameter with an fp32 master: reads the gradient 2B, master and exp_avg 8B; writes
# the parameter 2B, master and exp_avg 8B and the cleared gradient 2B per element
lplan = multi_tensor_plan([[model], [g16], [p32], [e1]])
timed("multi_tensor_lion_kernel<bf16,mixed> 138M params", lambda: C.multi_tensor_lion(*lplan.args(), code, True, 1e-4, 0.9, 0.99, 0.1, True, stream), P * 22,
      iters=3)
del p32, g16, mb, model, e1, e2, lplan
xq = torch.randn(64 * 1024 * 1024, device=dev).to(bf)
qbuf = quant.compress(xq, 8)
timed("minmax_uint8_compress 64M bf16, 8 chunks", lambda: quant.compress(xq, 8, out=qbuf), xq.numel() * 5)
timed("minmax_uint8_decompress 64M", lambda: quant.decompress(qbuf, xq, 8), xq.numel() * 3)
from bagua_b200.ops import nhwc  # noqa: E402

y = torch.randn(32, 64, 224, 224, device=dev).to(bf).contiguous(memory_format=torch.channels_last)
bias = torch.randn(64, device=dev).to(bf)
timed("bias_relu_fwd_kernel 32x64x224x224 NHWC", lambda: C.bias_relu_nhwc_fwd(y.data_ptr(), bias.data_ptr(), 32 * 224 * 224, 64, code, stream), y.numel() * 4)
gy = torch.randn_like(y)
gout = torch.empty_like(y)
bg32 = torch.zeros(64, device=dev)
timed("bias_relu_bwd_kernel 32x64x224x224 NHWC", lambda: C.bias_relu_nhwc_bwd(gy.data_ptr(), y.data_ptr(), gout.data_ptr(), bg32.data_ptr(), 32 * 224 * 224, 64, code, stream), y.numel() * 6)
pooled = torch.empty(32, 64, 112, 112, device=dev, dtype=bf).contiguous(memory_format=torch.channels_last)
idx = torch.empty(32 * 112 * 112 * 64, device=dev, dtype=torch.uint8)
timed("bias_relu_pool_fwd_kernel 32x64x224x224 -> 112x112", lambda: C.bias_relu_pool_nhwc_fwd(y.data_ptr(), bias.data_ptr(), pooled.data_ptr(), idx.data_ptr(), 32, 224, 224, 64, code, stream),
      y.numel() * 2 + pooled.numel() * 3)
gp = torch.randn_like(pooled)
timed("bias_relu_pool_bwd_kernel 112x112 -> 224x224", lambda: C.bias_relu_pool_nhwc_bwd(gp.data_ptr(), pooled.data_ptr(), idx.data_ptr(), gout.data_ptr(), bg32.data_ptr(), 32, 224, 224, 64, code, stream),
      pooled.numel() * 5 + y.numel() * 2)
# MoE exchange (GPT-2 medium MoE-8 on 8 GPUs: S = 8192 tokens, M = 1024, top-2, capacity 2048 → here all experts are local)
S, K, M, E_local, Cap = 8192, 2, 1024, 8, 2048
toks = torch.randn(S, M, device=dev).to(bf)
eidx = torch.stack([torch.randperm(E_local)[:K] for _ in range(S)]).to(dev)
sidx = torch.zeros(S, K, dtype=torch.int64)
eidx_cpu = eidx.cpu()
fill = [0] * E_local
for s_ in range(S):
    for k_ in range(K):
        e_ = int(eidx_cpu[s_, k_])
        sidx[s_, k_] = fill[e_] if fill[e_] < Cap else -1
        fill[e_] += 1
sidx = sidx.to(dev)
rows_buf = w.alloc(E_local * Cap * M * 2)
timed("moe_scatter_kernel<bf16> 8192 tok x top2 x 1024", lambda: C.moe_scatter(comm, rows_buf.buf, 0, toks.data_ptr(), eidx.data_ptr(), sidx.data_ptr(), 0, S, K, M, E_local, Cap, code, 64, stream),
      S * K * M * 2 * 2 + E_local * Cap * M * 2)
wts = torch.rand(S, K, device=dev)
res = torch.empty(S, M, device=dev, dtype=bf)
picked = torch.empty(S, K, M, device=dev, dtype=bf)
timed("moe_gather_kernel<bf16> 8192 tok x top2 x 1024 (+picked)", lambda: C.moe_gather(comm, rows_buf.buf, 0, res.data_ptr(), eidx.data_ptr(), sidx.data_ptr(), wts.data_ptr(), picked.data_ptr(), S, K, M,
                                                                                    E_local, Cap, code, 64, stream, False), S * K * M * 2 * 2 + S * M * 2)
for (G, Mm, Nn, Kk) in [(1, 16384, 4096, 1024), (1, 16384, 1024, 4096), (1, 8192, 8192, 8192)]:
    A = torch.randn(G, Mm, Kk, device=dev).to(bf)
    B = torch.randn(G, Nn, Kk, device=dev).to(bf)
    timed(f"grouped_gemm_tn_kernel G{G} M{Mm} N{Nn} K{Kk}", lambda: gemm.grouped_gemm_tn(A, B), (Mm * Kk + Nn * Kk + Mm * Nn) * 2 * G, flops=2.0 * G * Mm * Nn * Kk)
    timed(f"cuBLAS bmm            G{G} M{Mm} N{Nn} K{Kk}", lambda: torch.bmm(A, B.transpose(1, 2)), (Mm * Kk + Nn * Kk + Mm * Nn) * 2 * G, flops=2.0 * G * Mm * Nn * Kk)
torch.cuda.synchronize()
w.check()
peak = 3350.0  # GB/s, H100 SXM data sheet; MEASURED_PEAKS.json overrides
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:  # noqa: BLE001
    pass
clocks = sampler.stop()
for r in rows:
    r["frac_of_measured_hbm"] = r["GBps"] / peak
    print(json.dumps(r))
print(json.dumps({"clocks": clocks, "hbm_peak_GBps_measured": peak, "timing": "CUDA events, median of 5 (3 for the 138M-parameter optimizers), 512 MiB L2 flush before every launch"}))
