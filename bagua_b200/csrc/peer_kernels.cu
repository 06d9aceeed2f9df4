// Fused collective kernels over NVLink 4 / NVSwitch symmetric memory (sm_90a).
//
// These replace the reference's "kernel + separate NCCL call" sequences
// (rust/bagua-core/bagua-core-internal/src/comm_ops/*.rs, communicators/mod.rs:1121-1153): the reduction,
// the averaging scale, the dtype handling, the optimizer update and the data movement to/from the peers
// happen in ONE kernel that issues peer (P2P) or NVLS multicast loads/stores itself.
#include "dispatch.h"
#include "kernels.h"
#include "lamb.cuh"
#include "lars.cuh"
#include "lion.cuh"
#include "peer.cuh"

namespace bagua {
using namespace dev;

// ---------------------------------------------------------------------------------------------------------
// How a buffer of `total` 16-byte vectors is cut into `world` slices — rank r owns vectors [r·vpr, min((r+1)·vpr, total)) — and
// this thread's place in the grid-stride loops over them. A kernel builds it once, where it first needs it, and every phase reuses it.
struct Slicing {
    size_t total, vpr, tid, stride;
    __device__ __forceinline__ Slicing(size_t total_vecs, int world)
        : total(total_vecs),
          vpr((total_vecs + world - 1) / world),
          tid(static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x),
          stride(static_cast<size_t>(gridDim.x) * blockDim.x) {}
};

// The owned-slice schedule every reduction kernel runs. Each thread walks its share of slice `rank` grid-stride, U vectors per
// iteration, and issues every load of an iteration before it consumes any: U·P independent 16-byte peer loads in flight per thread
// is what keeps NVLink busy (NVLink latency is ~2 us: bandwidth = bytes in flight / latency, measured 7.5 GB/s per CTA without
// unrolling). load(raw, v) fills one Raw for vector v; consume(raw, v, j) gets it back with j = v − base, the index in the shard.
// ---------------------------------------------------------------------------------------------------------
template <int U, typename Raw, typename Load, typename Consume>
__device__ __forceinline__ void walk_owned_slice(const Slicing& sl, int rank, Load&& load, Consume&& consume) {
    const size_t base = static_cast<size_t>(rank) * sl.vpr;
    const size_t limit = (base + sl.vpr < sl.total ? base + sl.vpr : sl.total);  // exclusive end of my slice
    for (size_t j0 = base + sl.tid; j0 < limit; j0 += sl.stride * U) {
        Raw raw[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t v = j0 + u * sl.stride;
            if (v < limit) load(raw[u], v);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t v = j0 + u * sl.stride;
            if (v < limit) consume(raw[u], v, v - base);
        }
    }
}

// The owned-slice reduction: for every vector v of my slice, epi(v, j, acc) receives the fp32 sum over the P ranks' copies of
// src. The sum starts from my own copy and adds ranks rank+1, rank+2, … (mod P) in that order — the rotation also spreads the
// loads evenly over the links — or, with USE_MC, is one multimem.ld_reduce inside the switch.
template <typename T, int P, bool USE_MC, int U, typename Epi>
__device__ __forceinline__ void reduce_owned_slice(const PeerCtx& ctx, const PeerBuf& src, size_t off, const Slicing& sl, Epi&& epi) {
    using Raw = uint4[USE_MC ? 1 : P];
    walk_owned_slice<U, Raw>(
        sl, ctx.rank,
        [&](Raw& raw, size_t v) {
            if constexpr (USE_MC) {
                raw[0] = multimem_ld_reduce_add<T>(src.mc + off + v * 16);
            } else {
#pragma unroll
                for (int i = 0; i < P; ++i) raw[i] = ld_peer16(src.ptr[(ctx.rank + i) % P] + off + v * 16);
            }
        },
        [&](Raw& raw, size_t v, size_t j) {
            float acc[Vec16<T>::N];
            Vec16<T>::unpack(raw[0], acc);
#pragma unroll
            for (int i = 1; i < (USE_MC ? 1 : P); ++i) {
                float f[Vec16<T>::N];
                Vec16<T>::unpack(raw[i], f);
#pragma unroll
                for (int k = 0; k < Vec16<T>::N; ++k) acc[k] += f[k];
            }
            epi(v, j, acc);
        });
}

// Stores one 16-byte vector at index v of every rank's copy of dst: one multimem.st, or peer stores in the same rotated order as the
// loads. skip_self leaves my own copy alone.
template <int P, bool USE_MC>
__device__ __forceinline__ void publish16(const PeerCtx& ctx, const PeerBuf& dst, size_t off, size_t v, const uint4& val, bool skip_self = false) {
    if constexpr (USE_MC) {
        multimem_st16(dst.mc + off + v * 16, val);
    } else {
#pragma unroll
        for (int i = skip_self ? 1 : 0; i < P; ++i) st_peer16(dst.ptr[(ctx.rank + i) % P] + off + v * 16, val);
    }
}

// Column striping: f(v) for v = s·vpr + j of every slice s, with this thread's columns j ≡ (block, thread) mod grid — the columns
// walk_owned_slice gives it in slice s = rank. So CTA b touches the same column range of every slice in every phase, and the per-CTA
// barriers (CTA b of every rank) are all the synchronisation the kernels need; there is no grid-wide barrier.
template <int P, typename F>
__device__ __forceinline__ void for_each_striped(const Slicing& sl, F&& f) {
    for (size_t j = sl.tid; j < sl.vpr; j += sl.stride) {
#pragma unroll
        for (int s = 0; s < P; ++s) {
            const size_t v = static_cast<size_t>(s) * sl.vpr + j;
            if (v < sl.total) f(v);
        }
    }
}

// Vectors per thread per iteration of the pure reductions, and of the optimizer kernels, whose register budget is U·P·4 on top of
// the optimizer state.
template <int P, bool USE_MC>
constexpr int kReduceUnroll = USE_MC ? 8 : (P <= 2 ? 8 : (P <= 4 ? 4 : 2));
template <int P, bool USE_MC>
constexpr int kOptimizerUnroll = USE_MC ? 4 : (P <= 2 ? 4 : (P <= 4 ? 2 : 1));

// ---------------------------------------------------------------------------------------------------------
// allreduce, two-shot over peer pointers: rank r reduces slice r (reading it from every peer) and writes the
// result into slice r of every peer. src and dst may alias (in-place): slice r is only ever read and written
// by rank r between the two barriers.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P>
__global__ void __launch_bounds__(512) allreduce_twoshot_kernel(PeerCtx ctx, PeerBuf src, PeerBuf dst, size_t src_off,
                                                                size_t dst_off, size_t total_vecs, float scale) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        reduce_owned_slice<T, P, false, kReduceUnroll<P, false>>(ctx, src, src_off, Slicing(total_vecs, P), [&](size_t v, size_t, float* acc) {
#pragma unroll
            for (int k = 0; k < Vec16<T>::N; ++k) acc[k] *= scale;
            publish16<P, false>(ctx, dst, dst_off, v, Vec16<T>::pack(acc));
        });
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

// Same schedule through the switch: one multimem.ld_reduce returns the sum over all GPUs (reduced inside
// NVSwitch), one multimem.st lands the result on all GPUs. The world size is a runtime value here.
template <typename T>
__global__ void __launch_bounds__(512) allreduce_multimem_kernel(PeerCtx ctx, PeerBuf src, PeerBuf dst, size_t src_off,
                                                                 size_t dst_off, size_t total_vecs, float scale) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        walk_owned_slice<8, uint4>(
            Slicing(total_vecs, ctx.world), ctx.rank, [&](uint4& red, size_t v) { red = multimem_ld_reduce_add<T>(src.mc + src_off + v * 16); },
            [&](uint4& red, size_t v, size_t) {
                if (scale != 1.0f) {  // only then: unpacking and repacking may change NaN payloads
                    float f[Vec16<T>::N];
                    Vec16<T>::unpack(red, f);
#pragma unroll
                    for (int k = 0; k < Vec16<T>::N; ++k) f[k] *= scale;
                    red = Vec16<T>::pack(f);
                }
                multimem_st16(dst.mc + dst_off + v * 16, red);
            });
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

// ---------------------------------------------------------------------------------------------------------
// The two halves of the two-shot schedule as separate kernels, for hierarchical (multi-node) all-reduce:
//   reduce_scatter: rank r reduces slice r over the node's GPUs IN PLACE (its own buffer, slice r)   [intra-node, NVLink]
//   … the caller all-reduces slice r between nodes (NCCL / net plugin, 1/L of the bucket per GPU, all rails busy) …
//   all_gather:     rank r publishes slice r into every peer's buffer                                [intra-node, NVLink]
// Slice r of rank r's buffer is read and written by rank r only, so in-place is safe; the closing barrier of the
// first kernel ("everybody finished reading my other slices") is what allows the second one to overwrite them.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512) reduce_scatter_kernel(PeerCtx ctx, PeerBuf buf, size_t off, size_t total_vecs, float scale) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        char* mine = buf.ptr[ctx.rank] + off;
        reduce_owned_slice<T, P, USE_MC, kReduceUnroll<P, USE_MC>>(ctx, buf, off, Slicing(total_vecs, P), [&](size_t v, size_t, float* acc) {
#pragma unroll
            for (int k = 0; k < Vec16<T>::N; ++k) acc[k] *= scale;
            st_stream16(mine + v * 16, Vec16<T>::pack(acc));
        });
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512) all_gather_kernel(PeerCtx ctx, PeerBuf buf, size_t off, size_t total_vecs) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);  // nobody is still reading the slices that are about to be overwritten
    if (ok) {
        const char* mine = buf.ptr[ctx.rank] + off;
        walk_owned_slice<4, uint4>(
            Slicing(total_vecs, P), ctx.rank, [&](uint4& raw, size_t v) { raw = ld_stream16(mine + v * 16); },
            [&](uint4& raw, size_t v, size_t) { publish16<P, USE_MC>(ctx, buf, off, v, raw, /*skip_self=*/true); });  // mine is in place
        peer_barrier(ctx, e0 + 2);  // every slice has landed everywhere
    }
    store_epoch(ctx, e0 + 2);
}

// One-shot, push flavour, for latency-bound messages: every rank stores its message into slot [parity][rank]
// of every peer's staging area, ONE barrier, then reduces the P slots it received locally. The staging area is
// double-buffered by epoch parity, so no second barrier is needed (a rank can only be two calls ahead of a peer
// after that peer has left the call in between).
template <typename T, int P>
__global__ void __launch_bounds__(512) allreduce_oneshot_kernel(PeerCtx ctx, PeerBuf staging, size_t staging_off,
                                                                size_t slot_bytes, const char* in, char* out, size_t total_vecs,
                                                                float scale, uint32_t call_parity) {
    const uint32_t e0 = load_epoch(ctx);
    // Which half of the double-buffered staging area: a per-communicator CALL counter kept by the host (every rank issues the same
    // one-shot calls in the same order). It must not be derived from the per-CTA epochs: launches with different grids (and the
    // other kernel families, which advance epochs by 1 or 2) would put the CTAs of one rank out of step with each other.
    const size_t parity = (call_parity & 1u);
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (size_t v = tid; v < total_vecs; v += stride)
        publish16<P, false>(ctx, staging, staging_off + (parity * P + ctx.rank) * slot_bytes, v, ld_stream16(in + v * 16));
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        const char* mystage = staging.ptr[ctx.rank] + staging_off + parity * P * slot_bytes;
        for (size_t v = tid; v < total_vecs; v += stride) {
            float acc[Vec16<T>::N];
            Vec16<T>::unpack(ld_peer16(mystage + v * 16), acc);
#pragma unroll
            for (int p = 1; p < P; ++p) {
                float f[Vec16<T>::N];
                Vec16<T>::unpack(ld_peer16(mystage + p * slot_bytes + v * 16), f);
#pragma unroll
                for (int k = 0; k < Vec16<T>::N; ++k) acc[k] += f[k];
            }
#pragma unroll
            for (int k = 0; k < Vec16<T>::N; ++k) acc[k] *= scale;
            st_stream16(out + v * 16, Vec16<T>::pack(acc));
        }
    }
    store_epoch(ctx, e0 + 1);
}

// ---------------------------------------------------------------------------------------------------------
// The in-bucket optimizer rules, device side: Update<R> is the rule struct R of kernels.h (fp32 state of the owned shard, shard-local)
// with what the two kernels below need of it and of its parameters hp (R::Params). The kernels take R's fields and hp as kernel
// arguments of their own and build the rule inside: scalar pointer arguments are known to address global memory, and a struct
// argument's 8-byte alignment would let the compiler pair the loads of hp's fields, so either form compiles to other machine code.
//   setup(hp)         per-thread values, built once before the walk (Local; empty for most rules)
//   at_step(hp, t)    rebuilds the step-dependent fields of hp from the device step count t (loss scaling)
//   source(shard)     what the phase-B walk reads: the fp32 gradient shard, or the master for LAMB
//   coef(c)           the gradient coefficient of phase B
//   update<N>(...)    one 16-byte vector of the owned shard (N lanes at index j·N of the fp32 state): g[k]·scale is the gradient the
//                     update sees; w receives the new fp32 weights, which the caller publishes.
// ---------------------------------------------------------------------------------------------------------
template <class R>
struct Update;

template <>
struct Update<SgdRule> : SgdRule {
    struct Local {};
    __device__ __forceinline__ static Local setup(const Params&) { return {}; }
    __device__ __forceinline__ static void at_step(Params& hp, uint32_t t) { hp.first_step = t == 1u ? 1 : 0; }
    __device__ __forceinline__ const float* source(const float* shard) const { return shard; }
    __device__ __forceinline__ float coef(const float* c) const { return *c; }
    template <int N>
    __device__ __forceinline__ void update(Local&, const Params& hp, size_t j, const float* g, float scale, float* w) const {
        float m[N];
        float4* mp = reinterpret_cast<float4*>(master + j * N);
        float4* mo = reinterpret_cast<float4*>(momentum + j * N);
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            float4 a = mp[q];
            w[4 * q] = a.x, w[4 * q + 1] = a.y, w[4 * q + 2] = a.z, w[4 * q + 3] = a.w;
            if (hp.momentum != 0.f) {
                float4 bb = mo[q];
                m[4 * q] = bb.x, m[4 * q + 1] = bb.y, m[4 * q + 2] = bb.z, m[4 * q + 3] = bb.w;
            }
        }
#pragma unroll
        for (int k = 0; k < N; ++k) {
            float d = g[k] * scale + hp.weight_decay * w[k];
            if (hp.momentum != 0.f) {
                m[k] = hp.first_step ? d : hp.momentum * m[k] + (1.f - hp.dampening) * d;
                d = hp.nesterov ? d + hp.momentum * m[k] : m[k];
            }
            w[k] -= hp.lr * d;
        }
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            mp[q] = make_float4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
            if (hp.momentum != 0.f) mo[q] = make_float4(m[4 * q], m[4 * q + 1], m[4 * q + 2], m[4 * q + 3]);
        }
    }
};

// Adam / AdamW, update rule identical to flat_adam_kernel (multi_tensor.cu) / torch.optim.Adam[W]; inv_bc1 = 1/(1−β1^t),
// inv_sqrt_bc2 = 1/sqrt(1−β2^t).
template <>
struct Update<AdamRule> : AdamRule {
    struct Local {
        float inv_bc1, inv_sqrt_bc2;
    };
    __device__ __forceinline__ static Local setup(const Params& hp) { return {1.f / hp.bias_correction1, rsqrtf(hp.bias_correction2)}; }
    __device__ __forceinline__ static void at_step(Params& hp, uint32_t t) {
        hp.bias_correction1 = bias_correction(hp.beta1, t);
        hp.bias_correction2 = bias_correction(hp.beta2, t);
    }
    __device__ __forceinline__ const float* source(const float* shard) const { return shard; }
    __device__ __forceinline__ float coef(const float* c) const { return *c; }
    template <int N>
    __device__ __forceinline__ void update(Local& l, const Params& hp, size_t j, const float* g, float scale, float* w) const {
        float4* wp = reinterpret_cast<float4*>(master + j * N);
        float4* ap = reinterpret_cast<float4*>(exp_avg + j * N);
        float4* bp = reinterpret_cast<float4*>(exp_avg_sq + j * N);
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            float4 ww = wp[q], aa = ap[q], bb = bp[q];
            float wv[4] = {ww.x, ww.y, ww.z, ww.w}, av[4] = {aa.x, aa.y, aa.z, aa.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float gg = g[4 * q + k] * scale;
                if (hp.adamw)
                    wv[k] *= (1.f - hp.lr * hp.weight_decay);
                else
                    gg += hp.weight_decay * wv[k];
                av[k] = hp.beta1 * av[k] + (1.f - hp.beta1) * gg;
                bv[k] = hp.beta2 * bv[k] + (1.f - hp.beta2) * gg * gg;
                const float denom = sqrtf(bv[k]) * l.inv_sqrt_bc2 + hp.eps;
                wv[k] -= (hp.lr * l.inv_bc1) * (av[k] / denom);
                w[4 * q + k] = wv[k];
            }
            wp[q] = make_float4(wv[0], wv[1], wv[2], wv[3]);
            ap[q] = make_float4(av[0], av[1], av[2], av[3]);
            bp[q] = make_float4(bv[0], bv[1], bv[2], bv[3]);
        }
    }
};

// Lion (lion.cuh): x[k]·coef is the gradient, the fp32 master and exp_avg are updated in place; one moment instead of Adam's two, so
// 16 bytes of state per owned element instead of 24. No step-dependent parameter.
template <>
struct Update<LionRule> : LionRule {
    struct Local {};
    __device__ __forceinline__ static Local setup(const Params&) { return {}; }
    __device__ __forceinline__ static void at_step(Params&, uint32_t) {}
    __device__ __forceinline__ const float* source(const float* shard) const { return shard; }
    __device__ __forceinline__ float coef(const float* c) const { return *c; }
    template <int N>
    __device__ __forceinline__ void update(Local&, const Params& hp, size_t j, const float* x, float coef, float* w) const {
        float4* wp = reinterpret_cast<float4*>(master + j * N);
        float4* mp = reinterpret_cast<float4*>(exp_avg + j * N);
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            const float4 ww = wp[q], mm = mp[q];
            float wv[4] = {ww.x, ww.y, ww.z, ww.w}, mv[4] = {mm.x, mm.y, mm.z, mm.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                lion_apply(wv[k], mv[k], lion_grad(x[4 * q + k], coef), hp);
                w[4 * q + k] = wv[k];
            }
            wp[q] = make_float4(wv[0], wv[1], wv[2], wv[3]);
            mp[q] = make_float4(mv[0], mv[1], mv[2], mv[3]);
        }
    }
};

// segs = [nsegs][lo, hi, param] sorted by lo, disjoint, with gaps where the padding tensor lies. The last segment with lo ≤ e
// (−1: none), by bisection; the LAMB and LARS walks find it once per vector and advance it element by element, since a 16-byte
// vector may hold elements of several parameters.
__device__ __forceinline__ int lamb_segment_at(const int32_t* segs, int nsegs, int64_t e) {
    int lo = 0, hi = nsegs;  // first segment with lo > e
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (segs[3 * mid] <= e) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// LAMB's apply (phase B only, see lamb_ratio_kernel): w ← w − lr·r·u over the fp32 master, u recomputed from the stage-1 moments
// (lamb_direction, the same code that fed Σu²), r = ratio of the element's parameter (1 in the gaps of the segment table). The bias
// corrections at_step builds are the ones the moments kernel built from the same t. There is no gradient coefficient: with a vote,
// the kernel's coef is only the {coef, found_inf} pair the vote is read from.
template <>
struct Update<LambRule> : LambRule {
    struct Local {};
    __device__ __forceinline__ static Local setup(const Params&) { return {}; }
    __device__ __forceinline__ static void at_step(Params& hp, uint32_t t) {
        hp.bias_correction1 = bias_correction(hp.beta1, t);
        hp.bias_correction2 = bias_correction(hp.beta2, t);
    }
    __device__ __forceinline__ const float* source(const float*) const { return master; }
    __device__ __forceinline__ float coef(const float*) const { return 1.f; }
    template <int N>
    __device__ __forceinline__ void update(Local&, const Params& hp, size_t j, const float* w0, float, float* w) const {
        const float4* ap = reinterpret_cast<const float4*>(exp_avg + j * N);
        const float4* bp = reinterpret_cast<const float4*>(exp_avg_sq + j * N);
        int s = lamb_segment_at(segs, nsegs, static_cast<int64_t>(j * N));
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            const float4 aa = ap[q], bb = bp[q];
            const float av[4] = {aa.x, aa.y, aa.z, aa.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int64_t e = static_cast<int64_t>(j * N + 4 * q + k);
                while (s + 1 < nsegs && segs[3 * (s + 1)] <= e) ++s;
                const float r = (s >= 0 && e < segs[3 * s + 1]) ? ratio[segs[3 * s + 2]] : 1.f;
                w[4 * q + k] = lamb_apply(w0[4 * q + k], lamb_direction(w0[4 * q + k], av[k], bv[k], hp), r, hp);
            }
        }
        float4* wp = reinterpret_cast<float4*>(master + j * N);
#pragma unroll
        for (int q = 0; q < N / 4; ++q) wp[q] = make_float4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
    }
};

// LARS's momentum and apply (phase B only, the program of LAMB with a different pair: multi_tensor_lars_stage1 leaves fp64
// {Σw², Σg̃²} per block, lamb_ratio_kernel exchanges them per parameter into sums) from the gradient shard·coef (lars_grad, the code
// that fed Σg̃²; a null coef is 1). The trust of an element's parameter comes from the exchanged global sums and is taken again only
// when the walk enters another parameter (1 in the gaps of the segment table). No step-dependent parameter.
template <>
struct Update<LarsRule> : LarsRule {
    struct Local {
        float lt = 0.f;
        int cur = -2;  // parameter whose step size lt holds (−1: a gap)
    };
    __device__ __forceinline__ static Local setup(const Params&) { return {}; }
    __device__ __forceinline__ static void at_step(Params&, uint32_t) {}
    __device__ __forceinline__ const float* source(const float* shard) const { return shard; }
    __device__ __forceinline__ float coef(const float* c) const { return c != nullptr ? *c : 1.f; }
    template <int N>
    __device__ __forceinline__ void update(Local& l, const Params& hp, size_t j, const float* g, float c, float* w) const {
        float4* mp = reinterpret_cast<float4*>(master + j * N);
        float4* vp = reinterpret_cast<float4*>(momentum + j * N);
        int s = lamb_segment_at(segs, nsegs, static_cast<int64_t>(j * N));
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            const float4 ww = mp[q], vv = vp[q];
            float wv[4] = {ww.x, ww.y, ww.z, ww.w}, v[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int64_t e = static_cast<int64_t>(j * N + 4 * q + k);
                while (s + 1 < nsegs && segs[3 * (s + 1)] <= e) ++s;
                const int t = (s >= 0 && e < segs[3 * s + 1]) ? segs[3 * s + 2] : -1;
                if (t != l.cur) {
                    l.cur = t;
                    l.lt = lars_step_size(t >= 0 ? lars_trust(sums[2 * t], sums[2 * t + 1], hp) : 1.f, hp);
                }
                lars_apply(wv[k], v[k], lars_grad(g[4 * q + k], c), l.lt, hp);
                w[4 * q + k] = wv[k];
            }
            mp[q] = make_float4(wv[0], wv[1], wv[2], wv[3]);
            vp[q] = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
};

// ---------------------------------------------------------------------------------------------------------
// Gradient reduce-scatter  →  the rule (SGD, Adam, Lion) on the owned 1/P slice  →  all-gather of the updated WEIGHTS, in one
// kernel. Each rank keeps the fp32 master weights and the optimizer state only for its own slice (optimizer state is sharded P ways),
// the gradient bucket is zeroed for the next iteration on the way out, and the optimizer step overlaps the rest of backward because it
// runs inside the bucket's communication kernel.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P, bool USE_MC, class R, class... State>
__global__ void __launch_bounds__(512)
    allreduce_update_kernel(PeerCtx ctx, PeerBuf grads, PeerBuf weights, size_t g_off, size_t w_off, size_t total_vecs, State... state,
                            typename R::Params hp, float scale, int zero_grads) {
    const Update<R> rule{{state...}};
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    constexpr int N = Vec16<T>::N;
    const Slicing sl(total_vecs, P);
    if (ok) {
        auto local = rule.setup(hp);
        reduce_owned_slice<T, P, USE_MC, kOptimizerUnroll<P, USE_MC>>(ctx, grads, g_off, sl, [&](size_t v, size_t j, float* g) {
            float w[N];
            rule.template update<N>(local, hp, j, g, scale, w);
            publish16<P, USE_MC>(ctx, weights, w_off, v, Vec16<T>::pack(w));
        });
        ok = peer_barrier(ctx, e0 + 2);
    }
    if (ok && zero_grads) {
        // Block b of every peer has finished reading column-range b of all my slices: safe to clear them.
        char* mine = grads.ptr[ctx.rank] + g_off;
        for_each_striped<P>(sl, [&](size_t v) { st_stream16(mine + v * 16, make_uint4(0, 0, 0, 0)); });
    }
    store_epoch(ctx, e0 + 2);
}

// ---------------------------------------------------------------------------------------------------------
// Global-norm gradient clipping for the in-bucket optimizers. No shard may be updated before the norm over every bucket of every
// rank is known, so the single in-bucket kernel above becomes two phases around a norm exchange:
//   A  shard_grad_kernel, per bucket, inside backward on the comm stream: the owned-slice reduction (same order and the same
//      multimem / peer ld choice as allreduce_update_kernel) scaled by `scale` → the fp32 gradient of the owned slice in
//      `shard`; one fp64 Σx² per CTA in partials[block] (no atomics: reproducible, nothing to reset between steps); the bucket is
//      cleared after the closing barrier.
//   N  grad_norm_kernel, once per step: the rank's Σ over all partials (+ the parameters outside the buckets) → slot [rank] of
//      every peer's norm box → barrier → Σ over slots 0 .. P-1 in rank order, so every rank computes the same bits → total, coef.
//   B  shard_update_kernel, per bucket: the update of the shard scaled by coef (read from device memory: the host never sees
//      the norm) → all-gather of the weights → closing barrier, so no rank's trainer reads weights a peer is still writing.
// With ACCUM (gradient accumulation over micro-batches) phase A adds into the shard instead of overwriting it:
// s ← fl32(s_old + fl32(red·scale)), the product and the sum rounded separately (no FMA), and Σx² is taken over the new s. Every
// launch of an op walks the same vectors with the same grid, so the partials of the last micro-batch are Σs² of the accumulated
// shard and the norm exchange is unchanged. The old shard is loaded together with the peer loads of each unrolled iteration.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P, bool USE_MC, bool ACCUM>
__global__ void __launch_bounds__(512)
    shard_grad_kernel(PeerCtx ctx, PeerBuf grads, size_t g_off, size_t total_vecs, float* shard, double* partials, float scale, int zero_grads) {
    __shared__ double s_warp[512 / 32];
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    constexpr int N = Vec16<T>::N;
    const Slicing sl(total_vecs, P);
    double ss = 0.0;
    if (ok) {
        if constexpr (ACCUM) {
            // reduce_owned_slice's loads and sum, with the old shard loaded alongside (written out here: sharing them with
            // reduce_owned_slice changes the SASS of the kernels built on it)
            struct Raw {
                uint4 red[USE_MC ? 1 : P];
                float4 old[N / 4];
            };
            const size_t base = static_cast<size_t>(ctx.rank) * sl.vpr;
            walk_owned_slice<kReduceUnroll<P, USE_MC>, Raw>(
                sl, ctx.rank,
                [&](Raw& raw, size_t v) {
                    if constexpr (USE_MC) {
                        raw.red[0] = multimem_ld_reduce_add<T>(grads.mc + g_off + v * 16);
                    } else {
#pragma unroll
                        for (int i = 0; i < P; ++i) raw.red[i] = ld_peer16(grads.ptr[(ctx.rank + i) % P] + g_off + v * 16);
                    }
                    const float4* sp = reinterpret_cast<const float4*>(shard + (v - base) * N);
#pragma unroll
                    for (int q = 0; q < N / 4; ++q) raw.old[q] = sp[q];
                },
                [&](Raw& raw, size_t, size_t j) {
                    float g[N];
                    Vec16<T>::unpack(raw.red[0], g);
#pragma unroll
                    for (int i = 1; i < (USE_MC ? 1 : P); ++i) {
                        float f[N];
                        Vec16<T>::unpack(raw.red[i], f);
#pragma unroll
                        for (int k = 0; k < N; ++k) g[k] += f[k];
                    }
                    float4* sp = reinterpret_cast<float4*>(shard + j * N);
#pragma unroll
                    for (int q = 0; q < N / 4; ++q) {
                        const float o[4] = {raw.old[q].x, raw.old[q].y, raw.old[q].z, raw.old[q].w};
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            float& s = g[4 * q + k];
                            s = __fadd_rn(o[k], __fmul_rn(s, scale));
                            ss += static_cast<double>(s) * static_cast<double>(s);
                        }
                        sp[q] = make_float4(g[4 * q], g[4 * q + 1], g[4 * q + 2], g[4 * q + 3]);
                    }
                });
        } else {
            reduce_owned_slice<T, P, USE_MC, kReduceUnroll<P, USE_MC>>(ctx, grads, g_off, sl, [&](size_t, size_t j, float* g) {
                float4* sp = reinterpret_cast<float4*>(shard + j * N);
#pragma unroll
                for (int k = 0; k < N; ++k) {
                    g[k] *= scale;
                    ss += static_cast<double>(g[k]) * static_cast<double>(g[k]);
                }
#pragma unroll
                for (int q = 0; q < N / 4; ++q) sp[q] = make_float4(g[4 * q], g[4 * q + 1], g[4 * q + 2], g[4 * q + 3]);
            });
        }
        ok = peer_barrier(ctx, e0 + 2);
    }
    // the CTA's Σx² in a fixed order: a shuffle tree per warp, then the warps in index order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (unsigned w = 0; w < blockDim.x / 32; ++w) t += s_warp[w];
        partials[blockIdx.x] = t;
    }
    if (ok && zero_grads) {
        char* mine = grads.ptr[ctx.rank] + g_off;
        for_each_striped<P>(sl, [&](size_t v) { st_stream16(mine + v * 16, make_uint4(0, 0, 0, 0)); });
    }
    store_epoch(ctx, e0 + 2);
}

__device__ __forceinline__ void st_peer_f64(void* p, double v) {
    asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ double ld_peer_f64(const void* p) {
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}

// One CTA of kNormThreads threads. The box holds [2][kMaxPeers] doubles per rank, double-buffered by the host's call counter
// (`parity`) like the one-shot staging area: a rank can only write a half again two calls later, after every peer has left the
// call in between, so no closing barrier is needed. out = {total, coef}, coef = min(max_norm / (total + 1e-6), 1) in fp32 with
// torch's operation order (reciprocal, then the product); a NaN norm gives a NaN coef, as in torch.
constexpr int kNormThreads = 256;

// The exchange of both norm kernels: this rank's partials in a fixed order (+ *extra) → slot [rank] of every peer's box half →
// barrier `epoch` → the P slots of the own box added in rank order into `sum` (thread 0 only). False when the barrier failed.
__device__ __forceinline__ bool exchange_sumsq(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const double* partials, int nslots,
                                               const double* extra, uint32_t parity, uint32_t epoch, double& sum) {
    __shared__ double s_sum[kNormThreads];
    double s = 0.0;
    for (int i = threadIdx.x; i < nslots; i += kNormThreads) s += partials[i];
    s_sum[threadIdx.x] = s;
    __syncthreads();
#pragma unroll
    for (int o = kNormThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s_sum[threadIdx.x] += s_sum[threadIdx.x + o];
        __syncthreads();
    }
    const size_t half = box_off + static_cast<size_t>(parity & 1u) * kMaxPeers * sizeof(double);
    if (threadIdx.x < ctx.world) {
        const double mine = s_sum[0] + (extra != nullptr ? *extra : 0.0);
        st_peer_f64(box.ptr[threadIdx.x] + half + ctx.rank * sizeof(double), mine);
    }
    const bool ok = peer_barrier(ctx, epoch);
    if (ok && threadIdx.x == 0) {
        const char* mybox = box.ptr[ctx.rank] + half;
        sum = 0.0;
        for (int p = 0; p < ctx.world; ++p) sum += ld_peer_f64(mybox + p * sizeof(double));
    }
    return ok;
}

__global__ void __launch_bounds__(kNormThreads) grad_norm_kernel(PeerCtx ctx, PeerBuf box, size_t box_off, const double* partials, int nslots,
                                                                 const double* extra, float max_norm, uint32_t parity, float* out) {
    const uint32_t e0 = load_epoch(ctx);
    double sum = 0.0;
    const bool ok = exchange_sumsq(ctx, box, box_off, partials, nslots, extra, parity, e0 + 1, sum);
    if (threadIdx.x == 0) {
        float total = __int_as_float(0x7fc00000), coef = total;
        if (ok) {
            total = static_cast<float>(sqrt(sum));
            const float c = __fmul_rn(__frcp_rn(__fadd_rn(total, 1e-6f)), max_norm);
            coef = c > 1.f ? 1.f : c;
        }
        out[0] = total;
        out[1] = coef;
    }
    store_epoch(ctx, e0 + 1);
}

// The norm exchange of an optimizer with loss scaling: the same sum S, which is over the still-scaled gradient. Squares of finite
// fp32 values cannot overflow an fp64 sum, so S is non-finite iff some reduced gradient element is: that is the overflow vote, and
// every rank adds the same P numbers in the same order, so every rank casts the same one. out = {total, coef, found_inf} with
// total = sqrt(S)/scale (the norm of the unscaled gradient), coef = float(1/scale)·clip, clip as in grad_norm_kernel on `total`
// (1 when max_norm = +inf); *step, the optimizer's effective step count, advances unless the step is skipped. A failed barrier
// votes "skip" and leaves the counter alone.
__global__ void __launch_bounds__(kNormThreads) loss_scale_norm_kernel(PeerCtx ctx, PeerBuf box, size_t box_off, const double* partials, int nslots,
                                                                       const double* extra, const float* scale, float max_norm, uint32_t parity,
                                                                       float* out, uint32_t* step) {
    const uint32_t e0 = load_epoch(ctx);
    double sum = 0.0;
    const bool ok = exchange_sumsq(ctx, box, box_off, partials, nslots, extra, parity, e0 + 1, sum);
    if (threadIdx.x == 0) {
        float total = __int_as_float(0x7fc00000), coef = total, found_inf = 1.f;
        if (ok) {
            const double inv = 1.0 / static_cast<double>(*scale);
            total = static_cast<float>(sqrt(sum) * inv);
            float clip = 1.f;
            if (max_norm < INFINITY) {
                const float c = __fmul_rn(__frcp_rn(__fadd_rn(total, 1e-6f)), max_norm);
                clip = c > 1.f ? 1.f : c;
            }
            coef = __fmul_rn(static_cast<float>(inv), clip);
            found_inf = isfinite(sum) ? 0.f : 1.f;
            if (found_inf == 0.f) *step += 1u;
        }
        out[0] = total;
        out[1] = coef;
        out[2] = found_inf;
    }
    store_epoch(ctx, e0 + 1);
}

// Phase B: the shard's own vectors, U-unrolled like the reduction walk (all shard loads of an iteration before any update).
template <typename T, int P, bool USE_MC, typename Update>
__device__ __forceinline__ void update_owned_shard(const PeerCtx& ctx, const PeerBuf& weights, size_t w_off, const Slicing& sl, const float* shard,
                                                   Update&& update) {
    constexpr int N = Vec16<T>::N;
    using Raw = float4[N / 4];
    walk_owned_slice<kOptimizerUnroll<P, USE_MC>, Raw>(
        sl, ctx.rank,
        [&](Raw& raw, size_t v) {
            const float4* sp = reinterpret_cast<const float4*>(shard + (v - static_cast<size_t>(ctx.rank) * sl.vpr) * N);
#pragma unroll
            for (int q = 0; q < N / 4; ++q) raw[q] = sp[q];
        },
        [&](Raw& raw, size_t v, size_t j) {
            float g[N], w[N];
#pragma unroll
            for (int q = 0; q < N / 4; ++q) g[4 * q] = raw[q].x, g[4 * q + 1] = raw[q].y, g[4 * q + 2] = raw[q].z, g[4 * q + 3] = raw[q].w;
            update(j, g, w);
            publish16<P, USE_MC>(ctx, weights, w_off, v, Vec16<T>::pack(w));
        });
}

// Phase B of every rule: the update of the owned shard from rule.source(shard) with the coefficient rule.coef(coef), the all-gather of
// the weights, the closing barrier.
//
// VOTE (loss scaling): `coef` addresses {coef, found_inf} of loss_scale_norm_kernel and *step is the effective step count t that
// includes this step. The vote has the same bits on every rank, so the branch on it is uniform across ranks and CTAs: a skipped step
// touches no state, publishes nothing and only takes the closing barrier; a taken one rebuilds the step-dependent fields of the rule
// from t. Without VOTE `step` is not read and the rule's parameters are the host's.
template <typename T, int P, bool USE_MC, bool VOTE, class R, class... State>
__global__ void __launch_bounds__(512) shard_update_kernel(PeerCtx ctx, PeerBuf weights, size_t w_off, size_t total_vecs, const float* shard,
                                                           const float* coef, State... state, typename R::Params hp, const uint32_t* step) {
    const Update<R> rule{{state...}};
    const uint32_t e0 = load_epoch(ctx);
    const float c = rule.coef(coef);
    bool skip = false;
    if constexpr (VOTE) {
        skip = coef[1] != 0.f;
        rule.at_step(hp, *step);
    }
    if (!skip) {
        auto local = rule.setup(hp);
        update_owned_shard<T, P, USE_MC>(ctx, weights, w_off, Slicing(total_vecs, P), rule.source(shard),
                                         [&](size_t j, const float* g, float* w) { rule.template update<Vec16<T>::N>(local, hp, j, g, c, w); });
    }
    peer_barrier(ctx, e0 + 1);
    store_epoch(ctx, e0 + 1);
}

// ---------------------------------------------------------------------------------------------------------
// In-bucket LAMB. Its trust ratio is a norm over a whole parameter, and the owned slices cut parameters anywhere, so after phase A
// (shard_grad_kernel, unchanged) step() runs: the moments of each shard (multi_tensor_lamb_stage1 over the shard's segments, one
// parameter ∩ owned slice each, leaving fp64 {Σw², Σu²} per block) → lamb_ratio_kernel, once per step → shard_update_kernel per bucket.
//
// lamb_ratio_kernel, one CTA: parameter t's local pair is the sum of its segment's block pairs in block order; the pairs go to slot
// [rank][t] of every peer's box, double-buffered by the op's call counter like grad_norm_kernel (a rank writes a half again two calls
// later, after every peer has left the call in between), then the barrier, then the P slots in rank order → the same bits everywhere.
// ---------------------------------------------------------------------------------------------------------
constexpr int kRatioThreads = 512;
__global__ void __launch_bounds__(kRatioThreads) lamb_ratio_kernel(PeerCtx ctx, PeerBuf box, size_t box_off, const uint64_t* seg_ptr, const int32_t* seg_nblk,
                                                                   int nparams, uint32_t parity, float* ratio, double* sums) {
    const uint32_t e0 = load_epoch(ctx);
    const size_t half = box_off + static_cast<size_t>(parity & 1u) * kMaxPeers * nparams * 2 * sizeof(double);
    for (int t = threadIdx.x; t < nparams; t += blockDim.x) {
        const double* part = reinterpret_cast<const double*>(seg_ptr[t]);
        double a = 0.0, b = 0.0;
        for (int k = 0; k < seg_nblk[t]; ++k) a += part[2 * k], b += part[2 * k + 1];
        const size_t slot = half + (static_cast<size_t>(ctx.rank) * nparams + t) * 2 * sizeof(double);
        for (int p = 0; p < ctx.world; ++p) {
            st_peer_f64(box.ptr[p] + slot, a);
            st_peer_f64(box.ptr[p] + slot + sizeof(double), b);
        }
    }
    const bool ok = peer_barrier(ctx, e0 + 1);
    const char* mybox = box.ptr[ctx.rank] + half;
    for (int t = threadIdx.x; t < nparams; t += blockDim.x) {
        double a = __longlong_as_double(0x7ff8000000000000ll), b = a;
        if (ok) {
            a = 0.0, b = 0.0;
            for (int p = 0; p < ctx.world; ++p) {
                const char* slot = mybox + (static_cast<size_t>(p) * nparams + t) * 2 * sizeof(double);
                a += ld_peer_f64(slot);
                b += ld_peer_f64(slot + sizeof(double));
            }
        }
        ratio[t] = ok ? lamb_ratio(a, b) : __int_as_float(0x7fc00000);
        sums[2 * t] = a;
        sums[2 * t + 1] = b;
    }
    store_epoch(ctx, e0 + 1);
}


// Publication of an fp32 shard as the bucket's weights: the walk of the update kernels with a copy in place of the update, so
// Vec16<T>::pack(src) lands in every rank's copy of the owned slice. The weight EMA swaps its shard in with it and the master back
// out; every update kernel publishes pack(master), so publishing the master restores the live weights bit for bit. Unlike an
// update, which runs where the peers have passed the gradient exchange, this can follow any work of the trainer (an evaluation
// pass on one rank while another has finished its own): the opening barrier waits until no rank still reads the weights.
template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512) shard_publish_kernel(PeerCtx ctx, PeerBuf weights, size_t w_off, size_t total_vecs, const float* src) {
    const uint32_t e0 = load_epoch(ctx);
    const bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        update_owned_shard<T, P, USE_MC>(ctx, weights, w_off, Slicing(total_vecs, P), src, [](size_t, const float* s, float* w) {
#pragma unroll
            for (int k = 0; k < Vec16<T>::N; ++k) w[k] = s[k];
        });
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

// ---------------------------------------------------------------------------------------------------------
// Decentralized SGD, shift_one: out = (mine + peer's weights) / 2, the peer's bucket being read straight over
// NVLink (replaces grouped send/recv + average kernel, comm_ops/decentralized_full_precision_synchronous.rs:81-92).
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(512)
    peer_average_kernel(PeerCtx ctx, PeerBuf weights, size_t off, int peer, char* out, size_t total_vecs) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
        const char* mine = weights.ptr[ctx.rank] + off;
        const char* theirs = weights.ptr[peer] + off;
        for (size_t v = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < total_vecs; v += stride) {
            float a[Vec16<T>::N], b[Vec16<T>::N];
            const uint4 rb = ld_peer16(theirs + v * 16);
            Vec16<T>::unpack(ld_stream16(mine + v * 16), a);
            Vec16<T>::unpack(rb, b);
#pragma unroll
            for (int k = 0; k < Vec16<T>::N; ++k) a[k] = (a[k] + b[k]) * 0.5f;
            st_stream16(out + v * 16, Vec16<T>::pack(a));
        }
        // nobody may overwrite its weights (copy-back / optimizer step) before every reader is done
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}


// ---------------------------------------------------------------------------------------------------------
// Asynchronous model averaging: ONE launch per round (the reference runs clone + a 1-byte MIN allreduce + host sync +
// allreduce + apply kernel + two more host syncs, comm_ops/decentralized_full_precision_asynchronous.rs:97-162).
//
//   1. vote + snapshot   every CTA deposits "go / stop" in every peer's vote area and copies its columns of the weights
//                        into the symmetric `snap` buffer; the opening barrier carries the votes: if ANY rank wants to
//                        stop, every rank skips the round and reports it (that is the abort negotiation — no NCCL, no
//                        .item()).
//   2. mean              rank r averages slice r of the P snapshots (peer loads or multimem.ld_reduce) and publishes it
//                        into every rank's `avg` buffer (peer stores or multimem.st); barrier.
//   3. apply             w += mean − snapshot, but only while holding the device-side WEIGHT GATE: a word the trainer's
//                        stream acquires before a forward pass and releases after the optimizer step (gate kernels below).
//                        So the delta lands between two iterations — never under a forward/backward (what the reference's
//                        host mutex guarantees) and never interleaved with the optimizer's read-modify-write (which the
//                        reference does not guarantee) — without any host synchronisation, and a straggling peer only
//                        delays this background kernel, never the trainer.
//
// All three phases are column-striped (for_each_striped, and the owned-slice walk for phase 2), so the per-CTA barriers are all
// the synchronisation needed; there is no grid-wide barrier.
// gate words: [0] state (0 free, 1 trainer, 2 averaging), [1] "averaging is waiting" (fairness), [2] CTAs finished,
// [3] CTAs past the last cross-rank barrier, [4] decision of the acquiring CTA (1 apply, 2 skip).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512)
    async_average_kernel(PeerCtx ctx, char* w, PeerBuf snap, size_t snap_off, PeerBuf avg, size_t avg_off, size_t total_vecs, uint32_t seq,
                         int go, uint32_t* gate, unsigned long long gate_timeout_ns, volatile int* status) {
    __shared__ uint32_t s_votes[kMaxPeers];
    __shared__ int s_gate;
    constexpr int N = Vec16<T>::N;
    const uint32_t e0 = load_epoch(ctx);
    const Slicing sl(total_vecs, P);
    char* my_snap = snap.ptr[ctx.rank] + snap_off;
    // 1: snapshot (weights may be mid-update by the optimizer on another stream: every 16-byte vector is still a value the
    //    weight had at some instant, which is all the element-wise averaging algebra needs)
    for_each_striped<P>(sl, [&](size_t v) { st_stream16(my_snap + v * 16, ld_peer16(w + v * 16)); });
    bool ok = peer_barrier_vote(ctx, e0 + 1, (seq << 1) | (go ? 1u : 0u), s_votes);
    bool all_go = true;
    if (ok) {
#pragma unroll
        for (int p = 0; p < P; ++p) {
            if ((s_votes[p] >> 1) != (seq & 0x7fffffffu)) ok = false;  // a peer is in a different round: protocol violation
            all_go = all_go && (s_votes[p] & 1u);
        }
        if (!ok && threadIdx.x == 0) raise_error(ctx, 4);
    }
    if (ok && all_go) {
        // 2: mean of my slice → everybody's avg buffer
        const float inv = 1.0f / P;
        reduce_owned_slice<T, P, USE_MC, kReduceUnroll<P, USE_MC>>(ctx, snap, snap_off, sl, [&](size_t v, size_t, float* acc) {
#pragma unroll
            for (int k = 0; k < N; ++k) acc[k] *= inv;
            publish16<P, USE_MC>(ctx, avg, avg_off, v, Vec16<T>::pack(acc));
        });
        ok = peer_barrier(ctx, e0 + 2);
        if (ok) {
            // 3: take the weight gate — by the LAST CTA to get here, i.e. once everything that is left is local work, so the
            //    trainer (who lets a waiting averaging kernel go first) never waits on another rank. Bounded: if the trainer keeps
            //    the gate (e.g. an evaluation loop that never steps the optimizer) the whole kernel skips this round's apply.
            if (threadIdx.x == 0) {
                int got = 0;
                if (gate == nullptr) {
                    got = 1;
                } else if (atomicAdd(&gate[3], 1u) + 1u == gridDim.x) {
                    atomicExch(&gate[1], 1u);
                    const unsigned long long t0 = globaltimer_ns();
                    uint32_t spins = 0;
                    for (;;) {
                        if (atomicCAS(&gate[0], 0u, 2u) == 0u) {
                            got = 1;
                            break;
                        }
                        if ((++spins & 0xff) == 0 && (*ctx.abort != 0 || globaltimer_ns() - t0 > gate_timeout_ns)) break;
                        __nanosleep(200);
                    }
                    __threadfence();
                    atomicExch(&gate[4], got ? 1u : 2u);  // decision for the sibling CTAs
                } else {
                    const unsigned long long t0 = globaltimer_ns();
                    uint32_t d = 0, spins = 0;
                    while ((d = ld_acquire_gpu_u32(&gate[4])) == 0u) {
                        if ((++spins & 0xff) == 0 && globaltimer_ns() - t0 > 2 * gate_timeout_ns + ctx.timeout_ns) break;
                        __nanosleep(200);
                    }
                    got = d == 1u;
                }
                s_gate = got;
            }
            __syncthreads();
            if (s_gate) {
                const char* my_avg = avg.ptr[ctx.rank] + avg_off;
                for_each_striped<P>(sl, [&](size_t v) {
                    float a[N], sn[N], cur[N];
                    Vec16<T>::unpack(ld_peer16(my_avg + v * 16), a);       // written by the slice owner during this kernel
                    Vec16<T>::unpack(ld_stream16(my_snap + v * 16), sn);  // written by this very thread in phase 1
                    Vec16<T>::unpack(ld_peer16(w + v * 16), cur);         // the weights as they are NOW
#pragma unroll
                    for (int k = 0; k < N; ++k) cur[k] += a[k] - sn[k];
                    st_stream16(w + v * 16, Vec16<T>::pack(cur));
                });
            }
            if (gate != nullptr) {
                __syncthreads();
                if (threadIdx.x == 0) {
                    __threadfence();
                    if (atomicAdd(&gate[2], 1u) == gridDim.x - 1) {  // last CTA out hands the weights back and re-arms the words
                        gate[2] = 0u, gate[3] = 0u, gate[4] = 0u;
                        __threadfence();
                        atomicCAS(&gate[0], 2u, 0u);
                        atomicExch(&gate[1], 0u);
                    }
                }
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *status = !ok ? -1 : (all_go ? 1 : 0);
        __threadfence_system();
    }
    if (ok) store_epoch(ctx, e0 + 2);
}

// The trainer's side of the weight gate, enqueued on the compute stream. acquire: let a waiting averaging kernel go first
// (fairness word), then CAS free→trainer; bounded so that a wedged averaging kernel cannot hang training. release: plain store.
__global__ void gate_acquire_kernel(uint32_t* gate, unsigned long long timeout_ns) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const unsigned long long t0 = globaltimer_ns();
    uint32_t spins = 0;
    while (ld_acquire_gpu_u32(&gate[1]) != 0u && ld_acquire_gpu_u32(&gate[0]) != 1u) {
        if ((++spins & 0xff) == 0 && globaltimer_ns() - t0 > timeout_ns) break;
        __nanosleep(100);
    }
    for (;;) {
        const uint32_t prev = atomicCAS(&gate[0], 0u, 1u);
        if (prev == 0u || prev == 1u) break;
        if ((++spins & 0xff) == 0 && globaltimer_ns() - t0 > timeout_ns) {
            atomicExch(&gate[0], 1u);  // give up waiting: training goes on (the averaging kernel sees its CAS fail and skips)
            break;
        }
        __nanosleep(100);
    }
    __threadfence();
}
__global__ void gate_release_kernel(uint32_t* gate) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    __threadfence();
    atomicCAS(&gate[0], 1u, 0u);
}

// A bare cross-GPU barrier (1 CTA) — used for arena hand-over and by tests.
__global__ void peer_barrier_kernel(PeerCtx ctx) {
    const uint32_t e0 = load_epoch(ctx);
    peer_barrier(ctx, e0 + 1);
    store_epoch(ctx, e0 + 1);
}

// ---------------------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------------------
namespace {
constexpr const char* kFamily = "peer reduction kernels";

// The checks every peer launcher makes; returns the number of 16-byte vectors to process.
size_t peer_vecs(const char* what, size_t bytes, size_t off_a, size_t off_b, int nblocks) {
    if ((bytes | off_a | off_b) % 16) throw std::runtime_error(std::string("bagua: ") + what + " needs 16-byte aligned size/offsets");
    if (nblocks < 1 || nblocks > kMaxCommBlocks) throw std::runtime_error("bagua: peer kernel grid must be 1.." + std::to_string(kMaxCommBlocks));
    return bytes / 16;
}

// The checks of a rule's parameters, made by both of its launchers.
template <class Params>
void check_params(const char*, const Params&) {}
void check_params(const char* what, const AdamParams& hp) {
    if (hp.amsgrad) throw std::runtime_error(std::string("bagua: ") + what + " does not implement amsgrad");
}
}  // namespace

void launch_allreduce(const PeerCtx& ctx, const PeerBuf& src, const PeerBuf& dst, size_t src_off, size_t dst_off,
                      size_t bytes, int dtype, float scale, int variant, int nblocks, int nthreads, cudaStream_t stream) {
    const size_t vecs = peer_vecs("allreduce", bytes, src_off, dst_off, nblocks);
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        using T = decltype(tag);
        if (variant == AR_MULTIMEM) {
            if (!src.mc || !dst.mc) throw std::runtime_error("bagua: multimem allreduce requested but no multicast mapping");
            allreduce_multimem_kernel<T><<<nblocks, nthreads, 0, stream>>>(ctx, src, dst, src_off, dst_off, vecs, scale);
        } else {
            dispatch_world(ctx.world, [&](auto pw) {
                allreduce_twoshot_kernel<T, decltype(pw)::value><<<nblocks, nthreads, 0, stream>>>(ctx, src, dst, src_off, dst_off, vecs, scale);
            });
        }
    });
    check_launch("allreduce");
}

void launch_allreduce_oneshot(const PeerCtx& ctx, const PeerBuf& staging, size_t staging_off, size_t slot_bytes, const void* in, void* out,
                              size_t bytes, int dtype, float scale, int nblocks, int nthreads, cudaStream_t stream, uint32_t call_parity) {
    const size_t vecs = peer_vecs("one-shot allreduce", bytes, 0, 0, nblocks);
    if (bytes > slot_bytes) throw std::runtime_error("bagua: one-shot allreduce message larger than its staging slot");
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            allreduce_oneshot_kernel<decltype(tag), decltype(pw)::value><<<nblocks, nthreads, 0, stream>>>(
                ctx, staging, staging_off, slot_bytes, static_cast<const char*>(in), static_cast<char*>(out), vecs, scale, call_parity);
        });
    });
    check_launch("allreduce_oneshot");
}


void launch_reduce_scatter(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, float scale, bool use_multimem, int nblocks,
                           int nthreads, cudaStream_t stream) {
    const size_t vecs = peer_vecs("reduce_scatter", bytes, off, 0, nblocks);
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                reduce_scatter_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value><<<nblocks, nthreads, 0, stream>>>(ctx, buf, off, vecs,
                                                                                                                               scale);
            });
        });
    });
    check_launch("reduce_scatter");
}

void launch_all_gather(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, bool use_multimem, int nblocks, int nthreads,
                       cudaStream_t stream) {
    const size_t vecs = peer_vecs("all_gather", bytes, off, 0, nblocks);
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                all_gather_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value><<<nblocks, nthreads, 0, stream>>>(ctx, buf, off, vecs);
            });
        });
    });
    check_launch("all_gather");
}


void launch_shard_grad(const PeerCtx& ctx, const PeerBuf& grads, size_t g_off, size_t bytes, int dtype, float* shard, double* partials, float scale,
                       bool zero_grads, bool use_multimem, int nblocks, int nthreads, cudaStream_t stream, bool accumulate) {
    const size_t vecs = peer_vecs("shard_grad", bytes, g_off, 0, nblocks);
    if (nthreads % 32 || nthreads > 512) throw std::runtime_error("bagua: shard_grad needs whole warps, at most 512 threads");
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                dispatch_flag(accumulate, [&](auto acc) {
                    shard_grad_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value, decltype(acc)::value><<<nblocks, nthreads, 0, stream>>>(
                        ctx, grads, g_off, vecs, shard, partials, scale, zero_grads ? 1 : 0);
                });
            });
        });
    });
    check_launch("shard_grad");
}

// An accumulating phase-A op first launches its ACCUM instantiation mid-training, possibly while a peer kernel spins (see
// preload_gate_kernels): the op loads it when it is built.
void preload_shard_grad_accum(int dtype, int world, bool use_multimem) {
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                cudaFuncAttributes a;
                cudaFuncGetAttributes(&a, shard_grad_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value, true>);
            });
        });
    });
    cudaGetLastError();
}

void launch_grad_norm(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const double* partials, int nslots, const double* extra, float max_norm,
                      uint32_t parity, float* out, cudaStream_t stream) {
    if (box_off % 8) throw std::runtime_error("bagua: grad_norm box offset must be 8-byte aligned");
    grad_norm_kernel<<<1, kNormThreads, 0, stream>>>(ctx, box, box_off, partials, nslots, extra, max_norm, parity, out);
    check_launch("grad_norm");
}

void launch_loss_scale_norm(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const double* partials, int nslots, const double* extra,
                            const float* scale, float max_norm, uint32_t parity, float* out, uint32_t* step, cudaStream_t stream) {
    if (box_off % 8) throw std::runtime_error("bagua: loss_scale_norm box offset must be 8-byte aligned");
    if (scale == nullptr || step == nullptr) throw std::runtime_error("bagua: loss_scale_norm needs the loss scale and the step counter");
    loss_scale_norm_kernel<<<1, kNormThreads, 0, stream>>>(ctx, box, box_off, partials, nslots, extra, scale, max_norm, parity, out, step);
    check_launch("loss_scale_norm");
}


void launch_lamb_ratio(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const uint64_t* seg_ptr, const int32_t* seg_nblk, int nparams,
                       uint32_t parity, float* ratio, double* sums, cudaStream_t stream) {
    if (box_off % 8) throw std::runtime_error("bagua: lamb_ratio box offset must be 8-byte aligned");
    if (nparams < 1) throw std::runtime_error("bagua: lamb_ratio needs at least one parameter");
    lamb_ratio_kernel<<<1, kRatioThreads, 0, stream>>>(ctx, box, box_off, seg_ptr, seg_nblk, nparams, parity, ratio, sums);
    check_launch("lamb_ratio");
}

template <class R>
void launch_fused_update(const PeerCtx& ctx, const PeerBuf& grads, const PeerBuf& weights, size_t g_off, size_t w_off, size_t bytes, int dtype,
                         const R& rule, const typename R::Params& hp, float scale, bool zero_grads, bool use_multimem, int nblocks, int nthreads,
                         cudaStream_t stream) {
    const size_t vecs = peer_vecs(R::kFused, bytes, g_off, w_off, nblocks);
    check_params(R::kFused, hp);
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                std::apply(
                    [&](auto... state) {
                        allreduce_update_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value, R, decltype(state)...><<<nblocks, nthreads, 0, stream>>>(
                            ctx, grads, weights, g_off, w_off, vecs, state..., hp, scale, zero_grads ? 1 : 0);
                    },
                    rule.fields());
            });
        });
    });
    check_launch(R::kFused);
}
#define BAGUA_FUSED_UPDATE(R)                                                                                                                     \
    template void launch_fused_update(const PeerCtx&, const PeerBuf&, const PeerBuf&, size_t, size_t, size_t, int, const R&, const R::Params&, float, bool, bool, int, \
                                      int, cudaStream_t);
BAGUA_FUSED_UPDATE(SgdRule)
BAGUA_FUSED_UPDATE(AdamRule)
BAGUA_FUSED_UPDATE(LionRule)
#undef BAGUA_FUSED_UPDATE

template <class R>
void launch_shard_update(const PeerCtx& ctx, const PeerBuf& weights, size_t w_off, size_t bytes, int dtype, const float* shard, const float* coef,
                         const R& rule, const typename R::Params& hp, bool use_multimem, int nblocks, int nthreads, cudaStream_t stream,
                         const uint32_t* step) {
    const size_t vecs = peer_vecs(R::kShard, bytes, w_off, 0, nblocks);
    check_params(R::kShard, hp);
    if (step != nullptr && coef == nullptr) throw std::runtime_error(std::string("bagua: ") + R::kShard + " with a vote needs {coef, found_inf}");
    if constexpr (std::is_same_v<R, LionRule>) {
        if (coef == nullptr) throw std::runtime_error("bagua: shard_lion needs a gradient coefficient ({coef, found_inf} with a vote)");
    }
    if constexpr (std::is_same_v<R, LambRule>) {  // LAMB reads no coefficient: its coef is the vote
        if (coef != nullptr && step == nullptr) throw std::runtime_error("bagua: shard_lamb takes the vote and the step counter together");
    }
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                dispatch_flag(step != nullptr, [&](auto vote) {
                    std::apply(
                        [&](auto... state) {
                            shard_update_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value, decltype(vote)::value, R, decltype(state)...>
                                <<<nblocks, nthreads, 0, stream>>>(ctx, weights, w_off, vecs, shard, coef, state..., hp, step);
                        },
                        rule.fields());
                });
            });
        });
    });
    check_launch(R::kShard);
}
#define BAGUA_SHARD_UPDATE(R)                                                                                                                    \
    template void launch_shard_update(const PeerCtx&, const PeerBuf&, size_t, size_t, int, const float*, const float*, const R&, const R::Params&, bool, int, \
                                      int, cudaStream_t, const uint32_t*);
BAGUA_SHARD_UPDATE(SgdRule)
BAGUA_SHARD_UPDATE(AdamRule)
BAGUA_SHARD_UPDATE(LionRule)
BAGUA_SHARD_UPDATE(LambRule)
BAGUA_SHARD_UPDATE(LarsRule)
#undef BAGUA_SHARD_UPDATE


void launch_shard_publish(const PeerCtx& ctx, const PeerBuf& weights, size_t w_off, size_t bytes, int dtype, const float* src, bool use_multimem,
                          int nblocks, int nthreads, cudaStream_t stream) {
    const size_t vecs = peer_vecs("shard_publish", bytes, w_off, 0, nblocks);
    if (vecs == 0) return;
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                shard_publish_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value><<<nblocks, nthreads, 0, stream>>>(ctx, weights, w_off, vecs,
                                                                                                                              src);
            });
        });
    });
    check_launch("shard_publish");
}

// Loaded when the op is built, like the accumulating phase-A kernel: its first launch comes mid-training.
void preload_shard_publish(int dtype, int world, bool use_multimem) {
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                cudaFuncAttributes a;
                cudaFuncGetAttributes(&a, shard_publish_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value>);
            });
        });
    });
    cudaGetLastError();
}

void launch_peer_average(const PeerCtx& ctx, const PeerBuf& weights, size_t off, int peer, void* out, size_t bytes, int dtype,
                         int nblocks, int nthreads, cudaStream_t stream) {
    const size_t vecs = peer_vecs("peer_average", bytes, off, 0, nblocks);
    if (peer < 0 || peer >= ctx.world) throw std::runtime_error("bagua: peer_average peer rank out of range");
    dispatch_float(dtype, kFamily, [&](auto tag) {
        peer_average_kernel<decltype(tag)><<<nblocks, nthreads, 0, stream>>>(ctx, weights, off, peer, static_cast<char*>(out), vecs);
    });
    check_launch("peer_average");
}

void launch_async_average(const PeerCtx& ctx, void* w, const PeerBuf& snap, size_t snap_off, const PeerBuf& avg, size_t avg_off, size_t bytes, int dtype,
                          uint32_t seq, bool go, uint32_t* gate, unsigned long long gate_timeout_ns, int* status, bool use_multimem, int nblocks, int nthreads,
                          cudaStream_t stream) {
    const size_t vecs = peer_vecs("async_average", bytes, snap_off, avg_off, nblocks);
    if (vecs == 0) return;
    if (use_multimem && (!snap.mc || !avg.mc)) throw std::runtime_error("bagua: multimem async_average requested but no multicast mapping");
    dispatch_float(dtype, kFamily, [&](auto tag) {
        dispatch_world(ctx.world, [&](auto pw) {
            dispatch_mc(use_multimem, [&](auto mc) {
                async_average_kernel<decltype(tag), decltype(pw)::value, decltype(mc)::value><<<nblocks, nthreads, 0, stream>>>(
                    ctx, static_cast<char*>(w), snap, snap_off, avg, avg_off, vecs, seq, go ? 1 : 0, gate, gate_timeout_ns, status);
            });
        });
    });
    check_launch("async_average");
}

// CUDA loads kernels lazily, and loading one while another kernel is RUNNING can wait for that kernel to finish (programming guide,
// "Lazy Loading": concurrent execution is not guaranteed while a kernel still has to be loaded). The trainer-side gate kernels are
// launched precisely while an averaging kernel may be parked in front of the gate waiting for them — so they are loaded up front.
void preload_gate_kernels() {
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, gate_acquire_kernel);
    cudaFuncGetAttributes(&a, gate_release_kernel);
    cudaGetLastError();
}

void launch_gate_acquire(uint32_t* gate, unsigned long long timeout_ns, cudaStream_t stream) {
    gate_acquire_kernel<<<1, 32, 0, stream>>>(gate, timeout_ns);
    check_launch("gate_acquire");
}
void launch_gate_release(uint32_t* gate, cudaStream_t stream) {
    gate_release_kernel<<<1, 32, 0, stream>>>(gate);
    check_launch("gate_release");
}

void launch_peer_barrier(const PeerCtx& ctx, cudaStream_t stream) {
    peer_barrier_kernel<<<1, 32, 0, stream>>>(ctx);
    check_launch("peer_barrier");
}

}  // namespace bagua
