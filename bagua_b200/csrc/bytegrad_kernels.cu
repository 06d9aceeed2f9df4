// Quantised (MinMaxUInt8) collectives fused into single persistent kernels over NVSwitch peer memory.
//
// Reference pipeline per ByteGrad bucket (comm_ops/centralized_low_precision_synchronous.rs:22-73, SURVEY §3.4):
//   2P cub reductions + compress kernel + alltoall(NCCL send/recv) + decompress + chunk-reduce + 2 cub + compress +
//   allgather(NCCL) + decompress  ≈ 2P+7 launches, 2 collectives, 2 pool allocations.
// Here: ONE launch. Quantised payloads are stored straight into the destination rank's symmetric inbox (that IS the
// all-to-all), the P received copies of the owned chunk are dequantised + summed in fp32 on load, re-quantised, and
// stored into every rank's outbox (that IS the all-gather), then dequantised into the gradient bucket.
// Wire format, rounding and the reduce-in-T-then-requantise numerics are those of the reference so results are
// interchangeable with its python oracle (tests/internal/compressor.py).
#include <cstdlib>
#include <stdexcept>
#include <string>

#include "bulk_pipe.cuh"
#include "dispatch.h"
#include "kernels.h"
#include "peer.cuh"
#include "quant.cuh"

namespace bagua {
using namespace dev;

namespace {

__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// Device-wide barrier among the (co-resident) CTAs of this launch: a monotonically increasing arrival counter.
__device__ __forceinline__ void grid_barrier(unsigned long long* counter, unsigned long long target, const PeerCtx& ctx) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1ULL);
        unsigned long long t0 = 0;
        uint32_t spins = 0;
        while (ld_acquire_gpu_u64(counter) < target) {
            if ((++spins & 0x3ff) == 0) {
                unsigned long long now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                if (now - t0 > ctx.timeout_ns) {
                    atomicExch(ctx.error, 3);
                    break;
                }
            }
        }
        __threadfence();
    }
    __syncthreads();
}

// 16 consecutive elements of T starting at p (16-element aligned) → fp32
template <typename T>
__device__ __forceinline__ void load16(const T* p, float* f) {
    constexpr int PER = 16 / sizeof(T);  // elements per 16-byte vector
#pragma unroll
    for (int v = 0; v < 16 / PER; ++v) {
        uint4 raw = *reinterpret_cast<const uint4*>(p + v * PER);
        Vec16<T>::unpack(raw, f + v * PER);
    }
}
template <typename T>
__device__ __forceinline__ void store16(T* p, const float* f) {
    constexpr int PER = 16 / sizeof(T);
#pragma unroll
    for (int v = 0; v < 16 / PER; ++v) *reinterpret_cast<uint4*>(p + v * PER) = Vec16<T>::pack(f + v * PER);
}
template <typename T>
__device__ __forceinline__ float round_through(float v) {
    return to_f32<T>(from_f32<T>(v));
}
__device__ __forceinline__ uint4 quantize16(const float* f, const QuantParams& q) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
        w[i] = static_cast<uint32_t>(quantize(f[4 * i], q)) | (static_cast<uint32_t>(quantize(f[4 * i + 1], q)) << 8) |
               (static_cast<uint32_t>(quantize(f[4 * i + 2], q)) << 16) | (static_cast<uint32_t>(quantize(f[4 * i + 3], q)) << 24);
    return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void dequantize16(const uint4& raw, const QuantParams& q, float* f) {
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int b = 0; b < 4; ++b) f[4 * i + b] = dequantize(static_cast<uint8_t>((w[i] >> (8 * b)) & 0xffu), q);
}
template <typename T>
__device__ __forceinline__ QuantParams header_params(const char* chunk_base) {
    // header was written by another GPU during this kernel: read it with system-scope loads
    const uint32_t h0 = ld_relaxed_sys(reinterpret_cast<const uint32_t*>(chunk_base));
    float mn, mx;
    if (sizeof(T) == 4) {
        const uint32_t h1 = ld_relaxed_sys(reinterpret_cast<const uint32_t*>(chunk_base) + 1);
        mn = __uint_as_float(h0);
        mx = __uint_as_float(h1);
    } else {
        uint16_t lo = static_cast<uint16_t>(h0 & 0xffffu), hi = static_cast<uint16_t>(h0 >> 16);
        mn = to_f32<T>(*reinterpret_cast<T*>(&lo));
        mx = to_f32<T>(*reinterpret_cast<T*>(&hi));
    }
    return make_quant(mn, mx);
}
template <typename T>
__device__ __forceinline__ void write_header(char* chunk_base, float mn, float mx) {
    if (sizeof(T) == 4) {
        uint2 h = make_uint2(__float_as_uint(mn), __float_as_uint(mx));
        asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1,%2};" ::"l"(chunk_base), "r"(h.x), "r"(h.y) : "memory");
    } else {
        T a = from_f32<T>(mn), b = from_f32<T>(mx);
        uint32_t h = static_cast<uint32_t>(*reinterpret_cast<uint16_t*>(&a)) | (static_cast<uint32_t>(*reinterpret_cast<uint16_t*>(&b)) << 16);
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(chunk_base), "r"(h) : "memory");
    }
}

}  // namespace

// minmax scratch layout: uint32 [2 parities][kMaxPeers + 1][2]
__device__ __forceinline__ uint32_t* mm_slot(const ByteGradScratch& s, int parity, int idx) {
    return reinterpret_cast<uint32_t*>(s.minmax) + (static_cast<size_t>(parity) * (kMaxPeers + 1) + idx) * 2;
}

constexpr int kBgStages = 4;
constexpr int kBgTile = 16384;

template <typename T, int P>
__global__ void __launch_bounds__(512) bytegrad_kernel(PeerCtx ctx, T* data, size_t chunk, PeerBuf inbox, size_t inbox_off,
                                                       PeerBuf outbox, size_t outbox_off, ByteGradScratch scratch,
                                                       unsigned long long seq, unsigned long long gb_base, int average,
                                                       const T* grad, float beta1) {
    // The two passes over the locally produced bucket (A: min/max, B: quantise + send) stream their input through the TMA bulk-copy
    // engine into shared memory (bulk_pipe.cuh): 48 KB in flight per CTA without spending registers on it.
    extern __shared__ __align__(128) unsigned char bg_smem[];
    using Reader = BulkReader<kBgStages, kBgTile>;
    Reader rd;
    rd.init(bg_smem, ctx);
    const int parity = static_cast<int>(seq & 1ULL);
    const int nb = gridDim.x;
    const int bpc = nb / P;  // blocks per chunk in the scatter phases (host guarantees nb % P == 0)
    const size_t chunk_bytes = chunk + 32;  // chunk % 32 == 0 guaranteed by the host
    auto* gcount = reinterpret_cast<unsigned long long*>(scratch.grid_sync);
    const uint32_t e0 = load_epoch(ctx);
    const size_t groups = chunk / 16;  // 16-element groups per chunk

    // reset the other parity's min/max slots for the next launch (nobody touches them in this one)
    if (blockIdx.x == 0 && threadIdx.x <= P) {
        uint32_t* s = mm_slot(scratch, parity ^ 1, threadIdx.x);
        s[0] = kOrderedMinInit;
        s[1] = kOrderedMaxInit;
    }

    // ---- A: per-chunk min/max of my data ------------------------------------------------------------------
    // QAdam's compressed stage communicates the first moment: with `grad` given, the bucket IS the moment and the local update
    // m = β1·m + (1−β1)·g (reference bagua/torch_api/algorithms/q_adam.py:193-221, a python op on the comm thread there) is
    // applied in this same pass, rounded through T after each torch-level step (mul_, then add_ with alpha).
    const int cj = blockIdx.x / bpc, sb = blockIdx.x % bpc;
    {
        T* src = data + static_cast<size_t>(cj) * chunk;
        const T* gsrc = grad ? grad + static_cast<size_t>(cj) * chunk : nullptr;
        const float omb = 1.0f - beta1;
        float mn = INFINITY, mx = -INFINITY;
        const size_t step = static_cast<size_t>(bpc) * blockDim.x;
        size_t g = static_cast<size_t>(sb) * blockDim.x + threadIdx.x;
        if (!gsrc) {
            // read-only pass over my share of chunk cj (tiles sb, sb + bpc, ...), fed by the bulk-copy pipeline
            rd.start(src, chunk * sizeof(T), static_cast<size_t>(sb), static_cast<size_t>(bpc));
            const unsigned char* tile;
            uint32_t n;
            size_t off;
            while (rd.next(tile, n, off)) {
                for (uint32_t v = threadIdx.x * 16u; v < n; v += blockDim.x * 16u) {
                    float f[Vec16<T>::N];
                    Vec16<T>::unpack(lds16(tile + v), f);
#pragma unroll
                    for (int k = 0; k < Vec16<T>::N; ++k) mn = fminf(mn, f[k]), mx = fmaxf(mx, f[k]);
                }
                rd.release();
            }
            g = groups;   // nothing left for the per-thread loop below
        }
        for (; g < groups; g += step) {
            float f[16];
            load16<T>(src + g * 16, f);
            if (gsrc) {
                float gg[16];
                load16<T>(gsrc + g * 16, gg);
#pragma unroll
                for (int k = 0; k < 16; ++k) f[k] = round_through<T>(__fmaf_rn(omb, gg[k], round_through<T>(__fmul_rn(beta1, f[k]))));
                store16<T>(src + g * 16, f);
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) mn = fminf(mn, f[k]), mx = fmaxf(mx, f[k]);
        }
        // phase B reads what was just stored through the bulk-copy engine (async proxy): writer-side cross-proxy fence, the reader
        // issues its own before the first bulk copy (bulk_pipe.cuh) — the grid barrier in between carries the ordering across CTAs
        if (gsrc) asm volatile("fence.proxy.async;" ::: "memory");
        block_minmax(mn, mx);
        if (threadIdx.x == 0) {
            uint32_t* s = mm_slot(scratch, parity, cj);
            atomicMin(&s[0], f32_to_ordered(mn));
            atomicMax(&s[1], f32_to_ordered(mx));
        }
    }
    grid_barrier(gcount, gb_base + 1ULL * nb, ctx);

    // ---- B: quantise chunk cj and store it into rank cj's inbox slot [my rank]  (the all-to-all) ---------------
    {
        const uint32_t* s = mm_slot(scratch, parity, cj);
        const float mn = ordered_to_f32(__ldcg(&s[0])), mx = ordered_to_f32(__ldcg(&s[1]));
        const QuantParams q = make_quant(mn, mx);
        const T* src = data + static_cast<size_t>(cj) * chunk;
        char* dst = inbox.ptr[cj] + inbox_off + static_cast<size_t>(ctx.rank) * chunk_bytes;
        constexpr uint32_t GB = 16 * sizeof(T);   // bytes of one 16-element group in the tile
        // (with a momentum source phase A rewrote the bucket with generic stores from other CTAs: cross-proxy fence before the bulk reads)
        rd.start(src, chunk * sizeof(T), static_cast<size_t>(sb), static_cast<size_t>(bpc), grad != nullptr);
        const unsigned char* tile;
        uint32_t n;
        size_t off;
        while (rd.next(tile, n, off)) {
            const size_t e0 = off / sizeof(T);   // first element of this tile within the chunk
            for (uint32_t gi = threadIdx.x; gi * GB < n; gi += blockDim.x) {
                float f[16];
#pragma unroll
                for (uint32_t w = 0; w < GB / 16; ++w) Vec16<T>::unpack(lds16(tile + gi * GB + w * 16), f + w * Vec16<T>::N);
                st_peer16(dst + 32 + e0 + static_cast<size_t>(gi) * 16, quantize16(f, q));
            }
            rd.release();
        }
        if (sb == 0 && threadIdx.x == 0) write_header<T>(dst, mn, mx);
    }
    peer_barrier(ctx, e0 + 1);
    grid_barrier(gcount, gb_base + 2ULL * nb, ctx);

    // ---- C: dequantise + sum the P received copies of my chunk (fp32), keep the result, find its min/max ------------
    {
        const char* mybox = inbox.ptr[ctx.rank] + inbox_off;
        QuantParams qs[P];
#pragma unroll
        for (int s = 0; s < P; ++s) qs[s] = header_params<T>(mybox + static_cast<size_t>(s) * chunk_bytes);
        const float inv = average ? 1.0f / P : 1.0f;
        float mn = INFINITY, mx = -INFINITY;
        for (size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; g < groups; g += static_cast<size_t>(nb) * blockDim.x) {
            float acc[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) acc[k] = 0.f;
#pragma unroll
            for (int s = 0; s < P; ++s) {
                float f[16];
                dequantize16(ld_peer16(mybox + static_cast<size_t>(s) * chunk_bytes + 32 + g * 16), qs[s], f);
#pragma unroll
                for (int k = 0; k < 16; ++k) acc[k] += round_through<T>(f[k]);
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                acc[k] = round_through<T>(acc[k] * inv);
                mn = fminf(mn, acc[k]);
                mx = fmaxf(mx, acc[k]);
            }
            float4* r = reinterpret_cast<float4*>(scratch.reduced + g * 16);
#pragma unroll
            for (int v = 0; v < 4; ++v) r[v] = make_float4(acc[4 * v], acc[4 * v + 1], acc[4 * v + 2], acc[4 * v + 3]);
        }
        block_minmax(mn, mx);
        if (threadIdx.x == 0) {
            uint32_t* s = mm_slot(scratch, parity, P);
            atomicMin(&s[0], f32_to_ordered(mn));
            atomicMax(&s[1], f32_to_ordered(mx));
        }
    }
    grid_barrier(gcount, gb_base + 3ULL * nb, ctx);

    // ---- D: re-quantise the reduced chunk and store it into every rank's outbox slot [my rank] (the all-gather) -----
    {
        const uint32_t* s = mm_slot(scratch, parity, P);
        const float mn = ordered_to_f32(__ldcg(&s[0])), mx = ordered_to_f32(__ldcg(&s[1]));
        const QuantParams q = make_quant(mn, mx);
        for (size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; g < groups; g += static_cast<size_t>(nb) * blockDim.x) {
            float f[16];
            const float4* r = reinterpret_cast<const float4*>(scratch.reduced + g * 16);
#pragma unroll
            for (int v = 0; v < 4; ++v) {
                float4 x = __ldcg(&r[v]);
                f[4 * v] = x.x, f[4 * v + 1] = x.y, f[4 * v + 2] = x.z, f[4 * v + 3] = x.w;
            }
            const uint4 packed = quantize16(f, q);
#pragma unroll
            for (int i = 0; i < P; ++i) {
                const int p = (ctx.rank + i) % P;
                st_peer16(outbox.ptr[p] + outbox_off + static_cast<size_t>(ctx.rank) * chunk_bytes + 32 + g * 16, packed);
            }
        }
        if (blockIdx.x == 0 && threadIdx.x < P)
            write_header<T>(outbox.ptr[threadIdx.x] + outbox_off + static_cast<size_t>(ctx.rank) * chunk_bytes, mn, mx);
    }
    peer_barrier(ctx, e0 + 2);
    // every local CTA must know that every peer CTA has delivered: one more device-wide rendezvous
    grid_barrier(gcount, gb_base + 4ULL * nb, ctx);

    // ---- E: dequantise all P chunks from my outbox into the bucket ----------------------------------------------
    {
        const char* mybox = outbox.ptr[ctx.rank] + outbox_off;
        for (int s = 0; s < P; ++s) {
            const QuantParams q = header_params<T>(mybox + static_cast<size_t>(s) * chunk_bytes);
            T* dst = data + static_cast<size_t>(s) * chunk;
            // The payload was written by peer GPUs during this kernel: it is read with system-scope loads (the path validated on
            // 2/4/8 GPUs), four independent 16-byte loads in flight per thread — not through the bulk-copy engine, whose
            // async-proxy reads of bytes that arrived over NVLink moments ago have not been validated on a multi-GPU box.
            const size_t step = static_cast<size_t>(nb) * blockDim.x;
            const char* payload = mybox + static_cast<size_t>(s) * chunk_bytes + 32;
            size_t g = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
            for (; g + 3 * step < groups; g += 4 * step) {
                uint4 r0 = ld_peer16(payload + g * 16), r1 = ld_peer16(payload + (g + step) * 16), r2 = ld_peer16(payload + (g + 2 * step) * 16),
                      r3 = ld_peer16(payload + (g + 3 * step) * 16);
                float f[16];
                dequantize16(r0, q, f);
                store16<T>(dst + g * 16, f);
                dequantize16(r1, q, f);
                store16<T>(dst + (g + step) * 16, f);
                dequantize16(r2, q, f);
                store16<T>(dst + (g + 2 * step) * 16, f);
                dequantize16(r3, q, f);
                store16<T>(dst + (g + 3 * step) * 16, f);
            }
            for (; g < groups; g += step) {
                float f[16];
                dequantize16(ld_peer16(payload + g * 16), q, f);
                store16<T>(dst + g * 16, f);
            }
        }
    }
    store_epoch(ctx, e0 + 2);
}

// ---------------------------------------------------------------------------------------------------------
// Low-precision decentralized ring step in one kernel.
// box layout (per rank, symmetric): [2 parities][3 slots: from-left, from-right, own] x chunk_bytes
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(512) lpdec_ring_kernel(PeerCtx ctx, T* x, T* w, T* l, T* r, size_t numel, PeerBuf box, size_t box_off,
                                                         ByteGradScratch scratch, unsigned long long seq,
                                                         unsigned long long gb_base, int left, int right) {
    const int parity = static_cast<int>(seq & 1ULL);
    const int nb = gridDim.x;
    const size_t chunk_bytes = numel + 32;
    auto* gcount = reinterpret_cast<unsigned long long*>(scratch.grid_sync);
    const uint32_t e0 = load_epoch(ctx);
    const size_t groups = numel / 16;
    const size_t stride = static_cast<size_t>(nb) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const float f13 = static_cast<float>(1.0 / 3.0), f53 = static_cast<float>(5.0 / 3.0);

    if (blockIdx.x == 0 && threadIdx.x == 0) {
        uint32_t* s = mm_slot(scratch, parity ^ 1, 0);
        s[0] = kOrderedMinInit;
        s[1] = kOrderedMaxInit;
    }
    // 1: diff = x + L/3 + R/3 - 5W/3 (each step rounded to T like the reference's in-place kernels), min/max
    {
        float mn = INFINITY, mx = -INFINITY;
        for (size_t g = tid; g < groups; g += stride) {
            float fx[16], fl[16], fr[16], fw[16];
            load16<T>(x + g * 16, fx);
            load16<T>(l + g * 16, fl);
            load16<T>(r + g * 16, fr);
            load16<T>(w + g * 16, fw);
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                float d = round_through<T>(__fadd_rn(fx[k], round_through<T>(__fmul_rn(f13, fl[k]))));
                d = round_through<T>(__fadd_rn(d, round_through<T>(__fmul_rn(f13, fr[k]))));
                d = round_through<T>(__fsub_rn(d, round_through<T>(__fmul_rn(f53, fw[k]))));
                fx[k] = d;
                mn = fminf(mn, d);
                mx = fmaxf(mx, d);
            }
            store16<T>(x + g * 16, fx);
        }
        block_minmax(mn, mx);
        if (threadIdx.x == 0) {
            uint32_t* s = mm_slot(scratch, parity, 0);
            atomicMin(&s[0], f32_to_ordered(mn));
            atomicMax(&s[1], f32_to_ordered(mx));
        }
    }
    grid_barrier(gcount, gb_base + 1ULL * nb, ctx);
    // 2: quantise the diff; deposit at the left neighbour (its "from-right" slot), the right neighbour (its
    //    "from-left" slot) and locally ("own")
    {
        const uint32_t* s = mm_slot(scratch, parity, 0);
        const float mn = ordered_to_f32(__ldcg(&s[0])), mx = ordered_to_f32(__ldcg(&s[1]));
        const QuantParams q = make_quant(mn, mx);
        char* to_left = box.ptr[left] + box_off + (static_cast<size_t>(parity) * 3 + 1) * chunk_bytes;
        char* to_right = box.ptr[right] + box_off + (static_cast<size_t>(parity) * 3 + 0) * chunk_bytes;
        char* own = box.ptr[ctx.rank] + box_off + (static_cast<size_t>(parity) * 3 + 2) * chunk_bytes;
        for (size_t g = tid; g < groups; g += stride) {
            float f[16];
            load16<T>(x + g * 16, f);
            const uint4 packed = quantize16(f, q);
            st_peer16(to_left + 32 + g * 16, packed);
            st_peer16(to_right + 32 + g * 16, packed);
            st_peer16(own + 32 + g * 16, packed);
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            write_header<T>(to_left, mn, mx);
            write_header<T>(to_right, mn, mx);
            write_header<T>(own, mn, mx);
        }
    }
    peer_barrier(ctx, e0 + 1);
    grid_barrier(gcount, gb_base + 2ULL * nb, ctx);
    // 3: L += deq(from-left); R += deq(from-right); x = deq(own) + W; W = x
    {
        const char* base = box.ptr[ctx.rank] + box_off + static_cast<size_t>(parity) * 3 * chunk_bytes;
        const QuantParams ql = header_params<T>(base), qr = header_params<T>(base + chunk_bytes), qo = header_params<T>(base + 2 * chunk_bytes);
        for (size_t g = tid; g < groups; g += stride) {
            float a[16], d[16];
            load16<T>(l + g * 16, a);
            dequantize16(ld_peer16(base + 32 + g * 16), ql, d);
#pragma unroll
            for (int k = 0; k < 16; ++k) a[k] = __fadd_rn(a[k], round_through<T>(d[k]));
            store16<T>(l + g * 16, a);
            load16<T>(r + g * 16, a);
            dequantize16(ld_peer16(base + chunk_bytes + 32 + g * 16), qr, d);
#pragma unroll
            for (int k = 0; k < 16; ++k) a[k] = __fadd_rn(a[k], round_through<T>(d[k]));
            store16<T>(r + g * 16, a);
            load16<T>(w + g * 16, a);
            dequantize16(ld_peer16(base + 2 * chunk_bytes + 32 + g * 16), qo, d);
#pragma unroll
            for (int k = 0; k < 16; ++k) a[k] = __fadd_rn(round_through<T>(d[k]), a[k]);
            store16<T>(x + g * 16, a);
            store16<T>(w + g * 16, a);
        }
    }
    store_epoch(ctx, e0 + 1);
}

// ---------------------------------------------------------------------------------------------------------

// Host-side bookkeeping of a scratch instance: returns {sequence number, arrival base} for this launch and
// advances both (n_barriers grid barriers of nblocks arrivals each).
static void next_launch(const ByteGradScratch& s, int n_barriers, int nblocks, unsigned long long& seq, unsigned long long& base) {
    seq = s.host_state[0]++;
    base = s.host_state[1];
    s.host_state[1] += static_cast<unsigned long long>(n_barriers) * nblocks;
}

// Both kernels below synchronise their own CTAs with a counter barrier, i.e. every CTA of the grid must be resident at the same
// time. A cooperative launch makes the driver guarantee exactly that (the launch waits until the whole grid fits, or fails if
// it never can), instead of relying on the SMs happening to be free while cuDNN owns the GPU. BAGUA_COOPERATIVE_LAUNCH=0 → plain.
static bool use_cooperative() {
    static const bool on = [] {
        const char* e = std::getenv("BAGUA_COOPERATIVE_LAUNCH");
        return !(e && e[0] == '0');
    }();
    return on;
}
template <typename K>
static int clamp_grid_to_residency(K kernel, int nblocks, int nthreads, int multiple_of, size_t smem = 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, nthreads, smem) != cudaSuccess || per_sm < 1 || sms < 1) return nblocks;
    int cap = per_sm * sms;
    if (nblocks > cap) nblocks = cap / multiple_of * multiple_of;
    return nblocks < multiple_of ? multiple_of : nblocks;
}
template <typename K>
static void launch_grid_synced(K kernel, int nblocks, int nthreads, cudaStream_t stream, void** args, size_t smem = 0) {
    if (use_cooperative()) {
        cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kernel), dim3(nblocks), dim3(nthreads), args, smem, stream);
        if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: cooperative launch failed: ") + cudaGetErrorString(e));
    } else {
        cudaError_t e = cudaLaunchKernel(reinterpret_cast<const void*>(kernel), dim3(nblocks), dim3(nthreads), args, smem, stream);
        if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch failed: ") + cudaGetErrorString(e));
    }
}

void launch_bytegrad(const PeerCtx& ctx, void* data, size_t numel, int dtype, const PeerBuf& inbox, size_t inbox_off,
                     const PeerBuf& outbox, size_t outbox_off, const ByteGradScratch& scratch, bool average, int nblocks,
                     int nthreads, cudaStream_t stream, const void* grad, float beta1) {
    const int P = ctx.world;
    if (numel % (static_cast<size_t>(P) * 32)) throw std::runtime_error("bagua: bytegrad bucket must be a multiple of 32*nranks elements");
    if (nblocks % P || nblocks < P || nblocks > kMaxCommBlocks) throw std::runtime_error("bagua: bytegrad grid must be a multiple of nranks (≤ 256)");
    size_t chunk = numel / P;
    dispatch_float(dtype, "quantised collectives", [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(P, [&](auto pw) {
            constexpr int PP = decltype(pw)::value;
            auto kernel = bytegrad_kernel<T, PP>;
            constexpr size_t smem = BulkReader<kBgStages, kBgTile>::smem_bytes();
            static bool attr_set = false;   // per instantiation (this lambda body is instantiated per <T, PP>)
            if (!attr_set) {
                cudaError_t ae = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
                if (ae != cudaSuccess) throw std::runtime_error(std::string("bagua: bytegrad shared-memory opt-in failed: ") + cudaGetErrorString(ae));
                attr_set = true;
            }
            const int nb = clamp_grid_to_residency(kernel, nblocks, nthreads, P, smem);
            unsigned long long seq, base;
            next_launch(scratch, 4, nb, seq, base);
            PeerCtx c = ctx;
            T* d = static_cast<T*>(data);
            PeerBuf in = inbox, out = outbox;
            ByteGradScratch sc = scratch;
            int avg = average ? 1 : 0;
            const T* g = static_cast<const T*>(grad);
            void* args[] = {&c, &d, &chunk, &in, &inbox_off, &out, &outbox_off, &sc, &seq, &base, &avg, &g, &beta1};
            launch_grid_synced(kernel, nb, nthreads, stream, args, smem);
        });
    });
    check_launch("bytegrad");
}

void launch_lpdec_ring(const PeerCtx& ctx, void* x, void* w, void* l, void* r, size_t numel, int dtype, const PeerBuf& box,
                       size_t box_off, const ByteGradScratch& scratch, int left, int right, int nblocks, int nthreads,
                       cudaStream_t stream) {
    if (numel % 32) throw std::runtime_error("bagua: low-precision ring bucket must be a multiple of 32 elements");
    if (nblocks < 1 || nblocks > kMaxCommBlocks) throw std::runtime_error("bagua: bad grid for lpdec ring");
    dispatch_float(dtype, "quantised collectives", [&](auto tag) {
        using T = decltype(tag);
        auto kernel = lpdec_ring_kernel<T>;
        const int nb = clamp_grid_to_residency(kernel, nblocks, nthreads, 1);
        unsigned long long seq, base;
        next_launch(scratch, 2, nb, seq, base);
        PeerCtx c = ctx;
        T *xx = static_cast<T*>(x), *ww = static_cast<T*>(w), *ll = static_cast<T*>(l), *rr = static_cast<T*>(r);
        PeerBuf bx = box;
        ByteGradScratch sc = scratch;
        void* args[] = {&c, &xx, &ww, &ll, &rr, &numel, &bx, &box_off, &sc, &seq, &base, &left, &right};
        launch_grid_synced(kernel, nb, nthreads, stream, args);
    });
    check_launch("lpdec_ring");
}

}  // namespace bagua
