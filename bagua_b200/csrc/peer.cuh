// Device-side building blocks for kernels that talk to other GPUs over NVLink 4 / NVSwitch:
// system-scope flags, an epoch barrier over symmetric signal pads, 16-byte peer loads/stores and the
// NVLS multimem instructions. sm_90a only.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "common.h"

namespace bagua {
namespace dev {

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// 16-byte system-coherent load (peer memory is written by other GPUs during this kernel's lifetime, so
// it must not be served from a stale L1 line) and a plain 16-byte store.
__device__ __forceinline__ uint4 ld_peer16(const void* p) {
    uint4 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void st_peer16(void* p, const uint4& v) {
    asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}
// Streaming local accesses (read once / written once: keep them out of L1).
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
    uint4 v;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream16(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}

// ---- NVLS (in-switch) reduce-load and broadcast-store on a multicast address -------------------------
template <typename T>
__device__ __forceinline__ uint4 multimem_ld_reduce_add(const void* mc);
template <>
__device__ __forceinline__ uint4 multimem_ld_reduce_add<float>(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
template <>
__device__ __forceinline__ uint4 multimem_ld_reduce_add<__nv_bfloat16>(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
template <>
__device__ __forceinline__ uint4 multimem_ld_reduce_add<__half>(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st16(void* mc, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}

// ---- 16-byte vectors of T <-> fp32 lanes ---------------------------------------------------------------
template <typename T>
struct Vec16;
template <>
struct Vec16<float> {
    static constexpr int N = 4;
    __device__ static void unpack(const uint4& v, float* f) {
        f[0] = __uint_as_float(v.x);
        f[1] = __uint_as_float(v.y);
        f[2] = __uint_as_float(v.z);
        f[3] = __uint_as_float(v.w);
    }
    __device__ static uint4 pack(const float* f) {
        return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
    }
};
template <>
struct Vec16<__nv_bfloat16> {
    static constexpr int N = 8;
    __device__ static void unpack(const uint4& v, float* f) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            f[2 * i] = __uint_as_float(w[i] << 16);
            f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
    __device__ static uint4 pack(const float* f) {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
            w[i] = *reinterpret_cast<uint32_t*>(&h);
        }
        return make_uint4(w[0], w[1], w[2], w[3]);
    }
};
template <>
struct Vec16<__half> {
    static constexpr int N = 8;
    __device__ static void unpack(const uint4& v, float* f) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
            float2 x = __half22float2(h);
            f[2 * i] = x.x;
            f[2 * i + 1] = x.y;
        }
    }
    __device__ static uint4 pack(const float* f) {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
            w[i] = *reinterpret_cast<uint32_t*>(&h);
        }
        return make_uint4(w[0], w[1], w[2], w[3]);
    }
};

// A kernel that gives up (barrier time-out, abort, grid-barrier time-out, protocol violation) leaves a non-zero code in the
// device error word AND in its host-mapped mirror, which the host checks before every further peer op and in
// wait_pending_comm_ops: a failed collective is fatal for the job (replicas would silently diverge otherwise).
__device__ __forceinline__ void raise_error(const PeerCtx& ctx, int code) {
    atomicExch(ctx.error, code);
    *ctx.host_error = code;
    __threadfence_system();
}

// ---- cross-GPU barrier ----------------------------------------------------------------------------------
// Every CTA b of every rank owns flag row b. Thread p (< world) publishes `epoch` into rank p's slot
// [b][my_rank] with a system-scope release and spins with acquire loads on its own slot [b][p].
// Epochs only grow, so no reset pass and no ABA. The spin is bounded: a host-mapped abort flag
// (PeerComm.abort()) or a timeout makes the kernel give up, raise ctx.error and return false.
__device__ __forceinline__ bool peer_barrier(const PeerCtx& ctx, uint32_t epoch) {
    __shared__ int s_ok;
    if (threadIdx.x == 0) s_ok = 1;
    __syncthreads();  // also orders every thread's earlier global/peer writes before the release below
    if (threadIdx.x < ctx.world) {
        const int p = threadIdx.x;
        uint32_t* remote = ctx.flags[p] + blockIdx.x * kFlagStride + ctx.rank;
        st_release_sys(remote, epoch);
        const uint32_t* mine = ctx.flags[ctx.rank] + blockIdx.x * kFlagStride + p;
        unsigned long long t0 = 0;
        uint32_t spins = 0;
        while (static_cast<int32_t>(ld_acquire_sys(mine) - epoch) < 0) {
            if ((++spins & 0x3ff) == 0) {
                unsigned long long now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                if (*ctx.abort != 0 || now - t0 > ctx.timeout_ns) {
                    raise_error(ctx, *ctx.abort != 0 ? 2 : 1);
                    s_ok = 0;
                    break;
                }
            }
        }
    }
    __syncthreads();
    return s_ok != 0;
}

// The same barrier carrying one word per rank (an all-to-all of a uint32 riding on the flags): every CTA of rank r deposits
// `my_word` in slot [r] of every peer's vote area right before the releasing flag store, and after the acquire reads the P
// words deposited in its own pad into s_votes[0..world). All CTAs of a rank must pass the same word. A rank can only be one
// launch ahead of a peer's slowest CTA after that CTA has read its votes (stream order + the kernel's closing barrier), so
// the single vote area needs no double-buffering.
__device__ __forceinline__ bool peer_barrier_vote(const PeerCtx& ctx, uint32_t epoch, uint32_t my_word, uint32_t* s_votes) {
    __shared__ int s_ok_v;
    if (threadIdx.x == 0) s_ok_v = 1;
    __syncthreads();
    if (threadIdx.x < ctx.world) {
        const int p = threadIdx.x;
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(ctx.flags[p] + kVoteWordOffset + ctx.rank), "r"(my_word) : "memory");
        st_release_sys(ctx.flags[p] + blockIdx.x * kFlagStride + ctx.rank, epoch);
        const uint32_t* mine = ctx.flags[ctx.rank] + blockIdx.x * kFlagStride + p;
        unsigned long long t0 = 0;
        uint32_t spins = 0;
        bool ok = true;
        while (static_cast<int32_t>(ld_acquire_sys(mine) - epoch) < 0) {
            if ((++spins & 0x3ff) == 0) {
                unsigned long long now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                if (*ctx.abort != 0 || now - t0 > ctx.timeout_ns) {
                    raise_error(ctx, *ctx.abort != 0 ? 2 : 1);
                    s_ok_v = 0;
                    ok = false;
                    break;
                }
            }
        }
        if (ok) s_votes[p] = ld_relaxed_sys(ctx.flags[ctx.rank] + kVoteWordOffset + p);
    }
    __syncthreads();
    return s_ok_v != 0;
}

// Epoch bookkeeping: each CTA keeps its own counter so launches with different grid sizes compose.
__device__ __forceinline__ uint32_t load_epoch(const PeerCtx& ctx) { return ctx.epochs[blockIdx.x]; }
__device__ __forceinline__ void store_epoch(const PeerCtx& ctx, uint32_t e) {
    if (threadIdx.x == 0) ctx.epochs[blockIdx.x] = e;
}

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace dev
}  // namespace bagua
