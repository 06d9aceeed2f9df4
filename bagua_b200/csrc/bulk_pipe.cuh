// CTA-wide streaming reader on the TMA bulk-copy engine (sm_90a): global memory → ring of shared-memory stages via
// `cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes`, completion tracked by one mbarrier per stage.
//
// Why: the bandwidth a CTA can pull is (bytes in flight) / latency. A per-thread `ld.global` loop keeps at most a few 16-byte
// loads per thread in flight (registers), ~32 KB per 512-thread CTA — measured 18 GB/s per CTA in the quantised bucket kernels, a
// third of what an SM can stream. One elected thread issuing 16 KB bulk copies keeps STAGES-1 tiles (48 KB) in flight per CTA with
// no registers spent, and the consumers read their data from shared memory at full speed. The communication kernels of this
// library deliberately run on FEW CTAs (they share the GPU with the backward pass), so per-CTA throughput is what counts.
//
// Usage (all threads of the CTA call every method, in the same order):
//     extern __shared__ __align__(128) unsigned char smem[];
//     BulkReader<4, 16384> rd;  rd.init(smem, ctx);
//     rd.start(src, bytes, first_tile, tile_stride);          // this CTA reads tiles first, first+stride, ...
//     const unsigned char* tile; uint32_t n; size_t off;
//     while (rd.next(tile, n, off)) { ... consume tile[0..n) (off = byte offset in src) ...; rd.release(); }
// Waits are bounded by the communicator's time-out and raise the fatal error word instead of hanging the GPU.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "peer.cuh"

namespace bagua {
namespace dev {

__device__ __forceinline__ uint32_t smem_addr_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

template <int STAGES, int TILE>
struct BulkReader {
    static_assert(TILE % 128 == 0, "tile must keep shared-memory stages 128-byte aligned");
    unsigned char* stages;     // STAGES * TILE bytes
    uint64_t* full;            // STAGES mbarriers
    const PeerCtx* ctx;
    // stream state (identical in every thread)
    const unsigned char* src;
    size_t bytes, tiles, next_issue, next_consume, stride;
    uint32_t it;               // tiles consumed so far in this kernel: stage = it % STAGES, parity = (it / STAGES) & 1
    uint32_t issued;           // tiles issued so far in this kernel
    bool dead;

    static constexpr size_t smem_bytes() { return static_cast<size_t>(STAGES) * TILE + STAGES * sizeof(uint64_t) + 128; }

    __device__ __forceinline__ void init(unsigned char* smem, const PeerCtx& c) {
        stages = smem;
        full = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(STAGES) * TILE);
        ctx = &c;
        it = issued = 0;
        dead = false;
        tiles = next_issue = next_consume = 0;
        if (threadIdx.x == 0) {
#pragma unroll
            for (int s = 0; s < STAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr_u32(&full[s])), "r"(1));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
    }

    __device__ __forceinline__ void issue_one() {   // thread 0 only
        const size_t t = next_issue;
        const size_t off = t * TILE;
        const uint32_t n = static_cast<uint32_t>(bytes - off < TILE ? bytes - off : TILE);
        const uint32_t s = issued % STAGES;
        const uint32_t bar = smem_addr_u32(&full[s]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(n) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr_u32(stages + static_cast<size_t>(s) * TILE)),
                     "l"(src + off), "r"(n), "r"(bar)
                     : "memory");
    }

    // Begin streaming `nbytes` (multiple of 16, 16-byte aligned) from `p`; this CTA takes tiles first, first + tile_stride, ...
    // `after_peer_writes`: the bytes were written by other SMs / GPUs during this kernel (ordered by a barrier the caller has
    // passed): the issuing thread then needs a cross-proxy fence before the async-proxy reads.
    __device__ __forceinline__ void start(const void* p, size_t nbytes, size_t first_tile, size_t tile_stride, bool after_peer_writes = false) {
        src = static_cast<const unsigned char*>(p);
        bytes = nbytes;
        tiles = (nbytes + TILE - 1) / TILE;
        stride = tile_stride;
        next_issue = next_consume = first_tile;
        if (threadIdx.x == 0) {
            if (after_peer_writes) asm volatile("fence.proxy.async;" ::: "memory");
            for (int k = 0; k < STAGES - 1 && next_issue < tiles; ++k) {
                issue_one();
                next_issue += stride;
                ++issued;
            }
        } else {
            for (int k = 0; k < STAGES - 1 && next_issue < tiles; ++k) {
                next_issue += stride;
                ++issued;
            }
        }
    }

    // Next tile of this CTA's share, or false when the stream is exhausted.
    __device__ __forceinline__ bool next(const unsigned char*& tile, uint32_t& n, size_t& off) {
        if (next_consume >= tiles) return false;
        if (next_issue < tiles) {   // keep STAGES-1 tiles in flight: the stage being refilled was released by every thread (release())
            if (threadIdx.x == 0) issue_one();
            next_issue += stride;
            ++issued;
        }
        const uint32_t s = it % STAGES, parity = (it / STAGES) & 1u;
        const uint32_t bar = smem_addr_u32(&full[s]);
        if (!dead) {
            uint32_t done = 0, spins = 0;
            unsigned long long t0 = 0;
            while (!done) {
                asm volatile(
                    "{\n\t.reg .pred p;\n\t"
                    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                    "selp.u32 %0, 1, 0, p;\n\t}"
                    : "=r"(done)
                    : "r"(bar), "r"(parity)
                    : "memory");
                if (!done && (++spins & 0xfff) == 0) {
                    const unsigned long long now = globaltimer_ns();
                    if (t0 == 0) t0 = now;
                    if (now - t0 > ctx->timeout_ns) {
                        raise_error(*ctx, 5);   // a bulk copy never landed: fatal, but the GPU is not left hanging
                        dead = true;
                        break;
                    }
                }
            }
        }
        off = next_consume * TILE;
        n = static_cast<uint32_t>(bytes - off < TILE ? bytes - off : TILE);
        tile = stages + static_cast<size_t>(s) * TILE;
        return true;
    }

    // Every thread is done reading the current tile: its stage may be refilled.
    __device__ __forceinline__ void release() {
        __syncthreads();
        ++it;
        next_consume += stride;
    }
};

__device__ __forceinline__ uint4 lds16(const void* p) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_addr_u32(p)));
    return v;
}

}  // namespace dev
}  // namespace bagua
