// MoE expert-parallel token exchange as peer-memory kernels (sm_90a, NVLink 4 / NVSwitch).
//
// The reference dispatches with a dense one-hot einsum (S*E*C*M MACs) followed by torch's NCCL all_to_all_single, and
// combines with another all-to-all + einsum (bagua/torch_api/model_parallel/moe/sharded_moe.py:352-374). Here the
// all-to-all *is* the row copy: a token row is stored straight into the capacity slot of its expert in the owning GPU's
// symmetric buffer (scatter), and combined rows are loaded straight from the owners' buffers, weighted and summed
// (gather). One warp moves one row with 16-byte accesses; two cross-GPU barriers bracket each kernel.
#include <stdexcept>
#include <string>

#include "kernels.h"
#include "peer.cuh"

namespace bagua {
using namespace dev;

namespace {
constexpr int kMoeThreads = 256;  // 8 warps, one row each per iteration
}

// Buffer layout on every rank: rows[(src_rank * E_local + e_local) * C + c][M]   (= [world, E_local, C, M])
// Global expert e lives on rank e / E_local as local expert e % E_local.
template <typename T>
__global__ void __launch_bounds__(kMoeThreads)
    moe_scatter_kernel(PeerCtx ctx, PeerBuf dst, size_t dst_off, const T* __restrict__ rows_in, const int64_t* __restrict__ expert_idx,
                       const int64_t* __restrict__ slot_idx, const float* __restrict__ scale, int S, int K, int M, int E_local, int C) {
    const uint32_t e0 = load_epoch(ctx);
    const int world = ctx.world;
    const size_t row_bytes = static_cast<size_t>(M) * sizeof(T);
    const size_t vec_per_row = row_bytes / 16;
    // (my receive buffer was cleared by the launcher on this stream: slots nobody fills must read as zeros — the experts
    //  run on them and their weight gradients would otherwise pick up garbage)
    bool ok = peer_barrier(ctx, e0 + 1);
    // 2. one warp per (token, choice): store the row into the owner's slot
    if (ok) {
        const int lane = threadIdx.x & 31;
        const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
        const int nwarps = (gridDim.x * blockDim.x) >> 5;
        for (int item = warp; item < S * K; item += nwarps) {
            const int64_t slot = slot_idx[item];
            if (slot < 0) continue;  // dropped token
            const int64_t e = expert_idx[item];
            const int owner = static_cast<int>(e / E_local);
            const int el = static_cast<int>(e % E_local);
            const int s = item / K;
            const size_t drow = (static_cast<size_t>(ctx.rank) * E_local + el) * C + static_cast<size_t>(slot);
            char* d = dst.ptr[owner] + dst_off + drow * row_bytes;
            const char* src = reinterpret_cast<const char*>(rows_in) + static_cast<size_t>(s) * row_bytes;
            const float sc = scale ? scale[item] : 1.0f;
            // 4 independent 16-byte loads per lane before the first (NVLink) store: a row moves as 2 KB bursts, not 512 B round trips
            for (size_t v0 = lane; v0 < vec_per_row; v0 += 32 * 4) {
                uint4 raw[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const size_t v = v0 + static_cast<size_t>(j) * 32;
                    if (v < vec_per_row) raw[j] = ld_stream16(src + v * 16);
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const size_t v = v0 + static_cast<size_t>(j) * 32;
                    if (v >= vec_per_row) continue;
                    if (scale) {
                        float f[Vec16<T>::N];
                        Vec16<T>::unpack(raw[j], f);
#pragma unroll
                        for (int k = 0; k < Vec16<T>::N; ++k) f[k] *= sc;
                        raw[j] = Vec16<T>::pack(f);
                    }
                    st_peer16(d + v * 16, raw[j]);
                }
            }
        }
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

// out[s] = sum_k w[s,k] * rows_on_owner[(my_rank * E_local + e_local) * C + slot]; optionally also
// picked[s,k,:] = that row (saved for backward) and dots[s,k] = <grad_like[s], row>.
template <typename T>
__global__ void __launch_bounds__(kMoeThreads)
    moe_gather_kernel(PeerCtx ctx, PeerBuf src, size_t src_off, T* __restrict__ out, const int64_t* __restrict__ expert_idx,
                      const int64_t* __restrict__ slot_idx, const float* __restrict__ weights, T* __restrict__ picked, int S, int K, int M,
                      int E_local, int C, int local_layout) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);  // every owner's rows are complete (stream order before its kernel) and visible
    const size_t row_bytes = static_cast<size_t>(M) * sizeof(T);
    const size_t vec_per_row = row_bytes / 16;
    if (ok) {
        const int lane = threadIdx.x & 31;
        const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
        const int nwarps = (gridDim.x * blockDim.x) >> 5;
        for (int s = warp; s < S; s += nwarps) {
            char* o = reinterpret_cast<char*>(out) + static_cast<size_t>(s) * row_bytes;
            for (size_t v0 = lane; v0 < vec_per_row; v0 += 32 * 4) {
                float acc[4][Vec16<T>::N];
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int q = 0; q < Vec16<T>::N; ++q) acc[j][q] = 0.f;
                for (int k = 0; k < K; ++k) {
                    const int item = s * K + k;
                    const int64_t slot = slot_idx[item];
                    uint4 raw[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) raw[j] = make_uint4(0, 0, 0, 0);
                    float w = 0.f;
                    if (slot >= 0) {
                        const int64_t e = expert_idx[item];
                        const int owner = static_cast<int>(e / E_local);
                        const int el = static_cast<int>(e % E_local);
                        // pull layout: the row sits on its owner at [my rank][expert][slot];
                        // local layout (the owner's GEMM epilogue pushed it here): my buffer at [owner][expert][slot]
                        const int from = local_layout ? ctx.rank : owner;
                        const int major = local_layout ? owner : ctx.rank;
                        const size_t srow = (static_cast<size_t>(major) * E_local + el) * C + static_cast<size_t>(slot);
                        const char* rp = src.ptr[from] + src_off + srow * row_bytes;
                        w = weights ? weights[item] : 1.0f;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {   // four NVLink loads in flight per lane
                            const size_t v = v0 + static_cast<size_t>(j) * 32;
                            if (v < vec_per_row) raw[j] = ld_peer16(rp + v * 16);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const size_t v = v0 + static_cast<size_t>(j) * 32;
                        if (v >= vec_per_row) continue;
                        if (slot >= 0) {
                            float f[Vec16<T>::N];
                            Vec16<T>::unpack(raw[j], f);
#pragma unroll
                            for (int q = 0; q < Vec16<T>::N; ++q) acc[j][q] += w * f[q];
                        }
                        if (picked) st_stream16(reinterpret_cast<char*>(picked) + static_cast<size_t>(item) * row_bytes + v * 16, raw[j]);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const size_t v = v0 + static_cast<size_t>(j) * 32;
                    if (v < vec_per_row) st_stream16(o + v * 16, Vec16<T>::pack(acc[j]));
                }
            }
        }
        peer_barrier(ctx, e0 + 2);  // owners may recycle their buffers only after every reader is done
    }
    store_epoch(ctx, e0 + 2);
}

namespace {
template <typename F>
void dispatch_float(int dtype, F&& f) {
    switch (dtype) {
        case F32: f(float{}); break;
        case F16: f(__half{}); break;
        case BF16: f(__nv_bfloat16{}); break;
        default: throw std::runtime_error("bagua: MoE kernels need f32/f16/bf16, got dtype code " + std::to_string(dtype));
    }
}
void check(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of ") + what + " failed: " + cudaGetErrorString(e));
    count_launch();
}
void check_shape(int M, int dtype, int nblocks) {
    if ((static_cast<size_t>(M) * dtype_size(dtype)) % 16) throw std::runtime_error("bagua: MoE rows must be a multiple of 16 bytes");
    if (nblocks < 1 || nblocks > kMaxCommBlocks) throw std::runtime_error("bagua: bad grid for MoE kernel");
}
}  // namespace

void launch_moe_scatter(const PeerCtx& ctx, const PeerBuf& dst, size_t dst_off, const void* rows_in, const int64_t* expert_idx,
                        const int64_t* slot_idx, const float* scale, int S, int K, int M, int E_local, int C, int dtype, int nblocks,
                        cudaStream_t stream) {
    check_shape(M, dtype, nblocks);
    const size_t bytes = static_cast<size_t>(ctx.world) * E_local * C * M * dtype_size(dtype);
    cudaError_t me = cudaMemsetAsync(dst.ptr[ctx.rank] + dst_off, 0, bytes, stream);
    if (me != cudaSuccess) throw std::runtime_error(std::string("bagua: moe_scatter memset failed: ") + cudaGetErrorString(me));
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        moe_scatter_kernel<T><<<nblocks, kMoeThreads, 0, stream>>>(ctx, dst, dst_off, static_cast<const T*>(rows_in), expert_idx, slot_idx, scale, S, K,
                                                                  M, E_local, C);
    });
    check("moe_scatter");
}

void launch_moe_gather(const PeerCtx& ctx, const PeerBuf& src, size_t src_off, void* out, const int64_t* expert_idx, const int64_t* slot_idx,
                       const float* weights, void* picked, int S, int K, int M, int E_local, int C, int dtype, int nblocks,
                       cudaStream_t stream, bool local_layout) {
    check_shape(M, dtype, nblocks);
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        moe_gather_kernel<T><<<nblocks, kMoeThreads, 0, stream>>>(ctx, src, src_off, static_cast<T*>(out), expert_idx, slot_idx, weights,
                                                                 static_cast<T*>(picked), S, K, M, E_local, C, local_layout ? 1 : 0);
    });
    check("moe_gather");
}

}  // namespace bagua
