// Fused collective kernels over NVLink 4 / NVSwitch symmetric memory (sm_90a).
//
// These replace the reference's "kernel + separate NCCL call" sequences
// (rust/bagua-core/bagua-core-internal/src/comm_ops/*.rs, communicators/mod.rs:1121-1153): the reduction,
// the averaging scale, the dtype handling, the optimizer update and the data movement to/from the peers
// happen in ONE kernel that issues peer (P2P) or NVLS multicast loads/stores itself.
#include "kernels.h"
#include "peer.cuh"

namespace bagua {
using namespace dev;

// ---------------------------------------------------------------------------------------------------------
// allreduce, two-shot over peer pointers: rank r reduces slice r (reading it from every peer) and writes the
// result into slice r of every peer. src and dst may alias (in-place): slice r is only ever read and written
// by rank r between the two barriers.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P>
__global__ void __launch_bounds__(512) allreduce_twoshot_kernel(PeerCtx ctx, PeerBuf src, PeerBuf dst, size_t src_off,
                                                                size_t dst_off, size_t total_vecs, float scale) {
    // U vectors per thread per iteration keep U*P independent 16-byte peer loads in flight (NVLink latency is ~2 us:
    // bandwidth = bytes in flight / latency, measured 7.5 GB/s per CTA without unrolling)
    constexpr int U = P <= 2 ? 8 : (P <= 4 ? 4 : 2);
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        const size_t vpr = (total_vecs + P - 1) / P;
        const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);  // exclusive end of my slice
        for (size_t j0 = base + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j0 < limit; j0 += stride * U) {
            uint4 raw[U][P];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
#pragma unroll
                    for (int i = 0; i < P; ++i) raw[u][i] = ld_peer16(src.ptr[(ctx.rank + i) % P] + src_off + v * 16);  // rotate: links hit evenly
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
                    float acc[Vec16<T>::N];
                    Vec16<T>::unpack(raw[u][0], acc);
#pragma unroll
                    for (int i = 1; i < P; ++i) {
                        float f[Vec16<T>::N];
                        Vec16<T>::unpack(raw[u][i], f);
#pragma unroll
                        for (int k = 0; k < Vec16<T>::N; ++k) acc[k] += f[k];
                    }
#pragma unroll
                    for (int k = 0; k < Vec16<T>::N; ++k) acc[k] *= scale;
                    const uint4 out = Vec16<T>::pack(acc);
#pragma unroll
                    for (int i = 0; i < P; ++i) st_peer16(dst.ptr[(ctx.rank + i) % P] + dst_off + v * 16, out);
                }
            }
        }
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

// Same schedule through the switch: one multimem.ld_reduce returns the sum over all GPUs (reduced inside
// NVSwitch), one multimem.st lands the result on all GPUs.
template <typename T>
__global__ void __launch_bounds__(512) allreduce_multimem_kernel(PeerCtx ctx, PeerBuf src, PeerBuf dst, size_t src_off,
                                                                 size_t dst_off, size_t total_vecs, float scale) {
    constexpr int U = 8;  // independent in-switch reductions in flight per thread
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        const int P = ctx.world;
        const size_t vpr = (total_vecs + P - 1) / P;
        const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);
        for (size_t j0 = base + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j0 < limit; j0 += stride * U) {
            uint4 red[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) red[u] = multimem_ld_reduce_add<T>(src.mc + src_off + v * 16);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
                    if (scale != 1.0f) {
                        float f[Vec16<T>::N];
                        Vec16<T>::unpack(red[u], f);
#pragma unroll
                        for (int k = 0; k < Vec16<T>::N; ++k) f[k] *= scale;
                        red[u] = Vec16<T>::pack(f);
                    }
                    multimem_st16(dst.mc + dst_off + v * 16, red[u]);
                }
            }
        }
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
    constexpr int U = USE_MC ? 8 : (P <= 2 ? 8 : (P <= 4 ? 4 : 2));
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    if (ok) {
        const size_t vpr = (total_vecs + P - 1) / P;
        const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);
        char* mine = buf.ptr[ctx.rank] + off;
        for (size_t j0 = base + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j0 < limit; j0 += stride * U) {
            uint4 raw[U][USE_MC ? 1 : P];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
                    if (USE_MC) {
                        raw[u][0] = multimem_ld_reduce_add<T>(buf.mc + off + v * 16);
                    } else {
#pragma unroll
                        for (int i = 0; i < (USE_MC ? 1 : P); ++i) raw[u][i] = ld_peer16(buf.ptr[(ctx.rank + i) % P] + off + v * 16);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v >= limit) continue;
                float acc[Vec16<T>::N];
                Vec16<T>::unpack(raw[u][0], acc);
                if (!USE_MC) {
#pragma unroll
                    for (int i = 1; i < (USE_MC ? 1 : P); ++i) {
                        float f[Vec16<T>::N];
                        Vec16<T>::unpack(raw[u][i], f);
#pragma unroll
                        for (int k = 0; k < Vec16<T>::N; ++k) acc[k] += f[k];
                    }
                }
#pragma unroll
                for (int k = 0; k < Vec16<T>::N; ++k) acc[k] *= scale;
                st_stream16(mine + v * 16, Vec16<T>::pack(acc));
            }
        }
        peer_barrier(ctx, e0 + 2);
    }
    store_epoch(ctx, e0 + 2);
}

template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512) all_gather_kernel(PeerCtx ctx, PeerBuf buf, size_t off, size_t total_vecs) {
    constexpr int U = 4;
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);  // nobody is still reading the slices that are about to be overwritten
    if (ok) {
        const size_t vpr = (total_vecs + P - 1) / P;
        const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);
        const char* mine = buf.ptr[ctx.rank] + off;
        for (size_t j0 = base + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j0 < limit; j0 += stride * U) {
            uint4 raw[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) raw[u] = ld_stream16(mine + v * 16);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v >= limit) continue;
                if (USE_MC) {
                    multimem_st16(buf.mc + off + v * 16, raw[u]);
                } else {
#pragma unroll
                    for (int i = 1; i < P; ++i) st_peer16(buf.ptr[(ctx.rank + i) % P] + off + v * 16, raw[u]);  // my own copy is already in place
                }
            }
        }
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
    for (size_t v = tid; v < total_vecs; v += stride) {
        const uint4 mine = ld_stream16(in + v * 16);
#pragma unroll
        for (int i = 0; i < P; ++i) {
            const int p = (ctx.rank + i) % P;
            st_peer16(staging.ptr[p] + staging_off + (parity * P + ctx.rank) * slot_bytes + v * 16, mine);
        }
    }
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
// Gradient reduce-scatter  →  SGD(momentum) on the owned 1/P slice  →  all-gather of the updated WEIGHTS,
// in one kernel. Each rank keeps fp32 master weights and momentum only for its own slice (optimizer state is
// sharded P ways), the gradient bucket is zeroed for the next iteration on the way out, and the optimizer step
// overlaps the rest of backward because it runs inside the bucket's communication kernel.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512)
    allreduce_sgd_kernel(PeerCtx ctx, PeerBuf grads, PeerBuf weights, size_t g_off, size_t w_off, size_t total_vecs,
                         float* master, float* momentum_buf, SgdParams hp, float scale, int zero_grads) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    constexpr int N = Vec16<T>::N;
    const size_t vpr = (total_vecs + P - 1) / P;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (ok) {
        constexpr int U = USE_MC ? 4 : (P <= 2 ? 4 : (P <= 4 ? 2 : 1));  // vectors in flight per thread (register budget: U*P*4)
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);
        for (size_t j0 = base + tid; j0 < limit; j0 += stride * U) {
            uint4 raw[U][USE_MC ? 1 : P];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
                    if (USE_MC) {
                        raw[u][0] = multimem_ld_reduce_add<T>(grads.mc + g_off + v * 16);
                    } else {
#pragma unroll
                        for (int i = 0; i < (USE_MC ? 1 : P); ++i) raw[u][i] = ld_peer16(grads.ptr[(ctx.rank + i) % P] + g_off + v * 16);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v >= limit) continue;
                const size_t j = v - base;
                float g[N];
                Vec16<T>::unpack(raw[u][0], g);
                if (!USE_MC) {
#pragma unroll
                    for (int i = 1; i < (USE_MC ? 1 : P); ++i) {
                        float f[N];
                        Vec16<T>::unpack(raw[u][i], f);
#pragma unroll
                        for (int k = 0; k < N; ++k) g[k] += f[k];
                    }
                }
                // optimizer state of the owned slice: index j*N within the shard
                float w[N], m[N];
                float4* mp = reinterpret_cast<float4*>(master + j * N);
                float4* mo = reinterpret_cast<float4*>(momentum_buf + j * N);
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
                const uint4 out = Vec16<T>::pack(w);
                if (USE_MC) {
                    multimem_st16(weights.mc + w_off + v * 16, out);
                } else {
#pragma unroll
                    for (int i = 0; i < P; ++i) st_peer16(weights.ptr[(ctx.rank + i) % P] + w_off + v * 16, out);
                }
            }
        }
        ok = peer_barrier(ctx, e0 + 2);
    }
    if (ok && zero_grads) {
        // Block b of every peer has finished reading column-range b of all my slices: safe to clear them.
        char* mine = grads.ptr[ctx.rank] + g_off;
        const uint4 z = make_uint4(0, 0, 0, 0);
        for (size_t j = tid; j < vpr; j += stride) {
#pragma unroll
            for (int s = 0; s < P; ++s) {
                const size_t v = static_cast<size_t>(s) * vpr + j;
                if (v < total_vecs) st_stream16(mine + v * 16, z);
            }
        }
    }
    store_epoch(ctx, e0 + 2);
}

// ---------------------------------------------------------------------------------------------------------
// The same reduce-scatter → optimizer → all-gather kernel with Adam / AdamW on the owned shard (fp32 master weights and
// both moments sharded P ways). Update rule identical to flat_adam_kernel (multi_tensor.cu) / torch.optim.Adam[W].
// ---------------------------------------------------------------------------------------------------------
template <typename T, int P, bool USE_MC>
__global__ void __launch_bounds__(512)
    allreduce_adam_kernel(PeerCtx ctx, PeerBuf grads, PeerBuf weights, size_t g_off, size_t w_off, size_t total_vecs, float* master,
                          float* exp_avg, float* exp_avg_sq, AdamParams hp, float scale, int zero_grads) {
    const uint32_t e0 = load_epoch(ctx);
    bool ok = peer_barrier(ctx, e0 + 1);
    constexpr int N = Vec16<T>::N;
    const size_t vpr = (total_vecs + P - 1) / P;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (ok) {
        constexpr int U = USE_MC ? 4 : (P <= 2 ? 4 : (P <= 4 ? 2 : 1));
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);
        const float inv_bc1 = 1.f / hp.bias_correction1, inv_sqrt_bc2 = rsqrtf(hp.bias_correction2);
        for (size_t j0 = base + tid; j0 < limit; j0 += stride * U) {
            uint4 raw[U][USE_MC ? 1 : P];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
                    if (USE_MC) {
                        raw[u][0] = multimem_ld_reduce_add<T>(grads.mc + g_off + v * 16);
                    } else {
#pragma unroll
                        for (int i = 0; i < (USE_MC ? 1 : P); ++i) raw[u][i] = ld_peer16(grads.ptr[(ctx.rank + i) % P] + g_off + v * 16);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v >= limit) continue;
                const size_t j = v - base;
                float g[N];
                Vec16<T>::unpack(raw[u][0], g);
                if (!USE_MC) {
#pragma unroll
                    for (int i = 1; i < (USE_MC ? 1 : P); ++i) {
                        float f[N];
                        Vec16<T>::unpack(raw[u][i], f);
#pragma unroll
                        for (int k = 0; k < N; ++k) g[k] += f[k];
                    }
                }
                float4* wp = reinterpret_cast<float4*>(master + j * N);
                float4* ap = reinterpret_cast<float4*>(exp_avg + j * N);
                float4* bp = reinterpret_cast<float4*>(exp_avg_sq + j * N);
                float w[N];
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
                        const float denom = sqrtf(bv[k]) * inv_sqrt_bc2 + hp.eps;
                        wv[k] -= (hp.lr * inv_bc1) * (av[k] / denom);
                        w[4 * q + k] = wv[k];
                    }
                    wp[q] = make_float4(wv[0], wv[1], wv[2], wv[3]);
                    ap[q] = make_float4(av[0], av[1], av[2], av[3]);
                    bp[q] = make_float4(bv[0], bv[1], bv[2], bv[3]);
                }
                const uint4 out = Vec16<T>::pack(w);
                if (USE_MC) {
                    multimem_st16(weights.mc + w_off + v * 16, out);
                } else {
#pragma unroll
                    for (int i = 0; i < P; ++i) st_peer16(weights.ptr[(ctx.rank + i) % P] + w_off + v * 16, out);
                }
            }
        }
        ok = peer_barrier(ctx, e0 + 2);
    }
    if (ok && zero_grads) {
        char* mine = grads.ptr[ctx.rank] + g_off;
        const uint4 z = make_uint4(0, 0, 0, 0);
        for (size_t j = tid; j < vpr; j += stride) {
#pragma unroll
            for (int s = 0; s < P; ++s) {
                const size_t v = static_cast<size_t>(s) * vpr + j;
                if (v < total_vecs) st_stream16(mine + v * 16, z);
            }
        }
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
// Column striping: CTA b touches vectors {s·vpr + j : j ≡ (b, thread) mod grid} of every slice s in all three phases, so the
// per-CTA barriers (CTA b of every rank) are all the synchronisation needed; there is no grid-wide barrier.
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
    const size_t vpr = (total_vecs + P - 1) / P;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    char* my_snap = snap.ptr[ctx.rank] + snap_off;
    // 1: snapshot (weights may be mid-update by the optimizer on another stream: every 16-byte vector is still a value the
    //    weight had at some instant, which is all the element-wise averaging algebra needs)
    for (size_t j = tid; j < vpr; j += stride) {
#pragma unroll
        for (int s = 0; s < P; ++s) {
            const size_t v = static_cast<size_t>(s) * vpr + j;
            if (v < total_vecs) st_stream16(my_snap + v * 16, ld_peer16(w + v * 16));
        }
    }
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
        constexpr int U = USE_MC ? 8 : (P <= 2 ? 8 : (P <= 4 ? 4 : 2));
        const size_t base = static_cast<size_t>(ctx.rank) * vpr;
        const size_t limit = (base + vpr < total_vecs ? base + vpr : total_vecs);
        const float inv = 1.0f / P;
        for (size_t j0 = base + tid; j0 < limit; j0 += stride * U) {
            uint4 raw[U][USE_MC ? 1 : P];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v < limit) {
                    if (USE_MC) {
                        raw[u][0] = multimem_ld_reduce_add<T>(snap.mc + snap_off + v * 16);
                    } else {
#pragma unroll
                        for (int i = 0; i < (USE_MC ? 1 : P); ++i) raw[u][i] = ld_peer16(snap.ptr[(ctx.rank + i) % P] + snap_off + v * 16);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = j0 + u * stride;
                if (v >= limit) continue;
                float acc[N];
                Vec16<T>::unpack(raw[u][0], acc);
                if (!USE_MC) {
#pragma unroll
                    for (int i = 1; i < (USE_MC ? 1 : P); ++i) {
                        float f[N];
                        Vec16<T>::unpack(raw[u][i], f);
#pragma unroll
                        for (int k = 0; k < N; ++k) acc[k] += f[k];
                    }
                }
#pragma unroll
                for (int k = 0; k < N; ++k) acc[k] *= inv;
                const uint4 out = Vec16<T>::pack(acc);
                if (USE_MC) {
                    multimem_st16(avg.mc + avg_off + v * 16, out);
                } else {
#pragma unroll
                    for (int i = 0; i < P; ++i) st_peer16(avg.ptr[(ctx.rank + i) % P] + avg_off + v * 16, out);
                }
            }
        }
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
                for (size_t j = tid; j < vpr; j += stride) {
#pragma unroll
                    for (int s = 0; s < P; ++s) {
                        const size_t v = static_cast<size_t>(s) * vpr + j;
                        if (v >= total_vecs) continue;
                        float a[N], sn[N], cur[N];
                        Vec16<T>::unpack(ld_peer16(my_avg + v * 16), a);       // written by rank s during this kernel
                        Vec16<T>::unpack(ld_stream16(my_snap + v * 16), sn);  // written by this very thread in phase 1
                        Vec16<T>::unpack(ld_peer16(w + v * 16), cur);         // the weights as they are NOW
#pragma unroll
                        for (int k = 0; k < N; ++k) cur[k] += a[k] - sn[k];
                        st_stream16(w + v * 16, Vec16<T>::pack(cur));
                    }
                }
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
template <typename F>
void dispatch_world(int world, F&& f) {
    switch (world) {
        case 1: f(std::integral_constant<int, 1>{}); break;
        case 2: f(std::integral_constant<int, 2>{}); break;
        case 3: f(std::integral_constant<int, 3>{}); break;
        case 4: f(std::integral_constant<int, 4>{}); break;
        case 5: f(std::integral_constant<int, 5>{}); break;
        case 6: f(std::integral_constant<int, 6>{}); break;
        case 7: f(std::integral_constant<int, 7>{}); break;
        case 8: f(std::integral_constant<int, 8>{}); break;
        default: throw std::runtime_error("bagua: peer kernels support 1..8 ranks, got " + std::to_string(world));
    }
}
template <typename F>
void dispatch_float(int dtype, F&& f) {
    switch (dtype) {
        case F32: f(float{}); break;
        case F16: f(__half{}); break;
        case BF16: f(__nv_bfloat16{}); break;
        default: throw std::runtime_error("bagua: peer reduction kernels need f32/f16/bf16, got dtype code " + std::to_string(dtype));
    }
}
void check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of ") + what + " failed: " + cudaGetErrorString(e));
    count_launch();
}
void check_blocks(int nblocks) {
    if (nblocks < 1 || nblocks > kMaxCommBlocks) throw std::runtime_error("bagua: peer kernel grid must be 1.." + std::to_string(kMaxCommBlocks));
}
}  // namespace

void launch_allreduce(const PeerCtx& ctx, const PeerBuf& src, const PeerBuf& dst, size_t src_off, size_t dst_off,
                      size_t bytes, int dtype, float scale, int variant, int nblocks, int nthreads, cudaStream_t stream) {
    if (bytes % 16 || src_off % 16 || dst_off % 16) throw std::runtime_error("bagua: allreduce needs 16-byte aligned size/offsets");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        if (variant == AR_MULTIMEM) {
            if (!src.mc || !dst.mc) throw std::runtime_error("bagua: multimem allreduce requested but no multicast mapping");
            allreduce_multimem_kernel<T><<<nblocks, nthreads, 0, stream>>>(ctx, src, dst, src_off, dst_off, vecs, scale);
        } else {
            dispatch_world(ctx.world, [&](auto pw) {
                constexpr int P = decltype(pw)::value;
                allreduce_twoshot_kernel<T, P><<<nblocks, nthreads, 0, stream>>>(ctx, src, dst, src_off, dst_off, vecs, scale);
            });
        }
    });
    check_launch("allreduce");
}

void launch_allreduce_oneshot(const PeerCtx& ctx, const PeerBuf& staging, size_t staging_off, size_t slot_bytes, const void* in, void* out,
                              size_t bytes, int dtype, float scale, int nblocks, int nthreads, cudaStream_t stream, uint32_t call_parity) {
    if (bytes % 16) throw std::runtime_error("bagua: one-shot allreduce needs a 16-byte multiple");
    if (bytes > slot_bytes) throw std::runtime_error("bagua: one-shot allreduce message larger than its staging slot");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(ctx.world, [&](auto pw) {
            constexpr int P = decltype(pw)::value;
            allreduce_oneshot_kernel<T, P><<<nblocks, nthreads, 0, stream>>>(
                ctx, staging, staging_off, slot_bytes, static_cast<const char*>(in), static_cast<char*>(out), vecs, scale, call_parity);
        });
    });
    check_launch("allreduce_oneshot");
}

void launch_allreduce_sgd(const PeerCtx& ctx, const PeerBuf& grads, const PeerBuf& weights, size_t g_off, size_t w_off,
                          size_t bytes, int dtype, float* master, float* momentum, const SgdParams& hp, float scale,
                          bool zero_grads, bool use_multimem, int nblocks, int nthreads, cudaStream_t stream) {
    if (bytes % 16 || g_off % 16 || w_off % 16) throw std::runtime_error("bagua: allreduce_sgd needs 16-byte aligned size/offsets");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(ctx.world, [&](auto pw) {
            constexpr int P = decltype(pw)::value;
            if (use_multimem)
                allreduce_sgd_kernel<T, P, true><<<nblocks, nthreads, 0, stream>>>(ctx, grads, weights, g_off, w_off, vecs, master,
                                                                                 momentum, hp, scale, zero_grads ? 1 : 0);
            else
                allreduce_sgd_kernel<T, P, false><<<nblocks, nthreads, 0, stream>>>(ctx, grads, weights, g_off, w_off, vecs, master,
                                                                                  momentum, hp, scale, zero_grads ? 1 : 0);
        });
    });
    check_launch("allreduce_sgd");
}

void launch_reduce_scatter(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, float scale, bool use_multimem, int nblocks,
                           int nthreads, cudaStream_t stream) {
    if (bytes % 16 || off % 16) throw std::runtime_error("bagua: reduce_scatter needs 16-byte aligned size/offset");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(ctx.world, [&](auto pw) {
            constexpr int P = decltype(pw)::value;
            if (use_multimem)
                reduce_scatter_kernel<T, P, true><<<nblocks, nthreads, 0, stream>>>(ctx, buf, off, vecs, scale);
            else
                reduce_scatter_kernel<T, P, false><<<nblocks, nthreads, 0, stream>>>(ctx, buf, off, vecs, scale);
        });
    });
    check_launch("reduce_scatter");
}

void launch_all_gather(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, bool use_multimem, int nblocks, int nthreads,
                       cudaStream_t stream) {
    if (bytes % 16 || off % 16) throw std::runtime_error("bagua: all_gather needs 16-byte aligned size/offset");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(ctx.world, [&](auto pw) {
            constexpr int P = decltype(pw)::value;
            if (use_multimem)
                all_gather_kernel<T, P, true><<<nblocks, nthreads, 0, stream>>>(ctx, buf, off, vecs);
            else
                all_gather_kernel<T, P, false><<<nblocks, nthreads, 0, stream>>>(ctx, buf, off, vecs);
        });
    });
    check_launch("all_gather");
}

void launch_allreduce_adam(const PeerCtx& ctx, const PeerBuf& grads, const PeerBuf& weights, size_t g_off, size_t w_off, size_t bytes, int dtype,
                           float* master, float* exp_avg, float* exp_avg_sq, const AdamParams& hp, float scale, bool zero_grads, bool use_multimem,
                           int nblocks, int nthreads, cudaStream_t stream) {
    if (bytes % 16 || g_off % 16 || w_off % 16) throw std::runtime_error("bagua: allreduce_adam needs 16-byte aligned size/offsets");
    if (hp.amsgrad) throw std::runtime_error("bagua: allreduce_adam does not implement amsgrad");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(ctx.world, [&](auto pw) {
            constexpr int P = decltype(pw)::value;
            if (use_multimem)
                allreduce_adam_kernel<T, P, true><<<nblocks, nthreads, 0, stream>>>(ctx, grads, weights, g_off, w_off, vecs, master, exp_avg,
                                                                                  exp_avg_sq, hp, scale, zero_grads ? 1 : 0);
            else
                allreduce_adam_kernel<T, P, false><<<nblocks, nthreads, 0, stream>>>(ctx, grads, weights, g_off, w_off, vecs, master, exp_avg,
                                                                                   exp_avg_sq, hp, scale, zero_grads ? 1 : 0);
        });
    });
    check_launch("allreduce_adam");
}

void launch_peer_average(const PeerCtx& ctx, const PeerBuf& weights, size_t off, int peer, void* out, size_t bytes, int dtype,
                         int nblocks, int nthreads, cudaStream_t stream) {
    if (bytes % 16 || off % 16) throw std::runtime_error("bagua: peer_average needs 16-byte aligned size/offset");
    if (peer < 0 || peer >= ctx.world) throw std::runtime_error("bagua: peer_average peer rank out of range");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        peer_average_kernel<T><<<nblocks, nthreads, 0, stream>>>(ctx, weights, off, peer, static_cast<char*>(out), vecs);
    });
    check_launch("peer_average");
}

void launch_async_average(const PeerCtx& ctx, void* w, const PeerBuf& snap, size_t snap_off, const PeerBuf& avg, size_t avg_off, size_t bytes, int dtype,
                          uint32_t seq, bool go, uint32_t* gate, unsigned long long gate_timeout_ns, int* status, bool use_multimem, int nblocks, int nthreads,
                          cudaStream_t stream) {
    if (bytes % 16 || snap_off % 16 || avg_off % 16) throw std::runtime_error("bagua: async_average needs 16-byte aligned size/offsets");
    check_blocks(nblocks);
    const size_t vecs = bytes / 16;
    if (vecs == 0) return;
    if (use_multimem && (!snap.mc || !avg.mc)) throw std::runtime_error("bagua: multimem async_average requested but no multicast mapping");
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        dispatch_world(ctx.world, [&](auto pw) {
            constexpr int P = decltype(pw)::value;
            if (use_multimem)
                async_average_kernel<T, P, true><<<nblocks, nthreads, 0, stream>>>(ctx, static_cast<char*>(w), snap, snap_off, avg, avg_off, vecs, seq, go ? 1 : 0,
                                                                                 gate, gate_timeout_ns, status);
            else
                async_average_kernel<T, P, false><<<nblocks, nthreads, 0, stream>>>(ctx, static_cast<char*>(w), snap, snap_off, avg, avg_off, vecs, seq, go ? 1 : 0,
                                                                                  gate, gate_timeout_ns, status);
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
