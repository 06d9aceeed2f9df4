// Fused NHWC (channels_last) epilogues for convolutional blocks: bias + ReLU (+ 2x2/2 max-pool) forward and backward.
//
// In eager PyTorch a conv block is conv → bias add → ReLU → max-pool, each a full pass over the activation tensor, and
// the backward adds a ReLU mask pass, a (slow, strided) bias-gradient reduction and a generic max-pool backward. These
// bandwidth passes can cost more than the tensor-core convolutions themselves. Here every block epilogue is ONE pass with 16-byte accesses:
//   fwd : y = relu(conv_out + bias)                       (in place)          | out, idx = maxpool2(relu(conv_out + bias))
//   bwd : g' = g * (y > 0);  bias_grad += Σ g'                               | g_in = scatter(g * (out > 0), idx);  bias_grad += Σ
// The convolution itself stays a library call (cuDNN); it is run without bias so cuDNN skips its own bias-grad reduction.
//
// NaN follows torch: relu(NaN) = NaN, its gradient passes (the mask is !(y <= 0), as in threshold_backward), and the pool's
// argmax is the first maximum in scan order (0,0), (0,1), (1,0), (1,1) unless the window holds a NaN, then it is the last NaN
// (max_pool2d's `val > max || isnan(val)`). The window max is taken over the pre-bias input (bias and ReLU are monotone).
// Every pointer is accessed with 16-byte vectors (the pool's argmax bytes with 8-byte words); the launchers reject a
// misaligned one before anything reaches the device.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <stdexcept>
#include <string>

#include "kernels.h"
#include "peer.cuh"
#include "quant.cuh"

namespace bagua {
using namespace dev;

namespace {
constexpr int kThreads = 256;

template <typename T>
__device__ __forceinline__ void load8(const T* p, float* f) {  // 8 consecutive channels (16 bytes of bf16/f16)
    Vec16<T>::unpack(*reinterpret_cast<const uint4*>(p), f);
}
template <typename T>
__device__ __forceinline__ void store8(T* p, const float* f) {
    *reinterpret_cast<uint4*>(p) = Vec16<T>::pack(f);
}
// relu that keeps NaN (fmaxf(NaN, 0) would return 0); also the backward mask: keep where !(v <= 0)
__device__ __forceinline__ float relu_nan(float v) { return v <= 0.f ? 0.f : v; }

// ---- bias + relu -------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) bias_relu_fwd_kernel(T* __restrict__ y, const T* __restrict__ bias, size_t total_vecs, int cpv) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t v = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < total_vecs; v += stride) {
        float a[8], b[8];
        load8<T>(y + v * 8, a);
        load8<T>(bias + (v % cpv) * 8, b);
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = relu_nan(a[k] + b[k]);
        store8<T>(y + v * 8, a);
    }
}

// FIN variants: the bias-gradient reduction is finished INSIDE the kernel. Every CTA adds its partial sums to a zeroed fp32
// workspace, takes a ticket, and the CTA that draws the last ticket converts the sums to the bias dtype, writes them to
// `bias_grad_out` and leaves workspace + ticket counter zeroed for the next launch on this stream — no separate fill and cast
// launches around the kernel (26 tiny launches per VGG16 step otherwise).
template <typename T>
__device__ __forceinline__ void finish_bias_grad(float* ws, T* bias_grad_out, unsigned int* ticket, int C) {
    __shared__ bool is_last;
    __threadfence();  // this CTA's atomics are visible before its ticket is
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (is_last) {
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            bias_grad_out[c] = from_f32<T>(__ldcg(ws + c));  // L2 value: other CTAs' atomics never touched this SM's L1
            ws[c] = 0.f;
        }
        if (threadIdx.x == 0) *ticket = 0u;
    }
}

// block = (rows_per_iter x cpv) threads; thread keeps 8 channel partial sums over the rows it visits
template <typename T, bool FIN>
__global__ void __launch_bounds__(kThreads) bias_relu_bwd_kernel(const T* __restrict__ g, const T* __restrict__ y, T* __restrict__ gout,
                                                                 float* __restrict__ bias_grad, size_t rows, int C, T* __restrict__ bias_grad_out,
                                                                 unsigned int* __restrict__ ticket) {
    extern __shared__ float s_sum[];  // [C]
    const int cpv = C / 8;
    const int rpb = kThreads / cpv;
    const int cv = threadIdx.x % cpv, r = threadIdx.x / cpv;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s_sum[c] = 0.f;
    __syncthreads();
    float part[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (r < rpb) {
        for (size_t row = static_cast<size_t>(blockIdx.x) * rpb + r; row < rows; row += static_cast<size_t>(gridDim.x) * rpb) {
            const size_t off = row * C + cv * 8;
            float a[8], b[8];
            load8<T>(g + off, a);
            load8<T>(y + off, b);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                a[k] = b[k] <= 0.f ? 0.f : a[k];
                part[k] += a[k];
            }
            store8<T>(gout + off, a);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) atomicAdd(&s_sum[cv * 8 + k], part[k]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&bias_grad[c], s_sum[c]);
    if constexpr (FIN) finish_bias_grad<T>(bias_grad, bias_grad_out, ticket, C);
}

// ---- bias + relu + maxpool 2x2 stride 2 ----------------------------------------------------------------------------------
// x: [N, H, W, C]; out: [N, H/2, W/2, C]; idx: uint8 same shape as out (argmax position 0..3 = dy*2+dx)
template <typename T>
__global__ void __launch_bounds__(kThreads) bias_relu_pool_fwd_kernel(const T* __restrict__ x, const T* __restrict__ bias, T* __restrict__ out,
                                                                      uint8_t* __restrict__ idx, int N, int H, int W, int C) {
    const int cpv = C / 8, Ho = H / 2, Wo = W / 2;
    const size_t total = static_cast<size_t>(N) * Ho * Wo * cpv;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t v = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < total; v += stride) {
        const int cv = static_cast<int>(v % cpv);
        size_t t = v / cpv;
        const int wo = static_cast<int>(t % Wo);
        t /= Wo;
        const int ho = static_cast<int>(t % Ho);
        const int n = static_cast<int>(t / Ho);
        const size_t base = ((static_cast<size_t>(n) * H + 2 * ho) * W + 2 * wo) * C + cv * 8;
        float m[8], b[8], f[8];
        uint32_t arg[8];
        load8<T>(x + base, m);
#pragma unroll
        for (int k = 0; k < 8; ++k) arg[k] = 0;
        const size_t offs[3] = {static_cast<size_t>(C), static_cast<size_t>(W) * C, static_cast<size_t>(W) * C + C};
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            load8<T>(x + base + offs[q], f);
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (f[k] > m[k] || f[k] != f[k]) m[k] = f[k], arg[k] = q + 1;
        }
        load8<T>(bias + cv * 8, b);
#pragma unroll
        for (int k = 0; k < 8; ++k) m[k] = relu_nan(m[k] + b[k]);
        const size_t o = v * 8;
        store8<T>(out + o, m);
        uint2 packed;
        packed.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
        packed.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | (arg[7] << 24);
        *reinterpret_cast<uint2*>(idx + o) = packed;
    }
}

template <typename T, bool FIN>
__global__ void __launch_bounds__(kThreads) bias_relu_pool_bwd_kernel(const T* __restrict__ g, const T* __restrict__ out, const uint8_t* __restrict__ idx,
                                                                      T* __restrict__ gin, float* __restrict__ bias_grad, int N, int H, int W, int C,
                                                                      T* __restrict__ bias_grad_out, unsigned int* __restrict__ ticket) {
    extern __shared__ float s_sum[];
    const int cpv = C / 8, Ho = H / 2, Wo = W / 2;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s_sum[c] = 0.f;
    __syncthreads();
    // consecutive threads own consecutive channel vectors of the same output pixel; a thread keeps the same cv across its
    // grid-stride iterations when the stride is a multiple of cpv (grid chosen accordingly), so it can accumulate locally
    const size_t total = static_cast<size_t>(N) * Ho * Wo * cpv;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    float part[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const int cv = static_cast<int>((static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) % cpv);
    for (size_t v = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < total; v += stride) {
        size_t t = v / cpv;
        const int wo = static_cast<int>(t % Wo);
        t /= Wo;
        const int ho = static_cast<int>(t % Ho);
        const int n = static_cast<int>(t / Ho);
        float a[8], y[8];
        load8<T>(g + v * 8, a);
        load8<T>(out + v * 8, y);
        const uint2 packed = *reinterpret_cast<const uint2*>(idx + v * 8);
        uint32_t arg[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) arg[k] = (packed.x >> (8 * k)) & 0xffu, arg[4 + k] = (packed.y >> (8 * k)) & 0xffu;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            a[k] = y[k] <= 0.f ? 0.f : a[k];
            part[k] += a[k];
        }
        const size_t base = ((static_cast<size_t>(n) * H + 2 * ho) * W + 2 * wo) * C + cv * 8;
        const size_t offs[4] = {0, static_cast<size_t>(C), static_cast<size_t>(W) * C, static_cast<size_t>(W) * C + C};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float o[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = (arg[k] == static_cast<uint32_t>(q)) ? a[k] : 0.f;
            store8<T>(gin + base + offs[q], o);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) atomicAdd(&s_sum[cv * 8 + k], part[k]);
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&bias_grad[c], s_sum[c]);
    if constexpr (FIN) finish_bias_grad<T>(bias_grad, bias_grad_out, ticket, C);
}

template <typename F>
void dispatch_half(int dtype, F&& f) {
    switch (dtype) {
        case F16: f(__half{}); break;
        case BF16: f(__nv_bfloat16{}); break;
        default: throw std::runtime_error("bagua: NHWC fused epilogues support f16/bf16, got dtype code " + std::to_string(dtype));
    }
}
void check(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of ") + what + " failed: " + cudaGetErrorString(e));
    count_launch();
}
void check_c(int C) {
    if (C % 8 || C > 2048) throw std::runtime_error("bagua: NHWC fused epilogues need C % 8 == 0 and C <= 2048");
}
// The kernels access these pointers with 16-byte vectors (the argmax bytes with 8-byte words). A view into a packed buffer (a
// conv bias after a parameter whose size is not a multiple of 8) can be off by a few bytes; fail here instead of on the device.
void check_aligned(const char* kernel, const char* arg, const void* p, size_t bytes = 16) {
    if (reinterpret_cast<uintptr_t>(p) % bytes)
        throw std::runtime_error(std::string("bagua: ") + kernel + ": `" + arg + "` must be " + std::to_string(bytes) + "-byte aligned");
}
int grid_for(size_t items, int multiple_of = 1) {
    size_t b = (items + kThreads - 1) / kThreads;
    const size_t cap = 132 * 8;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    if (multiple_of > 1) b = (b + multiple_of - 1) / multiple_of * multiple_of;
    return static_cast<int>(b);
}
}  // namespace

void launch_bias_relu_nhwc_fwd(void* y, const void* bias, size_t rows, int C, int dtype, cudaStream_t stream) {
    check_c(C);
    check_aligned("bias_relu_nhwc_fwd", "y", y);
    check_aligned("bias_relu_nhwc_fwd", "bias", bias);
    const size_t vecs = rows * C / 8;
    if (!vecs) return;
    dispatch_half(dtype, [&](auto tag) {
        using T = decltype(tag);
        bias_relu_fwd_kernel<T><<<grid_for(vecs / 2 + 1), kThreads, 0, stream>>>(static_cast<T*>(y), static_cast<const T*>(bias), vecs, C / 8);
    });
    check("bias_relu_nhwc_fwd");
}

void launch_bias_relu_nhwc_bwd(const void* g, const void* y, void* gout, float* bias_grad, size_t rows, int C, int dtype, cudaStream_t stream,
                               void* bias_grad_out, unsigned int* ticket) {
    check_c(C);
    check_aligned("bias_relu_nhwc_bwd", "g", g);
    check_aligned("bias_relu_nhwc_bwd", "y", y);
    check_aligned("bias_relu_nhwc_bwd", "gout", gout);
    if (!rows) return;
    const int cpv = C / 8;
    if (cpv > kThreads) throw std::runtime_error("bagua: bias_relu_nhwc_bwd needs C <= 2048");
    const int rpb = kThreads / cpv;
    dispatch_half(dtype, [&](auto tag) {
        using T = decltype(tag);
        const int grid = grid_for(rows / rpb * kThreads / 4 + 1);
        if (bias_grad_out)  // in-kernel finish: `bias_grad` is the zeroed fp32 workspace
            bias_relu_bwd_kernel<T, true><<<grid, kThreads, C * sizeof(float), stream>>>(static_cast<const T*>(g), static_cast<const T*>(y),
                                                                                          static_cast<T*>(gout), bias_grad, rows, C,
                                                                                          static_cast<T*>(bias_grad_out), ticket);
        else
            bias_relu_bwd_kernel<T, false><<<grid, kThreads, C * sizeof(float), stream>>>(static_cast<const T*>(g), static_cast<const T*>(y),
                                                                                           static_cast<T*>(gout), bias_grad, rows, C, nullptr, nullptr);
    });
    check("bias_relu_nhwc_bwd");
}

void launch_bias_relu_pool_nhwc_fwd(const void* x, const void* bias, void* out, uint8_t* idx, int N, int H, int W, int C, int dtype,
                                    cudaStream_t stream) {
    check_c(C);
    if (H % 2 || W % 2) throw std::runtime_error("bagua: fused max-pool needs even H and W");
    check_aligned("bias_relu_pool_nhwc_fwd", "x", x);
    check_aligned("bias_relu_pool_nhwc_fwd", "bias", bias);
    check_aligned("bias_relu_pool_nhwc_fwd", "out", out);
    check_aligned("bias_relu_pool_nhwc_fwd", "idx", idx, 8);
    const size_t vecs = static_cast<size_t>(N) * (H / 2) * (W / 2) * (C / 8);
    if (!vecs) return;
    dispatch_half(dtype, [&](auto tag) {
        using T = decltype(tag);
        bias_relu_pool_fwd_kernel<T><<<grid_for(vecs), kThreads, 0, stream>>>(static_cast<const T*>(x), static_cast<const T*>(bias), static_cast<T*>(out),
                                                                               idx, N, H, W, C);
    });
    check("bias_relu_pool_nhwc_fwd");
}

void launch_bias_relu_pool_nhwc_bwd(const void* g, const void* out, const uint8_t* idx, void* gin, float* bias_grad, int N, int H, int W, int C,
                                    int dtype, cudaStream_t stream, void* bias_grad_out, unsigned int* ticket) {
    check_c(C);
    const int cpv = C / 8;
    if (kThreads % cpv) throw std::runtime_error("bagua: fused max-pool backward needs C/8 to divide 256");
    check_aligned("bias_relu_pool_nhwc_bwd", "g", g);
    check_aligned("bias_relu_pool_nhwc_bwd", "out", out);
    check_aligned("bias_relu_pool_nhwc_bwd", "idx", idx, 8);
    check_aligned("bias_relu_pool_nhwc_bwd", "gin", gin);
    const size_t vecs = static_cast<size_t>(N) * (H / 2) * (W / 2) * cpv;
    if (!vecs) return;
    dispatch_half(dtype, [&](auto tag) {
        using T = decltype(tag);
        // blockDim (256) is a multiple of cpv, hence so is the grid stride: a thread always sees the same channel vector
        const int grid = grid_for(vecs / 2 + 1);
        if (bias_grad_out)
            bias_relu_pool_bwd_kernel<T, true><<<grid, kThreads, C * sizeof(float), stream>>>(static_cast<const T*>(g), static_cast<const T*>(out), idx,
                                                                                               static_cast<T*>(gin), bias_grad, N, H, W, C,
                                                                                               static_cast<T*>(bias_grad_out), ticket);
        else
            bias_relu_pool_bwd_kernel<T, false><<<grid, kThreads, C * sizeof(float), stream>>>(static_cast<const T*>(g), static_cast<const T*>(out), idx,
                                                                                                static_cast<T*>(gin), bias_grad, N, H, W, C, nullptr, nullptr);
    });
    check("bias_relu_pool_nhwc_bwd");
}

}  // namespace bagua

// ---- C table for the torch extension ----------------------------------------------------------------------------------------
namespace bagua {
namespace {
thread_local std::string g_nhwc_error;
template <typename F>
int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& e) {
        g_nhwc_error = e.what();
        return 1;
    }
}
int api_bias_relu_fwd(void* y, const void* bias, size_t rows, int C, int dtype, void* stream) {
    return guarded([&] { launch_bias_relu_nhwc_fwd(y, bias, rows, C, dtype, static_cast<cudaStream_t>(stream)); });
}
int api_bias_relu_bwd(const void* g, const void* y, void* gout, float* bias_grad, size_t rows, int C, int dtype, void* stream, void* bias_grad_out,
                      unsigned int* ticket) {
    return guarded([&] { launch_bias_relu_nhwc_bwd(g, y, gout, bias_grad, rows, C, dtype, static_cast<cudaStream_t>(stream), bias_grad_out, ticket); });
}
int api_pool_fwd(const void* x, const void* bias, void* out, uint8_t* idx, int N, int H, int W, int C, int dtype, void* stream) {
    return guarded([&] { launch_bias_relu_pool_nhwc_fwd(x, bias, out, idx, N, H, W, C, dtype, static_cast<cudaStream_t>(stream)); });
}
int api_pool_bwd(const void* g, const void* out, const uint8_t* idx, void* gin, float* bias_grad, int N, int H, int W, int C, int dtype, void* stream,
                 void* bias_grad_out, unsigned int* ticket) {
    return guarded(
        [&] { launch_bias_relu_pool_nhwc_bwd(g, out, idx, gin, bias_grad, N, H, W, C, dtype, static_cast<cudaStream_t>(stream), bias_grad_out, ticket); });
}
const char* api_last_error() { return g_nhwc_error.c_str(); }
const BaguaNhwcApi g_nhwc_api = {api_bias_relu_fwd, api_bias_relu_bwd, api_pool_fwd, api_pool_bwd, api_last_error};
}  // namespace

extern "C" __attribute__((visibility("default"))) const BaguaNhwcApi* bagua_nhwc_api() { return &g_nhwc_api; }
}  // namespace bagua

