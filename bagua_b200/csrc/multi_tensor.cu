// Fused optimizers for sm_90a.
//
// The reference's "generic fused optimizer" is a pure-python storage-aliasing trick that still runs the stock
// per-op torch kernels (bagua/torch_api/contrib/fuse/optimizer.py:318-341; several passes over HBM per step).
// Here the whole update of a flat arena — grad unscale, weight decay, momentum / Adam moments, fp32 master
// update, cast of the new weights to the model dtype and zeroing of the gradient — is ONE pass with 16-byte
// accesses, i.e. the HBM3 floor for an optimizer step. A chunked multi-tensor variant covers parameters that
// are not contiguous.
#include <stdexcept>
#include <string>

#include "dispatch.h"
#include "kernels.h"
#include "lamb.cuh"
#include "lars.cuh"
#include "lion.cuh"
#include "quant.cuh"

namespace bagua {
using namespace dev;

namespace {
constexpr int kThreads = 512;
constexpr int kVec = 8;  // elements per thread per iteration

template <typename T>
struct alignas(sizeof(T) * kVec) Pack {
    T v[kVec];
};

template <typename T>
__device__ __forceinline__ void load_pack(const T* p, size_t i, float* f) {
    Pack<T> raw = *reinterpret_cast<const Pack<T>*>(p + i);
#pragma unroll
    for (int k = 0; k < kVec; ++k) f[k] = to_f32<T>(raw.v[k]);
}
template <typename T>
__device__ __forceinline__ void store_pack(T* p, size_t i, const float* f) {
    Pack<T> raw;
#pragma unroll
    for (int k = 0; k < kVec; ++k) raw.v[k] = from_f32<T>(f[k]);
    *reinterpret_cast<Pack<T>*>(p + i) = raw;
}

__device__ __forceinline__ void sgd_update(float& w, float g, float& m, const SgdParams& hp, float grad_scale) {
    float d = g * grad_scale + hp.weight_decay * w;
    if (hp.momentum != 0.f) {
        m = hp.first_step ? d : hp.momentum * m + (1.f - hp.dampening) * d;
        d = hp.nesterov ? d + hp.momentum * m : m;
    }
    w -= hp.lr * d;
}

__device__ __forceinline__ void adam_update(float& w, float g, float& m, float& v, const AdamParams& hp, float grad_scale) {
    g *= grad_scale;
    if (hp.adamw)
        w *= (1.f - hp.lr * hp.weight_decay);
    else
        g += hp.weight_decay * w;
    m = hp.beta1 * m + (1.f - hp.beta1) * g;
    v = hp.beta2 * v + (1.f - hp.beta2) * g * g;
    const float denom = sqrtf(v) / sqrtf(hp.bias_correction2) + hp.eps;
    w -= (hp.lr / hp.bias_correction1) * (m / denom);
}

inline int flat_grid(size_t numel) {
    size_t b = (numel + static_cast<size_t>(kThreads) * kVec - 1) / (static_cast<size_t>(kThreads) * kVec);
    const size_t cap = 132 * 4;  // 4 resident CTAs of 512 threads per SM (H100: 132 SMs)
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return static_cast<int>(b);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31u) == 0; }  // packs of 8 fp32 = 32 B
}  // namespace

// ---- flat SGD ---------------------------------------------------------------------------------------------------
template <typename PT, typename GT, typename MT, bool HAS_MODEL, bool VEC>
__global__ void __launch_bounds__(kThreads) flat_sgd_kernel(PT* __restrict__ param, GT* __restrict__ grad, float* __restrict__ mom,
                                                            MT* __restrict__ model, size_t n, SgdParams hp, float grad_scale,
                                                            int zero_grad) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool has_mom = hp.momentum != 0.f;
    if (VEC) {
        const size_t nv = n / kVec;
        for (size_t j = tid; j < nv; j += stride) {
            const size_t i = j * kVec;
            float w[kVec], g[kVec], m[kVec];
            load_pack<PT>(param, i, w);
            load_pack<GT>(grad, i, g);
            if (has_mom && !hp.first_step) load_pack<float>(mom, i, m);
#pragma unroll
            for (int k = 0; k < kVec; ++k) sgd_update(w[k], g[k], m[k], hp, grad_scale);
            store_pack<PT>(param, i, w);
            if (has_mom) store_pack<float>(mom, i, m);
            if (HAS_MODEL) store_pack<MT>(model, i, w);
            if (zero_grad) {
                float z[kVec] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                store_pack<GT>(grad, i, z);
            }
        }
    }
    const size_t start = VEC ? (n / kVec) * kVec : 0;
    for (size_t i = start + tid; i < n; i += stride) {
        float w = to_f32<PT>(param[i]), g = to_f32<GT>(grad[i]), m = (has_mom && !hp.first_step) ? mom[i] : 0.f;
        sgd_update(w, g, m, hp, grad_scale);
        param[i] = from_f32<PT>(w);
        if (has_mom) mom[i] = m;
        if (HAS_MODEL) model[i] = from_f32<MT>(w);
        if (zero_grad) grad[i] = from_f32<GT>(0.f);
    }
}

void launch_flat_sgd(void* param, int param_dtype, const void* grad, int grad_dtype, float* momentum_buf, void* model,
                     int model_dtype, size_t numel, const SgdParams& hp, float grad_scale, bool zero_grad, cudaStream_t stream) {
    if (!numel) return;
    if (hp.momentum != 0.f && !momentum_buf) throw std::runtime_error("bagua: flat_sgd with momentum needs a momentum buffer");
    const bool vec = aligned16(param) && aligned16(grad) && (!momentum_buf || aligned16(momentum_buf)) && (!model || aligned16(model));
    const int grid = flat_grid(numel);
    dispatch_float(param_dtype, "optimizer kernels", [&](auto pt) {
        using PT = decltype(pt);
        dispatch_float(grad_dtype, "optimizer kernels", [&](auto gt) {
            using GT = decltype(gt);
            auto* g = const_cast<GT*>(static_cast<const GT*>(grad));
            auto launch = [&](auto mt, auto has_model) {
                using MT = decltype(mt);
                constexpr bool HM = decltype(has_model)::value;
                if (vec)
                    flat_sgd_kernel<PT, GT, MT, HM, true><<<grid, kThreads, 0, stream>>>(
                        static_cast<PT*>(param), g, momentum_buf, static_cast<MT*>(model), numel, hp, grad_scale, zero_grad);
                else
                    flat_sgd_kernel<PT, GT, MT, HM, false><<<grid, kThreads, 0, stream>>>(
                        static_cast<PT*>(param), g, momentum_buf, static_cast<MT*>(model), numel, hp, grad_scale, zero_grad);
            };
            if (!model) {
                launch(float{}, std::false_type{});
            } else if (model_dtype == BF16) {
                launch(__nv_bfloat16{}, std::true_type{});
            } else if (model_dtype == F16) {
                launch(__half{}, std::true_type{});
            } else {
                throw std::runtime_error("bagua: flat_sgd model copy must be bf16 or f16");
            }
        });
    });
    check_launch("flat_sgd");
}

// ---- flat Adam / AdamW ----------------------------------------------------------------------------------------
template <typename PT, typename GT, typename MT, bool HAS_MODEL, bool VEC>
__global__ void __launch_bounds__(kThreads) flat_adam_kernel(PT* __restrict__ param, GT* __restrict__ grad, float* __restrict__ m1,
                                                             float* __restrict__ m2, MT* __restrict__ model, size_t n,
                                                             AdamParams hp, float grad_scale, int zero_grad) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (VEC) {
        const size_t nv = n / kVec;
        for (size_t j = tid; j < nv; j += stride) {
            const size_t i = j * kVec;
            float w[kVec], g[kVec], a[kVec], b[kVec];
            load_pack<PT>(param, i, w);
            load_pack<GT>(grad, i, g);
            load_pack<float>(m1, i, a);
            load_pack<float>(m2, i, b);
#pragma unroll
            for (int k = 0; k < kVec; ++k) adam_update(w[k], g[k], a[k], b[k], hp, grad_scale);
            store_pack<PT>(param, i, w);
            store_pack<float>(m1, i, a);
            store_pack<float>(m2, i, b);
            if (HAS_MODEL) store_pack<MT>(model, i, w);
            if (zero_grad) {
                float z[kVec] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                store_pack<GT>(grad, i, z);
            }
        }
    }
    const size_t start = VEC ? (n / kVec) * kVec : 0;
    for (size_t i = start + tid; i < n; i += stride) {
        float w = to_f32<PT>(param[i]), g = to_f32<GT>(grad[i]), a = m1[i], b = m2[i];
        adam_update(w, g, a, b, hp, grad_scale);
        param[i] = from_f32<PT>(w);
        m1[i] = a;
        m2[i] = b;
        if (HAS_MODEL) model[i] = from_f32<MT>(w);
        if (zero_grad) grad[i] = from_f32<GT>(0.f);
    }
}

void launch_flat_adam(void* param, int param_dtype, const void* grad, int grad_dtype, float* exp_avg, float* exp_avg_sq,
                      void* model, int model_dtype, size_t numel, const AdamParams& hp, float grad_scale, bool zero_grad,
                      cudaStream_t stream) {
    if (!numel) return;
    if (hp.amsgrad) throw std::runtime_error("bagua: flat_adam does not implement amsgrad");
    const bool vec = aligned16(param) && aligned16(grad) && aligned16(exp_avg) && aligned16(exp_avg_sq) && (!model || aligned16(model));
    const int grid = flat_grid(numel);
    dispatch_float(param_dtype, "optimizer kernels", [&](auto pt) {
        using PT = decltype(pt);
        dispatch_float(grad_dtype, "optimizer kernels", [&](auto gt) {
            using GT = decltype(gt);
            auto* g = const_cast<GT*>(static_cast<const GT*>(grad));
            auto launch = [&](auto mt, auto has_model) {
                using MT = decltype(mt);
                constexpr bool HM = decltype(has_model)::value;
                if (vec)
                    flat_adam_kernel<PT, GT, MT, HM, true><<<grid, kThreads, 0, stream>>>(
                        static_cast<PT*>(param), g, exp_avg, exp_avg_sq, static_cast<MT*>(model), numel, hp, grad_scale, zero_grad);
                else
                    flat_adam_kernel<PT, GT, MT, HM, false><<<grid, kThreads, 0, stream>>>(
                        static_cast<PT*>(param), g, exp_avg, exp_avg_sq, static_cast<MT*>(model), numel, hp, grad_scale, zero_grad);
            };
            if (!model) {
                launch(float{}, std::false_type{});
            } else if (model_dtype == BF16) {
                launch(__nv_bfloat16{}, std::true_type{});
            } else if (model_dtype == F16) {
                launch(__half{}, std::true_type{});
            } else {
                throw std::runtime_error("bagua: flat_adam model copy must be bf16 or f16");
            }
        });
    });
    check_launch("flat_adam");
}

// ---- multi-tensor (non-contiguous) variants -------------------------------------------------------------------
// Block b works on chunk block_to_chunk[b] of tensor block_to_tensor[b]; pointer table is [list][tensor].
template <typename T, bool HAS_MOM>
__global__ void __launch_bounds__(kThreads) multi_tensor_sgd_kernel(TensorListDesc d, SgdParams hp, float grad_scale) {
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    const T* g = reinterpret_cast<const T*>(d.ptrs[d.n_tensors + t]) + off;
    T* mo = HAS_MOM ? reinterpret_cast<T*>(d.ptrs[2 * d.n_tensors + t]) + off : nullptr;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        float w = to_f32<T>(p[i]);
        float m = (HAS_MOM && !hp.first_step) ? to_f32<T>(mo[i]) : 0.f;
        sgd_update(w, to_f32<T>(g[i]), m, hp, grad_scale);
        p[i] = from_f32<T>(w);
        if (HAS_MOM) mo[i] = from_f32<T>(m);
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) multi_tensor_adam_kernel(TensorListDesc d, AdamParams hp, float grad_scale) {
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    const T* g = reinterpret_cast<const T*>(d.ptrs[d.n_tensors + t]) + off;
    T* m1 = reinterpret_cast<T*>(d.ptrs[2 * d.n_tensors + t]) + off;
    T* m2 = reinterpret_cast<T*>(d.ptrs[3 * d.n_tensors + t]) + off;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        float w = to_f32<T>(p[i]), a = to_f32<T>(m1[i]), b = to_f32<T>(m2[i]);
        adam_update(w, to_f32<T>(g[i]), a, b, hp, grad_scale);
        p[i] = from_f32<T>(w);
        m1[i] = from_f32<T>(a);
        m2[i] = from_f32<T>(b);
    }
}

// Mixed precision: lists = [param(T), grad(T), exp_avg(f32), exp_avg_sq(f32), master(f32)] — low-precision parameters with fp32
// moments and fp32 master weights (the update happens on the master copy; the parameter receives the rounded result).
template <typename T>
__global__ void __launch_bounds__(kThreads) multi_tensor_adam_mp_kernel(TensorListDesc d, AdamParams hp, float grad_scale) {
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    const T* g = reinterpret_cast<const T*>(d.ptrs[d.n_tensors + t]) + off;
    float* m1 = reinterpret_cast<float*>(d.ptrs[2 * d.n_tensors + t]) + off;
    float* m2 = reinterpret_cast<float*>(d.ptrs[3 * d.n_tensors + t]) + off;
    float* mw = reinterpret_cast<float*>(d.ptrs[4 * d.n_tensors + t]) + off;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        float w = mw[i], a = m1[i], b = m2[i];
        adam_update(w, to_f32<T>(g[i]), a, b, hp, grad_scale);
        mw[i] = w;
        m1[i] = a;
        m2[i] = b;
        p[i] = from_f32<T>(w);
    }
}

// Mixed precision: lists = [param(T), grad(T), master(f32)(, momentum(f32))] — the SGD counterpart of the kernel above.
template <typename T, bool HAS_MOM>
__global__ void __launch_bounds__(kThreads) multi_tensor_sgd_mp_kernel(TensorListDesc d, SgdParams hp, float grad_scale) {
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    const T* g = reinterpret_cast<const T*>(d.ptrs[d.n_tensors + t]) + off;
    float* mw = reinterpret_cast<float*>(d.ptrs[2 * d.n_tensors + t]) + off;
    float* mo = HAS_MOM ? reinterpret_cast<float*>(d.ptrs[3 * d.n_tensors + t]) + off : nullptr;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        float w = mw[i];
        float m = (HAS_MOM && !hp.first_step) ? mo[i] : 0.f;
        sgd_update(w, to_f32<T>(g[i]), m, hp, grad_scale);
        mw[i] = w;
        if (HAS_MOM) mo[i] = m;
        p[i] = from_f32<T>(w);
    }
}

void launch_multi_tensor_sgd_mp(const TensorListDesc& d, int dtype, bool has_momentum, const SgdParams& hp, float grad_scale,
                                cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        if (has_momentum)
            multi_tensor_sgd_mp_kernel<T, true><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
        else
            multi_tensor_sgd_mp_kernel<T, false><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check_launch("multi_tensor_sgd_mp");
}

void launch_multi_tensor_adam_mp(const TensorListDesc& d, int dtype, const AdamParams& hp, float grad_scale, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        multi_tensor_adam_mp_kernel<T><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check_launch("multi_tensor_adam_mp");
}

void launch_multi_tensor_sgd(const TensorListDesc& d, int dtype, bool has_momentum, const SgdParams& hp, float grad_scale,
                             cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        if (has_momentum)
            multi_tensor_sgd_kernel<T, true><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
        else
            multi_tensor_sgd_kernel<T, false><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check_launch("multi_tensor_sgd");
}

void launch_multi_tensor_adam(const TensorListDesc& d, int dtype, const AdamParams& hp, float grad_scale, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        multi_tensor_adam_kernel<T><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check_launch("multi_tensor_adam");
}

// ---- LAMB: moments + per-block norms, then per-tensor trust ratio + apply ---------------------------------------
// Stage 1 leaves one fp64 {Σw², Σu²} pair per block (sums[2·block], no atomics); a block belongs to exactly one tensor, so stage 2
// gets a tensor's norms by adding its blocks' pairs in block order. Stage 2 recomputes u from the new moments and the unchanged w with
// the same lamb_direction, so no per-element buffer holds u between the launches.
// DEV_STEP (the in-bucket LAMB with loss scaling): coef addresses {coef, found_inf} and *step is the effective step count including
// this step; a skipped step returns before any write (its stale sums are not used), a taken one builds its bias corrections from t.
template <typename T, bool MIXED, bool DEV_STEP>
__global__ void __launch_bounds__(kThreads)
    multi_tensor_lamb_stage1_kernel(TensorListDesc d, LambParams hp, const float* coef, double* sums, int zero_grad, const uint32_t* step) {
    __shared__ double s_w[kThreads / 32], s_u[kThreads / 32];
    if constexpr (DEV_STEP) {
        if (coef[1] != 0.f) return;
        const uint32_t ts = *step;
        hp.bias_correction1 = bias_correction(hp.beta1, ts);
        hp.bias_correction2 = bias_correction(hp.beta2, ts);
    }
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    const T* p = reinterpret_cast<const T*>(d.ptrs[t]) + off;
    T* g = reinterpret_cast<T*>(d.ptrs[d.n_tensors + t]) + off;
    float* m1 = reinterpret_cast<float*>(d.ptrs[2 * d.n_tensors + t]) + off;
    float* m2 = reinterpret_cast<float*>(d.ptrs[3 * d.n_tensors + t]) + off;
    const float* mw = MIXED ? reinterpret_cast<const float*>(d.ptrs[4 * d.n_tensors + t]) + off : nullptr;
    const float c = coef != nullptr ? *coef : 1.f;
    double sw = 0.0, su = 0.0;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        const float w = MIXED ? mw[i] : to_f32<T>(p[i]);
        const float gg = coef != nullptr ? __fmul_rn(c, to_f32<T>(g[i])) : to_f32<T>(g[i]);
        float a = m1[i], b = m2[i];
        lamb_moments(gg, a, b, hp);
        const float u = lamb_direction(w, a, b, hp);
        m1[i] = a;
        m2[i] = b;
        if (zero_grad) g[i] = from_f32<T>(0.f);
        sw += static_cast<double>(w) * static_cast<double>(w);
        su += static_cast<double>(u) * static_cast<double>(u);
    }
    // fixed order: a shuffle tree per warp, then the warps in index order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sw += __shfl_xor_sync(0xffffffffu, sw, o);
        su += __shfl_xor_sync(0xffffffffu, su, o);
    }
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sw, s_u[threadIdx.x >> 5] = su;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (unsigned k = 0; k < blockDim.x / 32; ++k) a += s_w[k], b += s_u[k];
        sums[2 * blockIdx.x] = a;
        sums[2 * blockIdx.x + 1] = b;
    }
}

template <typename T, bool MIXED>
__global__ void __launch_bounds__(kThreads) multi_tensor_lamb_stage2_kernel(TensorListDesc d, LambParams hp, const double* sums) {
    __shared__ float s_ratio;
    const int t = d.block_to_tensor[blockIdx.x];
    const int chunk_idx = d.block_to_chunk[blockIdx.x];
    const size_t off = static_cast<size_t>(chunk_idx) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    if (threadIdx.x < 32) {  // the tensor's blocks are consecutive from blockIdx.x − chunk_idx: one warp adds their pairs in a fixed order
        const int first = blockIdx.x - chunk_idx;
        const int nb = static_cast<int>((n + d.chunk - 1) / d.chunk);
        double a = 0.0, b = 0.0;
        for (int k = threadIdx.x; k < nb; k += 32) a += sums[2 * (first + k)], b += sums[2 * (first + k) + 1];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if (threadIdx.x == 0) s_ratio = lamb_ratio(a, b);
    }
    __syncthreads();
    const float r = s_ratio;
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    const float* m1 = reinterpret_cast<const float*>(d.ptrs[2 * d.n_tensors + t]) + off;
    const float* m2 = reinterpret_cast<const float*>(d.ptrs[3 * d.n_tensors + t]) + off;
    float* mw = MIXED ? reinterpret_cast<float*>(d.ptrs[4 * d.n_tensors + t]) + off : nullptr;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        const float w = MIXED ? mw[i] : to_f32<T>(p[i]);
        const float nw = lamb_apply(w, lamb_direction(w, m1[i], m2[i], hp), r, hp);
        if (MIXED) mw[i] = nw;
        p[i] = from_f32<T>(nw);
    }
}

void launch_multi_tensor_lamb_stage1(const TensorListDesc& d, int dtype, bool mixed, const LambParams& hp, const float* coef, double* sums, bool zero_grad,
                                     cudaStream_t stream, const uint32_t* step) {
    if (d.n_blocks <= 0) return;
    if (step != nullptr && coef == nullptr) throw std::runtime_error("bagua: multi_tensor_lamb_stage1 with a device step needs {coef, found_inf}");
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        dispatch_flag(mixed, [&](auto mx) {
            dispatch_flag(step != nullptr, [&](auto dev) {
                multi_tensor_lamb_stage1_kernel<T, decltype(mx)::value, decltype(dev)::value><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, coef, sums,
                                                                                                                                 zero_grad ? 1 : 0, step);
            });
        });
    });
    check_launch("multi_tensor_lamb_stage1");
}

void launch_multi_tensor_lamb_stage2(const TensorListDesc& d, int dtype, bool mixed, const LambParams& hp, const double* sums, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        if (mixed)
            multi_tensor_lamb_stage2_kernel<T, true><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, sums);
        else
            multi_tensor_lamb_stage2_kernel<T, false><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, sums);
    });
    check_launch("multi_tensor_lamb_stage2");
}

// ---- LARS: per-block norms, then per-tensor trust + momentum + apply -------------------------------------------
// The block layout of the LAMB kernels above: stage 1 leaves one fp64 {Σw², Σg̃²} pair per block (no atomics, the gradient left in
// place for stage 2), stage 2 adds its tensor's block pairs in block order and recomputes g̃ with the same lars_grad.
// VOTE (the in-bucket LARS with loss scaling): coef addresses {coef, found_inf}; a skipped step returns before any write.
template <typename T, bool MIXED, bool VOTE>
__global__ void __launch_bounds__(kThreads) multi_tensor_lars_stage1_kernel(TensorListDesc d, const float* coef, double* sums) {
    __shared__ double s_w[kThreads / 32], s_g[kThreads / 32];
    if constexpr (VOTE) {
        if (coef[1] != 0.f) return;
    }
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    const T* p = reinterpret_cast<const T*>(d.ptrs[t]) + off;
    const T* g = reinterpret_cast<const T*>(d.ptrs[d.n_tensors + t]) + off;
    const float* mw = MIXED ? reinterpret_cast<const float*>(d.ptrs[3 * d.n_tensors + t]) + off : nullptr;
    const float c = coef != nullptr ? *coef : 1.f;
    double sw = 0.0, sg = 0.0;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        const float w = MIXED ? mw[i] : to_f32<T>(p[i]);
        const float gt = lars_grad(to_f32<T>(g[i]), c);
        sw += static_cast<double>(w) * static_cast<double>(w);
        sg += static_cast<double>(gt) * static_cast<double>(gt);
    }
    // fixed order: a shuffle tree per warp, then the warps in index order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sw += __shfl_xor_sync(0xffffffffu, sw, o);
        sg += __shfl_xor_sync(0xffffffffu, sg, o);
    }
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sw, s_g[threadIdx.x >> 5] = sg;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (unsigned k = 0; k < blockDim.x / 32; ++k) a += s_w[k], b += s_g[k];
        sums[2 * blockIdx.x] = a;
        sums[2 * blockIdx.x + 1] = b;
    }
}

template <typename T, bool MIXED>
__global__ void __launch_bounds__(kThreads)
    multi_tensor_lars_stage2_kernel(TensorListDesc d, LarsParams hp, const float* coef, const double* sums, int zero_grad) {
    __shared__ float s_trust;
    const int t = d.block_to_tensor[blockIdx.x];
    const int chunk_idx = d.block_to_chunk[blockIdx.x];
    const size_t off = static_cast<size_t>(chunk_idx) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    if (threadIdx.x < 32) {  // the tensor's blocks are consecutive from blockIdx.x − chunk_idx: one warp adds their pairs in a fixed order
        const int first = blockIdx.x - chunk_idx;
        const int nb = static_cast<int>((n + d.chunk - 1) / d.chunk);
        double a = 0.0, b = 0.0;
        for (int k = threadIdx.x; k < nb; k += 32) a += sums[2 * (first + k)], b += sums[2 * (first + k) + 1];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if (threadIdx.x == 0) s_trust = lars_trust(a, b, hp);
    }
    __syncthreads();
    const float lt = lars_step_size(s_trust, hp);
    const float c = coef != nullptr ? *coef : 1.f;
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    T* g = reinterpret_cast<T*>(d.ptrs[d.n_tensors + t]) + off;
    float* mo = reinterpret_cast<float*>(d.ptrs[2 * d.n_tensors + t]) + off;
    float* mw = MIXED ? reinterpret_cast<float*>(d.ptrs[3 * d.n_tensors + t]) + off : nullptr;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        float w = MIXED ? mw[i] : to_f32<T>(p[i]), v = mo[i];
        lars_apply(w, v, lars_grad(to_f32<T>(g[i]), c), lt, hp);
        mo[i] = v;
        if (MIXED) mw[i] = w;
        p[i] = from_f32<T>(w);
        if (zero_grad) g[i] = from_f32<T>(0.f);
    }
}

void launch_multi_tensor_lars_stage1(const TensorListDesc& d, int dtype, bool mixed, const float* coef, double* sums, cudaStream_t stream, bool vote) {
    if (d.n_blocks <= 0) return;
    if (vote && coef == nullptr) throw std::runtime_error("bagua: multi_tensor_lars_stage1 with a vote needs {coef, found_inf}");
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        dispatch_flag(mixed, [&](auto mx) {
            dispatch_flag(vote, [&](auto vt) {
                multi_tensor_lars_stage1_kernel<T, decltype(mx)::value, decltype(vt)::value><<<d.n_blocks, kThreads, 0, stream>>>(d, coef, sums);
            });
        });
    });
    check_launch("multi_tensor_lars_stage1");
}

void launch_multi_tensor_lars_stage2(const TensorListDesc& d, int dtype, bool mixed, const LarsParams& hp, const float* coef, const double* sums, bool zero_grad,
                                     cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        dispatch_flag(mixed, [&](auto mx) {
            multi_tensor_lars_stage2_kernel<T, decltype(mx)::value><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, coef, sums, zero_grad ? 1 : 0);
        });
    });
    check_launch("multi_tensor_lars_stage2");
}

// ---- Lion: one pass, the gradient cleared on the way ---------------------------------------------------------------------
// lists = [param(T), grad(T), (master(f32) when MIXED,) exp_avg(f32)]; the update is lion.cuh's, with coef 1.
template <typename T, bool MIXED>
__global__ void __launch_bounds__(kThreads) multi_tensor_lion_kernel(TensorListDesc d, LionParams hp, int zero_grad) {
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    T* p = reinterpret_cast<T*>(d.ptrs[t]) + off;
    T* g = reinterpret_cast<T*>(d.ptrs[d.n_tensors + t]) + off;
    float* mw = MIXED ? reinterpret_cast<float*>(d.ptrs[2 * d.n_tensors + t]) + off : nullptr;
    float* ea = reinterpret_cast<float*>(d.ptrs[(MIXED ? 3 : 2) * d.n_tensors + t]) + off;
    for (size_t i = threadIdx.x; i < len; i += blockDim.x) {
        float w = MIXED ? mw[i] : to_f32<T>(p[i]), m = ea[i];
        lion_apply(w, m, lion_grad(to_f32<T>(g[i]), 1.f), hp);
        ea[i] = m;
        if (MIXED) mw[i] = w;
        p[i] = from_f32<T>(w);
        if (zero_grad) g[i] = from_f32<T>(0.f);
    }
}

void launch_multi_tensor_lion(const TensorListDesc& d, int dtype, bool mixed, const LionParams& hp, bool zero_grad, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, "optimizer kernels", [&](auto tag) {
        using T = decltype(tag);
        dispatch_flag(mixed, [&](auto mx) {
            multi_tensor_lion_kernel<T, decltype(mx)::value><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, zero_grad ? 1 : 0);
        });
    });
    check_launch("multi_tensor_lion");
}

// ---- exponential moving average of fp32 weights ---------------------------------------------------------------------
// lists = [source(f32), ema(f32)]: e ← e + w·(m − e) with three separately rounded operations (the intrinsics keep the compiler from
// contracting the product and the sum into an FMA), so a host fp32 emulation reproduces every bit. This is torch's lerp for w < 0.5.
// A chunk takes 16-byte accesses when both of its pointers are 16-byte aligned (chunk offsets are multiples of 65536 elements, so
// that is a property of the tensors' base addresses) and scalar ones otherwise: the lists may hold arbitrary views. `vote`
// (nullable) is the loss-scaled step's found_inf word: when it is set the kernel writes nothing.
__device__ __forceinline__ float ema_step(float e, float m, float w) { return __fadd_rn(e, __fmul_rn(w, __fsub_rn(m, e))); }

__global__ void __launch_bounds__(kThreads) multi_tensor_ema_kernel(TensorListDesc d, float w, const float* vote) {
    if (vote != nullptr && *vote != 0.f) return;
    const int t = d.block_to_tensor[blockIdx.x];
    const size_t off = static_cast<size_t>(d.block_to_chunk[blockIdx.x]) * d.chunk;
    const size_t n = static_cast<size_t>(d.sizes[t]);
    const size_t len = (n - off) < static_cast<size_t>(d.chunk) ? (n - off) : static_cast<size_t>(d.chunk);
    const float* src = reinterpret_cast<const float*>(d.ptrs[t]) + off;
    float* ema = reinterpret_cast<float*>(d.ptrs[d.n_tensors + t]) + off;
    size_t done = 0;
    if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(ema)) & 15u) == 0) {
        const size_t nv = len / 4;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* e4 = reinterpret_cast<float4*>(ema);
        for (size_t i = threadIdx.x; i < nv; i += blockDim.x) {
            const float4 m = s4[i];
            float4 e = e4[i];
            e.x = ema_step(e.x, m.x, w);
            e.y = ema_step(e.y, m.y, w);
            e.z = ema_step(e.z, m.z, w);
            e.w = ema_step(e.w, m.w, w);
            e4[i] = e;
        }
        done = nv * 4;
    }
    for (size_t i = done + threadIdx.x; i < len; i += blockDim.x) ema[i] = ema_step(ema[i], src[i], w);
}

void launch_multi_tensor_ema(const TensorListDesc& d, float weight, const float* vote, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    multi_tensor_ema_kernel<<<d.n_blocks, kThreads, 0, stream>>>(d, weight, vote);
    check_launch("multi_tensor_ema");
}

// ---- QAdam momentum pre-step -------------------------------------------------------------------------------------
template <typename GT>
__global__ void __launch_bounds__(kThreads) qadam_momentum_kernel(float* __restrict__ m, const GT* __restrict__ g, size_t n, float beta1) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        m[i] = beta1 * m[i] + (1.f - beta1) * to_f32<GT>(g[i]);
}

void launch_qadam_momentum(float* exp_avg, const void* grad, int grad_dtype, size_t numel, float beta1, cudaStream_t stream) {
    if (!numel) return;
    dispatch_float(grad_dtype, "optimizer kernels", [&](auto tag) {
        using GT = decltype(tag);
        qadam_momentum_kernel<GT><<<flat_grid(numel), kThreads, 0, stream>>>(exp_avg, static_cast<const GT*>(grad), numel, beta1);
    });
    check_launch("qadam_momentum");
}

}  // namespace bagua
