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

#include "kernels.h"
#include "quant.cuh"

namespace bagua {
using namespace dev;

namespace {
constexpr int kThreads = 512;
constexpr int kVec = 8;  // elements per thread per iteration

void check(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of ") + what + " failed: " + cudaGetErrorString(e));
    count_launch();
}

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

template <typename F>
void dispatch_float(int dtype, F&& f) {
    switch (dtype) {
        case F32: f(float{}); break;
        case F16: f(__half{}); break;
        case BF16: f(__nv_bfloat16{}); break;
        default: throw std::runtime_error("bagua: optimizer kernels need f32/f16/bf16, got dtype code " + std::to_string(dtype));
    }
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
    dispatch_float(param_dtype, [&](auto pt) {
        using PT = decltype(pt);
        dispatch_float(grad_dtype, [&](auto gt) {
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
    check("flat_sgd");
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
    dispatch_float(param_dtype, [&](auto pt) {
        using PT = decltype(pt);
        dispatch_float(grad_dtype, [&](auto gt) {
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
    check("flat_adam");
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

void launch_multi_tensor_adam_mp(const TensorListDesc& d, int dtype, const AdamParams& hp, float grad_scale, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        multi_tensor_adam_mp_kernel<T><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check("multi_tensor_adam_mp");
}

void launch_multi_tensor_sgd(const TensorListDesc& d, int dtype, bool has_momentum, const SgdParams& hp, float grad_scale,
                             cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        if (has_momentum)
            multi_tensor_sgd_kernel<T, true><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
        else
            multi_tensor_sgd_kernel<T, false><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check("multi_tensor_sgd");
}

void launch_multi_tensor_adam(const TensorListDesc& d, int dtype, const AdamParams& hp, float grad_scale, cudaStream_t stream) {
    if (d.n_blocks <= 0) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        multi_tensor_adam_kernel<T><<<d.n_blocks, kThreads, 0, stream>>>(d, hp, grad_scale);
    });
    check("multi_tensor_adam");
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
    dispatch_float(grad_dtype, [&](auto tag) {
        using GT = decltype(tag);
        qadam_momentum_kernel<GT><<<flat_grid(numel), kThreads, 0, stream>>>(exp_avg, static_cast<const GT*>(grad), numel, beta1);
    });
    check("qadam_momentum");
}

}  // namespace bagua
