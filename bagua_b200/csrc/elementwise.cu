// Single-GPU bandwidth kernels: MinMaxUInt8 (de)compression, chunk reduce, async-average apply, axpby, cast.
// Counterparts of the reference's scalar kernels (kernels/bagua_kernels.cu:196-690) written for HBM3:
// 16-byte accesses where alignment allows, grid sized to the 132 SMs of an H100, min/max fused into one pass
// (the reference does 2 cub reductions per chunk from a host loop, bagua_kernels.cu:540-546).
#include <stdexcept>
#include <string>

#include "kernels.h"
#include "quant.cuh"

namespace bagua {
using namespace dev;

namespace {
constexpr int kThreads = 512;
inline int grid_for(size_t work_items, int per_thread = 4, int max_blocks = 132 * 8) {
    size_t b = (work_items + static_cast<size_t>(kThreads) * per_thread - 1) / (static_cast<size_t>(kThreads) * per_thread);
    if (b < 1) b = 1;
    if (b > static_cast<size_t>(max_blocks)) b = max_blocks;
    return static_cast<int>(b);
}
void check(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of ") + what + " failed: " + cudaGetErrorString(e));
    count_launch();
}
template <typename F>
void dispatch_float(int dtype, F&& f) {
    switch (dtype) {
        case F32: f(float{}); break;
        case F16: f(__half{}); break;
        case BF16: f(__nv_bfloat16{}); break;
        default: throw std::runtime_error("bagua: kernel needs f32/f16/bf16, got dtype code " + std::to_string(dtype));
    }
}
}  // namespace

// ---- min/max per chunk ---------------------------------------------------------------------------------
__global__ void minmax_init_kernel(uint32_t* mm, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) mm[i] = (i & 1) ? kOrderedMaxInit : kOrderedMinInit;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) chunk_minmax_kernel(const T* __restrict__ in, size_t chunk, int first_chunk,
                                                                uint32_t* __restrict__ mm) {
    const int c = first_chunk + blockIdx.y;
    const T* p = in + static_cast<size_t>(c) * chunk;
    float mn = INFINITY, mx = -INFINITY;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < chunk; i += stride) {
        float v = to_f32<T>(p[i]);
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
    block_minmax(mn, mx);
    if (threadIdx.x == 0) {
        atomicMin(&mm[2 * c], f32_to_ordered(mn));
        atomicMax(&mm[2 * c + 1], f32_to_ordered(mx));
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) chunk_quantize_kernel(const T* __restrict__ in, size_t chunk, size_t chunk_bytes,
                                                                  int first_chunk, const uint32_t* __restrict__ mm,
                                                                  uint8_t* __restrict__ out) {
    const int c = first_chunk + blockIdx.y;
    const float mn = ordered_to_f32(mm[2 * c]);
    const float mx = ordered_to_f32(mm[2 * c + 1]);
    const QuantParams q = make_quant(mn, mx);
    const T* p = in + static_cast<size_t>(c) * chunk;
    uint8_t* o = out + static_cast<size_t>(c) * chunk_bytes;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < chunk; i += stride)
        o[32 + i] = quantize(to_f32<T>(p[i]), q);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        T* hdr = reinterpret_cast<T*>(o);
        hdr[0] = from_f32<T>(mn);
        hdr[1] = from_f32<T>(mx);
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) chunk_dequantize_kernel(const uint8_t* __restrict__ in, size_t chunk,
                                                                    size_t chunk_bytes, T* __restrict__ out) {
    const int c = blockIdx.y;
    const uint8_t* src = in + static_cast<size_t>(c) * chunk_bytes;
    const T* hdr = reinterpret_cast<const T*>(src);
    const QuantParams q = make_quant(to_f32<T>(hdr[0]), to_f32<T>(hdr[1]));
    T* o = out + static_cast<size_t>(c) * chunk;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < chunk; i += stride)
        o[i] = from_f32<T>(dequantize(src[32 + i], q));
}

void launch_minmax_uint8_compress(const void* in, size_t numel, int dtype, int n_chunks, int target_chunk, uint8_t* out,
                                  float* minmax_scratch, cudaStream_t stream) {
    if (n_chunks <= 0 || numel % n_chunks) throw std::runtime_error("bagua: compress needs numel divisible by n_chunks");
    const size_t chunk = numel / n_chunks;
    if (chunk == 0) return;
    const size_t chunk_bytes = minmax_uint8_chunk_bytes(chunk);
    const int first = target_chunk < 0 ? 0 : target_chunk;
    const int count = target_chunk < 0 ? n_chunks : 1;
    auto* mm = reinterpret_cast<uint32_t*>(minmax_scratch);
    minmax_init_kernel<<<(2 * n_chunks + 255) / 256, 256, 0, stream>>>(mm, 2 * n_chunks);
    dim3 grid(grid_for(chunk, 8, 132 * 4 / (count > 4 ? 4 : 1)), count);
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        chunk_minmax_kernel<T><<<grid, kThreads, 0, stream>>>(static_cast<const T*>(in), chunk, first, mm);
        chunk_quantize_kernel<T><<<grid, kThreads, 0, stream>>>(static_cast<const T*>(in), chunk, chunk_bytes, first, mm, out);
    });
    check("minmax_uint8_compress");
    count_launch(2);  // init + min/max + quantise = 3 launches
}

void launch_minmax_uint8_decompress(const uint8_t* in, size_t numel, int dtype, int n_chunks, void* out, cudaStream_t stream) {
    if (n_chunks <= 0 || numel % n_chunks) throw std::runtime_error("bagua: decompress needs numel divisible by n_chunks");
    const size_t chunk = numel / n_chunks;
    if (chunk == 0) return;
    dim3 grid(grid_for(chunk, 8, 132 * 4 / (n_chunks > 4 ? 4 : 1)), n_chunks);
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        chunk_dequantize_kernel<T><<<grid, kThreads, 0, stream>>>(in, chunk, minmax_uint8_chunk_bytes(chunk), static_cast<T*>(out));
    });
    check("minmax_uint8_decompress");
}

// ---- element-wise family ---------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) async_apply_kernel(T* __restrict__ w, const T* __restrict__ red,
                                                               const T* __restrict__ snap, size_t n, float inv_p) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        w[i] = from_f32<T>(to_f32<T>(w[i]) + (to_f32<T>(red[i]) * inv_p - to_f32<T>(snap[i])));
}

void launch_async_apply(void* w, const void* red, const void* snap, size_t numel, int dtype, float inv_p, cudaStream_t stream) {
    if (!numel) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        async_apply_kernel<T><<<grid_for(numel), kThreads, 0, stream>>>(static_cast<T*>(w), static_cast<const T*>(red),
                                                                       static_cast<const T*>(snap), numel, inv_p);
    });
    check("async_apply");
}

template <typename T>
__global__ void __launch_bounds__(kThreads) reduce_chunks_kernel(T* __restrict__ data, size_t chunk, int n_chunks, int target,
                                                                 float scale) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < chunk; i += stride) {
        float acc = 0.f;
        for (int c = 0; c < n_chunks; ++c) acc += to_f32<T>(data[static_cast<size_t>(c) * chunk + i]);
        data[static_cast<size_t>(target) * chunk + i] = from_f32<T>(acc * scale);
    }
}

void launch_reduce_chunks(void* data, size_t chunk_elems, int n_chunks, int target_chunk, int dtype, bool average,
                          cudaStream_t stream) {
    if (!chunk_elems) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        reduce_chunks_kernel<T><<<grid_for(chunk_elems), kThreads, 0, stream>>>(static_cast<T*>(data), chunk_elems, n_chunks,
                                                                                target_chunk, average ? 1.0f / n_chunks : 1.0f);
    });
    check("reduce_chunks");
}

template <typename T>
__global__ void __launch_bounds__(kThreads) axpby_kernel(T* __restrict__ x, const T* __restrict__ y, size_t n, float a, float b) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        x[i] = from_f32<T>(a * to_f32<T>(x[i]) + b * to_f32<T>(y[i]));
}

void launch_axpby(void* x, const void* y, size_t numel, int dtype, float a, float b, cudaStream_t stream) {
    if (!numel) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        axpby_kernel<T><<<grid_for(numel), kThreads, 0, stream>>>(static_cast<T*>(x), static_cast<const T*>(y), numel, a, b);
    });
    check("axpby");
}

template <typename T>
__global__ void __launch_bounds__(kThreads) scale_kernel(T* __restrict__ x, size_t n, float a) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        x[i] = from_f32<T>(a * to_f32<T>(x[i]));
}

void launch_scale(void* x, size_t numel, int dtype, float a, cudaStream_t stream) {
    if (!numel) return;
    dispatch_float(dtype, [&](auto tag) {
        using T = decltype(tag);
        scale_kernel<T><<<grid_for(numel), kThreads, 0, stream>>>(static_cast<T*>(x), numel, a);
    });
    check("scale");
}

template <typename TI, typename TO>
__global__ void __launch_bounds__(kThreads) cast_kernel(const TI* __restrict__ in, TO* __restrict__ out, size_t n) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = from_f32<TO>(to_f32<TI>(in[i]));
}

void launch_cast(const void* in, int in_dtype, void* out, int out_dtype, size_t numel, cudaStream_t stream) {
    if (!numel) return;
    dispatch_float(in_dtype, [&](auto ti) {
        using TI = decltype(ti);
        dispatch_float(out_dtype, [&](auto to) {
            using TO = decltype(to);
            cast_kernel<TI, TO><<<grid_for(numel), kThreads, 0, stream>>>(static_cast<const TI*>(in), static_cast<TO*>(out), numel);
        });
    });
    check("cast");
}

}  // namespace bagua
