// MinMaxUInt8 quantisation math shared by the single-GPU kernels and the fused ByteGrad / ring kernels.
// Bit-compatible with the reference's wire format and rounding (kernels/bagua_kernels.cu:404-501; python
// oracle tests/internal/compressor.py:4-33): scale = 255/(max-min+1e-7), upper = rint(max*scale),
// lower = upper-255, q = min(rint(x*scale), upper) - lower, x' = (q + lower)/scale.
#pragma once
#ifndef BAGUA_QUANT_HOST_EMULATION
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#endif

#include <cstdint>

namespace bagua {
namespace dev {

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// Order-preserving float <-> uint encoding so min/max can use integer atomics.
__device__ __forceinline__ uint32_t f32_to_ordered(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_f32(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
constexpr uint32_t kOrderedMinInit = 0xffffffffu;  // identity for atomicMin
constexpr uint32_t kOrderedMaxInit = 0u;           // identity for atomicMax

struct QuantParams {
    float scale;
    float lower;
    float upper;
    float inv_scale;   // correctly rounded 1/scale, computed once per chunk
};

__device__ __forceinline__ QuantParams make_quant(float mn, float mx) {
    QuantParams q;
    q.scale = __fdiv_rn(255.0f, __fadd_rn(__fsub_rn(mx, mn), 1e-7f));
    q.upper = rintf(__fmul_rn(mx, q.scale));
    q.lower = __fsub_rn(q.upper, 255.0f);
    q.inv_scale = __frcp_rn(q.scale);
    return q;
}
// float → uint8: on the device this is one saturating convert (an out-of-range value — the −1 that round-half-even can produce
// at the lower end — becomes 0); the host emulation has to spell the saturation out because the C++ cast is undefined there.
__device__ __forceinline__ uint8_t f32_to_u8_sat(float v) {
#ifdef BAGUA_QUANT_HOST_EMULATION
    return static_cast<uint8_t>(v < 0.f ? 0.f : (v > 255.f ? 255.f : v));
#else
    return static_cast<uint8_t>(v);
#endif
}
__device__ __forceinline__ uint8_t quantize(float x, const QuantParams& q) {
    float level = fminf(rintf(__fmul_rn(x, q.scale)), q.upper);
    return f32_to_u8_sat(__fsub_rn(level, q.lower));
}
// x' = (q + lower) / scale, evaluated as a multiplication by the chunk's reciprocal: an IEEE fp32 division is ~10 issue slots per
// ELEMENT (MUFU.RCP + Newton steps + FCHK + slow-path call) and made up 39 % of the SASS of bytegrad_kernel<bf16, 8>, a kernel that Nsight
// Compute showed to be instruction-issue bound; the product differs from the quotient by at most one fp32 ulp, far below
// a quantisation level, and every rank decodes with the same code, so replicas stay bit-identical. -DBAGUA_DEQUANT_IEEE_DIV restores the
// division (bit-exact with the reference's formula, bagua_kernels.cu:456-501).
__device__ __forceinline__ float dequantize(uint8_t v, const QuantParams& q) {
#ifdef BAGUA_DEQUANT_IEEE_DIV
    return __fdiv_rn(__fadd_rn(static_cast<float>(v), q.lower), q.scale);
#else
    return __fmul_rn(__fadd_rn(static_cast<float>(v), q.lower), q.inv_scale);
#endif
}

#ifndef BAGUA_QUANT_HOST_EMULATION   // tests/cpp/quant_emulation.cpp compiles the scalar math above for the host
// Block-wide min/max of per-thread partials; result valid in thread 0.
__device__ __forceinline__ void block_minmax(float& mn, float& mx) {
    __shared__ float s_mn[32], s_mx[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();  // protect s_mn/s_mx reuse across calls
    if (lane == 0) s_mn[warp] = mn, s_mx[warp] = mx;
    __syncthreads();
    if (warp == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        mn = lane < nw ? s_mn[lane] : INFINITY;
        mx = lane < nw ? s_mx[lane] : -INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
    }
}

#endif  // BAGUA_QUANT_HOST_EMULATION

}  // namespace dev
}  // namespace bagua
