// The LAMB update rule, shared by the multi-tensor FusedLAMB kernels (multi_tensor.cu) and the in-bucket sharded kernels
// (peer_kernels.cu). Every rounding is explicit (no FMA contraction), so the update direction u that feeds Σu² in one kernel and
// the u that a later kernel applies are the same bits, whichever kernel computes them.
//
//   m ← β1·m + (1−β1)·g        v ← β2·v + (1−β2)·g²
//   u = (m / bc1) / (sqrt(v) / sqrt(bc2) + eps) + wd·w      (evaluated as (m·(1/bc1)) / (sqrt(v)·rsqrt(bc2) + eps) + wd·w)
//   r = ‖w‖ / ‖u‖ over the whole parameter (fp64 sums, one rounding to fp32) when wd ≠ 0 and both norms > 0, else 1
//   w ← w − lr·r·u
#pragma once
#include "kernels.h"

namespace bagua {
namespace dev {

__device__ __forceinline__ void lamb_moments(float g, float& m, float& v, const LambParams& hp) {
    m = __fadd_rn(__fmul_rn(hp.beta1, m), __fmul_rn(1.f - hp.beta1, g));
    v = __fadd_rn(__fmul_rn(hp.beta2, v), __fmul_rn(__fmul_rn(1.f - hp.beta2, g), g));
}

// One division per element: the bias corrections enter as their correctly rounded reciprocals (loop-invariant).
__device__ __forceinline__ float lamb_direction(float w, float m, float v, const LambParams& hp) {
    const float denom = __fadd_rn(__fmul_rn(__fsqrt_rn(v), __frsqrt_rn(hp.bias_correction2)), hp.eps);
    return __fadd_rn(__fdiv_rn(__fmul_rn(m, __frcp_rn(hp.bias_correction1)), denom), __fmul_rn(hp.weight_decay, w));
}

// The trust ratio from a parameter's global Σw² and Σu². Computed for every parameter; lamb_apply ignores it without weight decay.
__device__ __forceinline__ float lamb_ratio(double w2, double u2) {
    return (w2 > 0.0 && u2 > 0.0) ? static_cast<float>(sqrt(w2) / sqrt(u2)) : 1.f;
}

__device__ __forceinline__ float lamb_apply(float w, float u, float ratio, const LambParams& hp) {
    const float r = hp.weight_decay != 0.f ? ratio : 1.f;
    return __fsub_rn(w, __fmul_rn(__fmul_rn(hp.lr, r), u));
}

}  // namespace dev
}  // namespace bagua
