// The LARS update rule (You et al. 2017; the MLPerf ResNet-50 form), shared by the multi-tensor FusedLARS kernels (multi_tensor.cu)
// and the in-bucket sharded kernels (peer_kernels.cu). Every rounding is explicit (no FMA contraction), so the g̃ that feeds Σg̃² in
// one kernel and the g̃ that a later kernel applies are the same bits, whichever kernel computes them.
//
//   g̃ = coef·g                               coef: the clip / unscale coefficient of the norm exchange, 1 without one
//   W = Σw², G = Σg̃² over the whole parameter (fp64)
//   trust = eta·√W / (√G + wd·√W)             in double, rounded to fp32 once, when wd ≠ 0 and W > 0 and G > 0;
//           NaN when W or G is NaN;            1 otherwise (a weight_decay = 0 group gets plain momentum SGD)
//   v ← μ·v + (lr·trust)·(g̃ + wd·w)           the momentum buffer holds the lr-scaled step
//   w ← w − v
#pragma once
#include "kernels.h"

namespace bagua {
namespace dev {

__device__ __forceinline__ float lars_grad(float g, float coef) { return __fmul_rn(coef, g); }

// Taken once per parameter (per segment change in the sharded kernel), never per element.
__device__ __forceinline__ float lars_trust(double w2, double g2, const LarsParams& hp) {
    if (isnan(w2) || isnan(g2)) return __int_as_float(0x7fc00000);
    if (hp.weight_decay == 0.f || !(w2 > 0.0) || !(g2 > 0.0)) return 1.f;
    const double sw = __dsqrt_rn(w2);
    const double den = __dadd_rn(__dsqrt_rn(g2), __dmul_rn(static_cast<double>(hp.weight_decay), sw));
    return static_cast<float>(__ddiv_rn(__dmul_rn(static_cast<double>(hp.trust_coefficient), sw), den));
}

// lr·trust, the step size of every element of the parameter.
__device__ __forceinline__ float lars_step_size(float trust, const LarsParams& hp) { return __fmul_rn(hp.lr, trust); }

// One element: v and w in place, gt = lars_grad(g, coef), lt = lars_step_size(trust, hp).
__device__ __forceinline__ void lars_apply(float& w, float& v, float gt, float lt, const LarsParams& hp) {
    const float d = __fadd_rn(gt, __fmul_rn(hp.weight_decay, w));
    v = __fadd_rn(__fmul_rn(hp.momentum, v), __fmul_rn(lt, d));
    w = __fsub_rn(w, v);
}

}  // namespace dev
}  // namespace bagua
