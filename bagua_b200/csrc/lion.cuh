// The Lion update rule (Chen et al. 2023, "Symbolic Discovery of Optimization Algorithms", Algorithm 2), shared by the multi-tensor
// FusedLion kernel (multi_tensor.cu) and the in-bucket sharded kernels (peer_kernels.cu), so both paths give the same bits. Every
// product and sum is rounded on its own (no FMA contraction): a host fp32 replay made of separate * and + reproduces it exactly.
//
//   g = coef·x                    x: the reduced gradient or the fp32 gradient shard; coef: 1/N, the exchange's coefficient, or 1
//   u = b1·m + c1·g
//   w ← w·d − lr·sign(u)          decoupled weight decay (d = 1 − lr·wd) before the sign step
//   m ← b2·m + c2·g
//
// sign(u) is +1 / −1, +0 for ±0 and NaN for NaN: a NaN gradient element makes its weight NaN instead of a silent no-op.
#pragma once
#include "kernels.h"

namespace bagua {
namespace dev {

__device__ __forceinline__ float lion_grad(float x, float coef) { return __fmul_rn(x, coef); }

__device__ __forceinline__ float lion_sign(float u) { return u > 0.f ? 1.f : (u < 0.f ? -1.f : (u == u ? 0.f : u)); }

// One element: w and m in place, g = lion_grad(x, coef).
__device__ __forceinline__ void lion_apply(float& w, float& m, float g, const LionParams& hp) {
    const float u = __fadd_rn(__fmul_rn(hp.b1, m), __fmul_rn(hp.c1, g));
    w = __fsub_rn(__fmul_rn(w, hp.d), __fmul_rn(hp.lr, lion_sign(u)));
    m = __fadd_rn(__fmul_rn(hp.b2, m), __fmul_rn(hp.c2, g));
}

}  // namespace dev
}  // namespace bagua
