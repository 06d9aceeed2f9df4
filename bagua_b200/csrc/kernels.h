// Host-callable launchers of every CUDA kernel in bagua_b200 (implemented in *.cu, sm_90a).
#pragma once
#include <cuda_runtime.h>

#include <cmath>
#include <cstddef>
#include <cstdint>
#include <tuple>
#include <type_traits>

#include "common.h"

namespace bagua {

enum AllReduceVariant : int { AR_ONE_SHOT = 0, AR_TWO_SHOT = 1, AR_MULTIMEM = 2 };

struct SgdParams {
    float lr;
    float momentum;
    float dampening;
    float weight_decay;
    int nesterov;
    int first_step;
};

struct AdamParams {
    float lr;
    float beta1;
    float beta2;
    float eps;
    float weight_decay;
    float bias_correction1;  // 1 - beta1^t
    float bias_correction2;  // 1 - beta2^t
    int adamw;               // decoupled weight decay
    int amsgrad;             // unsupported (kept for ABI stability)
};

// LAMB (You et al. 2019) with apex FusedLAMB's defaults: bias correction, decoupled weight decay inside the update direction, the
// trust ratio ‖w‖/‖u‖ applied only where weight_decay != 0 (see lamb.cuh).
struct LambParams {
    float lr;
    float beta1;
    float beta2;
    float eps;
    float weight_decay;
    float bias_correction1;  // 1 - beta1^t
    float bias_correction2;  // 1 - beta2^t
};

// LARS (You et al. 2017, the MLPerf ResNet-50 form): trust = trust_coefficient·‖w‖/(‖g̃‖ + wd·‖w‖) per parameter where
// weight_decay != 0, momentum buffer v ← μ·v + lr·trust·(g̃ + wd·w), w ← w − v (see lars.cuh). No step-dependent field.
struct LarsParams {
    float lr;
    float momentum;
    float weight_decay;
    float trust_coefficient;
};

// Lion (Chen et al. 2023, Algorithm 2) as fp32 constants, each worked out in double from the group's hyper-parameters and rounded
// once (lion_params): b1 = β1, c1 = 1 − β1, b2 = β2, c2 = 1 − β2, d = 1 − lr·wd (see lion.cuh). No step-dependent field.
struct LionParams {
    float lr;
    float b1;
    float c1;
    float b2;
    float c2;
    float d;
};

inline LionParams lion_params(double lr, double beta1, double beta2, double weight_decay) {
    return LionParams{static_cast<float>(lr), static_cast<float>(beta1), static_cast<float>(1.0 - beta1), static_cast<float>(beta2),
                      static_cast<float>(1.0 - beta2), static_cast<float>(1.0 - lr * weight_decay)};
}

// 1 - beta^step of the in-bucket Adam and LAMB ops and of FusedLAMB: in double, rounded once. Also callable from device code: the
// kernels that take the step count from device memory (loss scaling) build their bias corrections with it.
#ifdef __CUDACC__
__host__ __device__
#endif
inline float bias_correction(float beta, uint64_t step) {
    return static_cast<float>(1.0 - pow(static_cast<double>(beta), static_cast<double>(step)));
}

inline AdamParams adam_params(float lr, float beta1, float beta2, float eps, float weight_decay, bool adamw, uint64_t step) {
    return AdamParams{lr, beta1, beta2, eps, weight_decay, bias_correction(beta1, step), bias_correction(beta2, step), adamw ? 1 : 0, 0};
}

inline LambParams lamb_params(float lr, float beta1, float beta2, float eps, float weight_decay, uint64_t step) {
    return LambParams{lr, beta1, beta2, eps, weight_decay, bias_correction(beta1, step), bias_correction(beta2, step)};
}

// ---- in-bucket optimizer rules (peer_kernels.cu) ---------------------------------------------------------------
// What an in-bucket optimizer kernel receives of its rule, by value: the fp32 state of the owned shard (shard-local, like the master)
// and, as an argument of its own, the rule's Params. fields() lists the fields in order, kFused / kShard name the rule's fused and
// phase-B kernels in messages and op kinds.
struct SgdRule {
    static constexpr const char* kFused = "allreduce_sgd";
    static constexpr const char* kShard = "shard_sgd";
    using Params = SgdParams;
    float* master;
    float* momentum;
    auto fields() const { return std::tuple(master, momentum); }
};
// Params carry the bias corrections of THIS step
struct AdamRule {
    static constexpr const char* kFused = "allreduce_adam";
    static constexpr const char* kShard = "shard_adam";
    using Params = AdamParams;
    float* master;
    float* exp_avg;
    float* exp_avg_sq;
    auto fields() const { return std::tuple(master, exp_avg, exp_avg_sq); }
};
// g = fl(x·coef) with x the reduced gradient (coef = scale) or the fp32 gradient shard (see lion.cuh)
struct LionRule {
    static constexpr const char* kFused = "allreduce_lion";
    static constexpr const char* kShard = "shard_lion";
    using Params = LionParams;
    float* master;
    float* exp_avg;
    auto fields() const { return std::tuple(master, exp_avg); }
};
// Phase B only: w ← w − lr·r·u on the owned slice, u recomputed from the stage-1 moments, r = ratio[segs[3s+2]] for the elements
// [segs[3s], segs[3s+1]) of the shard (1 elsewhere, and everywhere when weight_decay == 0).
struct LambRule {
    static constexpr const char* kShard = "shard_lamb";
    using Params = LambParams;
    float* master;
    const float* exp_avg;
    const float* exp_avg_sq;
    const int32_t* segs;
    int nsegs;
    const float* ratio;
    auto fields() const { return std::tuple(master, exp_avg, exp_avg_sq, segs, nsegs, ratio); }
};
// Phase B only: momentum and update of the owned slice with trust = lars_trust(sums of segs[3s+2]) for the elements [segs[3s],
// segs[3s+1]) (1 in the gaps), g̃ = shard·*coef (coef nullable = 1).
struct LarsRule {
    static constexpr const char* kShard = "shard_lars";
    using Params = LarsParams;
    float* master;
    float* momentum;
    const int32_t* segs;
    int nsegs;
    const double* sums;
    auto fields() const { return std::tuple(master, momentum, segs, nsegs, sums); }
};

// ---- peer kernels (peer_kernels.cu) ------------------------------------------------------------------------
void launch_allreduce(const PeerCtx& ctx, const PeerBuf& src, const PeerBuf& dst, size_t src_off, size_t dst_off, size_t bytes,
                      int dtype, float scale, int variant, int nblocks, int nthreads, cudaStream_t stream);
void launch_allreduce_oneshot(const PeerCtx& ctx, const PeerBuf& staging, size_t staging_off, size_t slot_bytes, const void* in, void* out,
                              size_t bytes, int dtype, float scale, int nblocks, int nthreads, cudaStream_t stream, uint32_t call_parity);
// Halves of the two-shot schedule (hierarchical all-reduce): in-place reduce of slice `rank` over the group (scaled), and
// publication of slice `rank` to every peer. Slices are ceil(vecs / world) 16-byte vectors.
void launch_reduce_scatter(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, float scale, bool use_multimem, int nblocks,
                           int nthreads, cudaStream_t stream);
void launch_all_gather(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, bool use_multimem, int nblocks, int nthreads,
                       cudaStream_t stream);
// reduce-scatter(grads) → the rule on the owned shard (fp32 master + state sharded world ways) → all-gather of the weights, and the
// gradient bucket cleared when zero_grads; g = red·scale. Instantiated for SgdRule, AdamRule and LionRule.
template <class Rule>
void launch_fused_update(const PeerCtx& ctx, const PeerBuf& grads, const PeerBuf& weights, size_t g_off, size_t w_off, size_t bytes, int dtype,
                         const Rule& rule, const typename Rule::Params& hp, float scale, bool zero_grads, bool use_multimem, int nblocks, int nthreads,
                         cudaStream_t stream);
// Global-norm clipping of the in-bucket optimizers (see shard_grad_kernel): phase A reduce-scatters a bucket into the fp32 gradient
// `shard` of the owned slice (scaled) and leaves one fp64 Σx² per CTA in partials[block]; grad_norm sums partials[0..nslots) and
// *extra (nullable), exchanges the per-rank sums through the symmetric `box` (2·kMaxPeers doubles at box_off) and writes
// out = {total, coef}; phase B applies the rule to the shard scaled by *coef and all-gathers the weights. With `accumulate` phase A
// adds the scaled reduction into the shard (gradient accumulation) and Σx² is the accumulated shard's; preload_shard_grad_accum
// loads that instantiation for one dtype / world / flavour.
void launch_shard_grad(const PeerCtx& ctx, const PeerBuf& grads, size_t g_off, size_t bytes, int dtype, float* shard, double* partials, float scale,
                       bool zero_grads, bool use_multimem, int nblocks, int nthreads, cudaStream_t stream, bool accumulate = false);
void preload_shard_grad_accum(int dtype, int world, bool use_multimem);
void launch_grad_norm(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const double* partials, int nslots, const double* extra, float max_norm,
                      uint32_t parity, float* out, cudaStream_t stream);
//
// Loss scaling: loss_scale_norm is grad_norm with the loss scale *scale read from device memory. With S the sum over all ranks,
// out = {total = sqrt(S)/scale, coef = (1/scale)·min(max_norm/(total + 1e-6), 1) (max_norm = +inf: no bound), found_inf = !isfinite(S)}
// and *step += !found_inf, the optimizer's effective step count. The phase-B launchers take that counter as `step` (nullable = the
// behaviour above): `coef` then addresses {coef, found_inf}; on found_inf the kernel goes straight to its closing barrier, otherwise
// the rule's bias corrections / first_step are rebuilt on the device from t = *step.
void launch_loss_scale_norm(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const double* partials, int nslots, const double* extra,
                            const float* scale, float max_norm, uint32_t parity, float* out, uint32_t* step, cudaStream_t stream);
// Phase B of every rule: the update of the owned shard from the fp32 gradient `shard` (LAMB: from the master; shard unused) with the
// coefficient *coef (LARS: nullable = 1; LAMB: none), then the all-gather of the weights and a closing barrier. With `step` (loss
// scaling, see above) coef addresses {coef, found_inf}, which LAMB takes as its vote alone.
template <class Rule>
void launch_shard_update(const PeerCtx& ctx, const PeerBuf& weights, size_t w_off, size_t bytes, int dtype, const float* shard, const float* coef,
                         const Rule& rule, const typename Rule::Params& hp, bool use_multimem, int nblocks, int nthreads, cudaStream_t stream,
                         const uint32_t* step = nullptr);
// In-bucket LAMB and LARS. The moments (LAMB) or the norms (LARS) of every shard run as launch_multi_tensor_{lamb,lars}_stage1 over
// the shard's segments (one parameter ∩ the owned slice each). lamb_ratio: parameter t's local pair ({Σw², Σu²} or {Σw², Σg̃²}) is the
// fixed-order sum of the seg_nblk[t] stage-1 partials at seg_ptr[t] (0 blocks: no segment on this rank); the per-rank pairs are
// exchanged through the symmetric `box` (2 halves · kMaxPeers · nparams double2 at box_off, half = parity) and summed in rank order →
// ratio[t] (fp32, identical bits on every rank; unused by LARS) and sums[2t], sums[2t+1]. launch_shard_update then applies the rule.
void launch_lamb_ratio(const PeerCtx& ctx, const PeerBuf& box, size_t box_off, const uint64_t* seg_ptr, const int32_t* seg_nblk, int nparams,
                       uint32_t parity, float* ratio, double* sums, cudaStream_t stream);
// Weight EMA of the in-bucket optimizers: publishes the fp32 shard `src` (the owned slice, shard-local like the master) rounded with
// Vec16<T>::pack into every rank's copy of the weights, between an opening and a closing barrier. preload_shard_publish loads the
// instantiation for one dtype / world / flavour.
void launch_shard_publish(const PeerCtx& ctx, const PeerBuf& weights, size_t w_off, size_t bytes, int dtype, const float* src, bool use_multimem,
                          int nblocks, int nthreads, cudaStream_t stream);
void preload_shard_publish(int dtype, int world, bool use_multimem);
void launch_peer_average(const PeerCtx& ctx, const PeerBuf& weights, size_t off, int peer, void* out, size_t bytes, int dtype,
                         int nblocks, int nthreads, cudaStream_t stream);
void launch_peer_barrier(const PeerCtx& ctx, cudaStream_t stream);
// One round of asynchronous model averaging in one launch (vote + snapshot → mean of the snapshots → w += mean − snapshot under the
// device-side weight gate); `status` (host-mapped) receives 1 = averaged, 0 = some rank voted stop, -1 = barrier failure.
void launch_async_average(const PeerCtx& ctx, void* w, const PeerBuf& snap, size_t snap_off, const PeerBuf& avg, size_t avg_off, size_t bytes, int dtype,
                          uint32_t seq, bool go, uint32_t* gate, unsigned long long gate_timeout_ns, int* status, bool use_multimem, int nblocks, int nthreads,
                          cudaStream_t stream);
void preload_gate_kernels();
void launch_gate_acquire(uint32_t* gate, unsigned long long timeout_ns, cudaStream_t stream);
void launch_gate_release(uint32_t* gate, cudaStream_t stream);

// ---- fused NHWC conv-block epilogues (nhwc_fused.cu); tensors are [N,H,W,C] f16/bf16, rows = N*H*W --------------------
void launch_bias_relu_nhwc_fwd(void* y, const void* bias, size_t rows, int C, int dtype, cudaStream_t stream);
// bias_grad_out/ticket == nullptr: `bias_grad` (fp32, zeroed by the caller) receives the channel sums.  Otherwise `bias_grad` is a
// zeroed fp32 workspace that the kernel leaves zeroed again, the sums land in `bias_grad_out` (tensor dtype), `ticket` is a zeroed counter.
void launch_bias_relu_nhwc_bwd(const void* g, const void* y, void* gout, float* bias_grad, size_t rows, int C, int dtype, cudaStream_t stream,
                               void* bias_grad_out = nullptr, unsigned int* ticket = nullptr);
void launch_bias_relu_pool_nhwc_fwd(const void* x, const void* bias, void* out, uint8_t* idx, int N, int H, int W, int C, int dtype,
                                    cudaStream_t stream);
void launch_bias_relu_pool_nhwc_bwd(const void* g, const void* out, const uint8_t* idx, void* gin, float* bias_grad, int N, int H, int W, int C,
                                    int dtype, cudaStream_t stream, void* bias_grad_out = nullptr, unsigned int* ticket = nullptr);

// C table of the four epilogue launchers for the optional torch extension (csrc/torch_hooks/nhwc_functions.cpp): C++ autograd
// Functions call the kernels without a Python frame. Every entry returns 0 or non-zero with the message in last_error().
extern "C" {
struct BaguaNhwcApi {
    int (*bias_relu_fwd)(void* y, const void* bias, size_t rows, int C, int dtype, void* stream);
    int (*bias_relu_bwd)(const void* g, const void* y, void* gout, float* bias_grad, size_t rows, int C, int dtype, void* stream, void* bias_grad_out,
                         unsigned int* ticket);
    int (*pool_fwd)(const void* x, const void* bias, void* out, uint8_t* idx, int N, int H, int W, int C, int dtype, void* stream);
    int (*pool_bwd)(const void* g, const void* out, const uint8_t* idx, void* gin, float* bias_grad, int N, int H, int W, int C, int dtype, void* stream,
                    void* bias_grad_out, unsigned int* ticket);
    const char* (*last_error)();
};
const BaguaNhwcApi* bagua_nhwc_api();
}

// ---- wgmma grouped GEMM (gemm_wgmma.cu) --------------------------------------------------------------------------
// C[g] = act(A[g]·B[g]^T + bias[g]); A [G,M,K], B [G,N,K], C [G,M,N] bf16 (K-contiguous operands), bias fp32 [G,N] or null; act: 0 none, 1 GELU(tanh)
bool grouped_gemm_supported(int M, int N, int K);
void launch_grouped_gemm_tn(const void* A, const void* B, void* C, const float* bias, int G, int M, int N, int K, int act, cudaStream_t stream);
// Same GEMM with the MoE combine all-to-all as its epilogue: A [G, world*cap, K] with rows ordered [source rank][slot]; the
// tile rows of source rank s are stored into `out` ON RANK s at [this rank][g][slot][N] (peer stores over NVLink).
void launch_grouped_gemm_tn_push(const void* A, const void* B, const float* bias, int G, int N, int K, int act, const PeerCtx& ctx, const PeerBuf& out,
                                 size_t out_off, int cap, cudaStream_t stream);

// ---- MoE expert-parallel token exchange (moe_kernels.cu) ------------------------------------------------
// Symmetric row buffers have layout [world(src rank), E_local, C, M]. scatter: rows_in[s] → owner's slot (optionally scaled
// per (s,k)); gather: out[s] = Σ_k w[s,k]·owner_row, optionally saving the fetched rows in picked[S,K,M].
void launch_moe_scatter(const PeerCtx& ctx, const PeerBuf& dst, size_t dst_off, const void* rows_in, const int64_t* expert_idx,
                        const int64_t* slot_idx, const float* scale, int S, int K, int M, int E_local, int C, int dtype, int nblocks,
                        cudaStream_t stream);
void launch_moe_gather(const PeerCtx& ctx, const PeerBuf& src, size_t src_off, void* out, const int64_t* expert_idx, const int64_t* slot_idx,
                       const float* weights, void* picked, int S, int K, int M, int E_local, int C, int dtype, int nblocks,
                       cudaStream_t stream, bool local_layout = false);  // local_layout: rows were pushed into MY buffer at [owner][e][slot]

// ---- quantised (MinMaxUInt8) collectives (bytegrad_kernels.cu) ------------------------------------------
// Wire format per chunk (same as the reference, kernels/bagua_kernels.cu:456-501): [min:T][max:T][pad → 32 B][u8 payload, padded → 32 B]
inline size_t align32(size_t x) { return (x + 31) / 32 * 32; }
inline size_t minmax_uint8_chunk_bytes(size_t chunk_elems) { return align32(chunk_elems) + 32; }

// Scratch of ONE quantised op instance (never shared between op types: parity bookkeeping is per instance).
struct ByteGradScratch {
    float* minmax;        // device: uint32 [2 parities][kMaxPeers + 1][2] order-encoded running min/max
    uint32_t* grid_sync;  // device: one 64-bit arrival counter of the intra-GPU grid barrier
    float* reduced;       // device: fp32 scratch for the owner's reduced chunk (chunk elements)
    unsigned long long* host_state;  // host: [0] launch sequence number, [1] total grid-barrier arrivals issued so far
};

// Fused ByteGrad bucket op: quantise P chunks → store chunk j into rank j's inbox → barrier → dequant+sum (fp32) the P
// received versions of my chunk → (÷P) → requantise → store into every rank's outbox slot → barrier → dequantise all P
// chunks into the bucket. `inbox`/`outbox` are symmetric buffers of P * minmax_uint8_chunk_bytes(chunk) bytes.
void launch_bytegrad(const PeerCtx& ctx, void* data, size_t numel, int dtype, const PeerBuf& inbox, size_t inbox_off,
                     const PeerBuf& outbox, size_t outbox_off, const ByteGradScratch& scratch, bool average, int nblocks,
                     int nthreads, cudaStream_t stream, const void* grad = nullptr, float beta1 = 0.f);  // grad: QAdam m = β1·m + (1−β1)·g in phase A

// Low-precision decentralized ring step (comm_ops/decentralized_low_precision_synchronous.rs:28-153) in one kernel.
// x: weights (in/out), w: replica of own weights, l/r: replicas of the left/right neighbours.
// box: symmetric buffer with 3 slots of minmax_uint8_chunk_bytes(numel): [0] from-left, [1] from-right, [2] own.
void launch_lpdec_ring(const PeerCtx& ctx, void* x, void* w, void* l, void* r, size_t numel, int dtype, const PeerBuf& box,
                       size_t box_off, const ByteGradScratch& scratch, int left, int right, int nblocks, int nthreads,
                       cudaStream_t stream);

// ---- single-GPU element-wise / quantisation kernels (elementwise.cu) --------------------------------------
// compress `numel` elements split in `n_chunks` equal chunks; target_chunk < 0 ⇒ all chunks.
void launch_minmax_uint8_compress(const void* in, size_t numel, int dtype, int n_chunks, int target_chunk, uint8_t* out,
                                  float* minmax_scratch, cudaStream_t stream);
void launch_minmax_uint8_decompress(const uint8_t* in, size_t numel, int dtype, int n_chunks, void* out, cudaStream_t stream);
// w += red / P - snap   (async model average apply, kernels/bagua_kernels.cu:257-267)
void launch_async_apply(void* w, const void* red, const void* snap, size_t numel, int dtype, float inv_p, cudaStream_t stream);
// out[target] = (sum over chunks of in) (* 1/P when average) — scatter-gather reduce (K7)
void launch_reduce_chunks(void* data, size_t chunk_elems, int n_chunks, int target_chunk, int dtype, bool average,
                          cudaStream_t stream);
void launch_axpby(void* x, const void* y, size_t numel, int dtype, float a, float b, cudaStream_t stream);  // x = a*x + b*y
void launch_scale(void* x, size_t numel, int dtype, float a, cudaStream_t stream);                            // x *= a
void launch_cast(const void* in, int in_dtype, void* out, int out_dtype, size_t numel, cudaStream_t stream);

// ---- fused optimizers (multi_tensor.cu) ------------------------------------------------------------------------
// Flat variants run over one contiguous arena (what with_bagua + fuse produce); `model` (optional) receives the
// updated weights in the model dtype when fp32 master weights are kept (bf16/fp16 training).
void launch_flat_sgd(void* param, int param_dtype, const void* grad, int grad_dtype, float* momentum_buf, void* model,
                     int model_dtype, size_t numel, const SgdParams& hp, float grad_scale, bool zero_grad, cudaStream_t stream);
void launch_flat_adam(void* param, int param_dtype, const void* grad, int grad_dtype, float* exp_avg, float* exp_avg_sq,
                      void* model, int model_dtype, size_t numel, const AdamParams& hp, float grad_scale, bool zero_grad,
                      cudaStream_t stream);
// Multi-tensor variants: arbitrary (non-contiguous) tensor lists, chunked over a device-resident descriptor table.
struct TensorListDesc {
    const uint64_t* ptrs;   // device array [n_lists][n_tensors] of pointers
    const int64_t* sizes;   // device array [n_tensors]
    const int32_t* block_to_tensor;
    const int32_t* block_to_chunk;
    int n_tensors;
    int n_blocks;
    int chunk;
};
void launch_multi_tensor_sgd(const TensorListDesc& d, int dtype, bool has_momentum, const SgdParams& hp, float grad_scale,
                             cudaStream_t stream);
void launch_multi_tensor_adam(const TensorListDesc& d, int dtype, const AdamParams& hp, float grad_scale, cudaStream_t stream);
// mixed precision: lists [param(T), grad(T), exp_avg(f32), exp_avg_sq(f32), master(f32)]
void launch_multi_tensor_adam_mp(const TensorListDesc& d, int dtype, const AdamParams& hp, float grad_scale, cudaStream_t stream);
// mixed precision: lists [param(T), grad(T), master(f32)(, momentum(f32) when has_momentum)]
void launch_multi_tensor_sgd_mp(const TensorListDesc& d, int dtype, bool has_momentum, const SgdParams& hp, float grad_scale,
                                cudaStream_t stream);
// LAMB in two launches, lists [param(T), grad(T), exp_avg(f32), exp_avg_sq(f32)(, master(f32) when mixed)]. Stage 1: the moments with
// g = grad·*coef (coef nullable = 1), fp64 {Σw², Σu²} of each block in sums[2·block], gradient cleared when zero_grad. Stage 2: each
// block sums its tensor's block partials in a fixed order, forms the trust ratio and applies w ← w − lr·r·u (u recomputed from the
// new moments); mixed writes the fp32 master and the parameter rounded once. With `step` (device, nullable) coef addresses
// {coef, found_inf}: on found_inf stage 1 touches nothing, otherwise it takes its bias corrections from t = *step.
void launch_multi_tensor_lamb_stage1(const TensorListDesc& d, int dtype, bool mixed, const LambParams& hp, const float* coef, double* sums, bool zero_grad,
                                     cudaStream_t stream, const uint32_t* step = nullptr);
void launch_multi_tensor_lamb_stage2(const TensorListDesc& d, int dtype, bool mixed, const LambParams& hp, const double* sums, cudaStream_t stream);
// LARS in two launches, lists [param(T), grad(T), momentum(f32)(, master(f32) when mixed)]. Stage 1: fp64 {Σw², Σg̃²} of each block
// in sums[2·block] with g̃ = grad·*coef (coef nullable = 1); it reads lists 0, 1 (and the master) only and never clears the gradient.
// With `vote` coef addresses {coef, found_inf} and a found_inf step writes nothing. Stage 2: each block sums its tensor's block
// partials in a fixed order, forms the trust (lars.cuh) and applies the momentum and the update with the same g̃; mixed writes the
// fp32 master and the parameter rounded once; the gradient is cleared when zero_grad.
void launch_multi_tensor_lars_stage1(const TensorListDesc& d, int dtype, bool mixed, const float* coef, double* sums, cudaStream_t stream, bool vote = false);
void launch_multi_tensor_lars_stage2(const TensorListDesc& d, int dtype, bool mixed, const LarsParams& hp, const float* coef, const double* sums, bool zero_grad,
                                     cudaStream_t stream);
// Lion in one launch, lists [param(T), grad(T), (master(f32) when mixed,) exp_avg(f32)]: lion.cuh's update with g = grad; mixed writes
// the fp32 master and the parameter rounded once; the gradient is cleared in the same pass when zero_grad.
void launch_multi_tensor_lion(const TensorListDesc& d, int dtype, bool mixed, const LionParams& hp, bool zero_grad, cudaStream_t stream);
// Exponential moving average of fp32 weights, lists [source(f32), ema(f32)]: e ← fl(e + fl(w·fl(m − e))), three separately rounded
// operations. `vote` (nullable): with *vote != 0 (an overflowed loss-scaled step) nothing is written.
void launch_multi_tensor_ema(const TensorListDesc& d, float weight, const float* vote, cudaStream_t stream);
// QAdam momentum pre-step (bagua/torch_api/algorithms/q_adam.py:193-221): m = beta1*m + (1-beta1)*g
void launch_qadam_momentum(float* exp_avg, const void* grad, int grad_dtype, size_t numel, float beta1, cudaStream_t stream);

}  // namespace bagua
