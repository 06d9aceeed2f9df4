// Host-callable launchers of every CUDA kernel in bagua_b200 (implemented in *.cu, sm_90a).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
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

// ---- peer kernels (peer_kernels.cu) ------------------------------------------------------------------------
void launch_allreduce(const PeerCtx& ctx, const PeerBuf& src, const PeerBuf& dst, size_t src_off, size_t dst_off, size_t bytes,
                      int dtype, float scale, int variant, int nblocks, int nthreads, cudaStream_t stream);
void launch_allreduce_oneshot(const PeerCtx& ctx, const PeerBuf& staging, size_t staging_off, size_t slot_bytes, const void* in, void* out,
                              size_t bytes, int dtype, float scale, int nblocks, int nthreads, cudaStream_t stream, uint32_t call_parity);
void launch_allreduce_sgd(const PeerCtx& ctx, const PeerBuf& grads, const PeerBuf& weights, size_t g_off, size_t w_off,
                          size_t bytes, int dtype, float* master, float* momentum, const SgdParams& hp, float scale,
                          bool zero_grads, bool use_multimem, int nblocks, int nthreads, cudaStream_t stream);
// Halves of the two-shot schedule (hierarchical all-reduce): in-place reduce of slice `rank` over the group (scaled), and
// publication of slice `rank` to every peer. Slices are ceil(vecs / world) 16-byte vectors.
void launch_reduce_scatter(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, float scale, bool use_multimem, int nblocks,
                           int nthreads, cudaStream_t stream);
void launch_all_gather(const PeerCtx& ctx, const PeerBuf& buf, size_t off, size_t bytes, int dtype, bool use_multimem, int nblocks, int nthreads,
                       cudaStream_t stream);
// Adam / AdamW variant (fp32 master + both moments sharded world ways); hp carries the bias corrections of THIS step.
void launch_allreduce_adam(const PeerCtx& ctx, const PeerBuf& grads, const PeerBuf& weights, size_t g_off, size_t w_off, size_t bytes, int dtype,
                           float* master, float* exp_avg, float* exp_avg_sq, const AdamParams& hp, float scale, bool zero_grads, bool use_multimem,
                           int nblocks, int nthreads, cudaStream_t stream);
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
// QAdam momentum pre-step (bagua/torch_api/algorithms/q_adam.py:193-221): m = beta1*m + (1-beta1)*g
void launch_qadam_momentum(float* exp_avg, const void* grad, int grad_dtype, size_t numel, float beta1, cudaStream_t stream);

}  // namespace bagua
