// PeerComm (per-group NVSwitch communicator state) and the native comm ops a bucket can run.
//
// Reference counterparts: BaguaSingleCommunicator (communicators/mod.rs:26-73, 474-489) and the six comm ops
// (comm_ops/*.rs). Here a "communicator" is nothing but symmetric signal pads + an abort/timeout flag: the
// collectives themselves are kernels (peer_kernels.cu, bytegrad_kernels.cu) that load/store peer memory.
#pragma once
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "kernels.h"
#include "scheduler.h"

namespace bagua {

class PeerComm {
public:
    // flag_ptrs[p] = address (mapped in this process) of rank p's signal pad, ≥ kMaxCommBlocks*kMaxPeers*4 bytes, zeroed.
    PeerComm(int rank, int world, int device, const std::vector<uint64_t>& flag_ptrs, double timeout_s);
    ~PeerComm();
    PeerComm(const PeerComm&) = delete;
    const PeerCtx& ctx() const { return ctx_; }
    int rank() const { return ctx_.rank; }
    int world() const { return ctx_.world; }
    int device() const { return device_; }
    void abort();            // make every spinning kernel of this comm give up (ncclCommAbort analogue)
    void reset_abort();
    bool aborted() const;
    int error_code();        // synchronising read of the device error word (0 ok, 1 timeout, 2 aborted, 3 grid timeout, 4 protocol)
    // Non-synchronising read of the host-mapped mirror of the error word: what a failed kernel left behind (0 = healthy).
    int host_error() const { return __atomic_load_n(host_words_ + 1, __ATOMIC_ACQUIRE); }
    // Throws when a kernel of this communicator has failed: a collective that was skipped on some rank means diverged replicas,
    // so the failure is fatal for every later op (the reference's NCCL path blocks and then panics via its watchdog instead).
    void check_fatal(const char* what) const;
    void clear_error();
    void set_timeout(double seconds);
    uint32_t next_oneshot_parity() { return oneshot_calls_++ & 1u; }
    static size_t signal_pad_bytes() { return (static_cast<size_t>(kMaxCommBlocks) * kMaxPeers + kVoteWords) * sizeof(uint32_t); }

private:
    PeerCtx ctx_{};
    int device_;
    int* host_words_ = nullptr;  // host-mapped: [0] abort flag, [1] error mirror
    uint32_t oneshot_calls_ = 0;
};

struct SymmBuf {
    PeerBuf buf{};
    size_t bytes = 0;
    SymmBuf() = default;
    SymmBuf(const std::vector<uint64_t>& ptrs, uint64_t mc, size_t nbytes);
    bool has_multicast() const { return buf.mc != nullptr; }
};

struct LaunchCfg {
    int nblocks = 32;
    int nthreads = 512;
};

// Per-instance scratch of a quantised op (device allocations + host counters).
class QuantScratch {
public:
    QuantScratch(int device, size_t reduced_elems);
    ~QuantScratch();
    QuantScratch(const QuantScratch&) = delete;
    const ByteGradScratch& get() const { return s_; }

private:
    ByteGradScratch s_{};
    unsigned long long host_state_[2] = {0, 0};
    int device_;
};

class AllReduceOp final : public CommOp {
public:
    AllReduceOp(std::shared_ptr<PeerComm> comm, SymmBuf src, SymmBuf dst, size_t src_off, size_t dst_off, size_t bytes,
                int dtype, float scale, int variant, LaunchCfg cfg)
        : comm_(std::move(comm)), src_(src), dst_(dst), src_off_(src_off), dst_off_(dst_off), bytes_(bytes), dtype_(dtype),
          scale_(scale), variant_(variant), cfg_(cfg) {}
    const char* kind() const override { return variant_ == AR_MULTIMEM ? "allreduce_multimem" : "allreduce_twoshot"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    void set_variant(int v, LaunchCfg cfg) { variant_ = v, cfg_ = cfg; }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf src_, dst_;
    size_t src_off_, dst_off_, bytes_;
    int dtype_;
    float scale_;
    int variant_;
    LaunchCfg cfg_;
};

class AllReduceOneShotOp final : public CommOp {
public:
    AllReduceOneShotOp(std::shared_ptr<PeerComm> comm, SymmBuf staging, size_t staging_off, size_t slot_bytes, uint64_t in, uint64_t out,
                       size_t bytes, int dtype, float scale, LaunchCfg cfg)
        : comm_(std::move(comm)), staging_(staging), staging_off_(staging_off), slot_bytes_(slot_bytes), in_(in), out_(out), bytes_(bytes), dtype_(dtype),
          scale_(scale), cfg_(cfg) {}
    const char* kind() const override { return "allreduce_oneshot"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // the staging half alternates with the communicator's call counter

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf staging_;
    size_t staging_off_;
    size_t slot_bytes_;
    uint64_t in_, out_;
    size_t bytes_;
    int dtype_;
    float scale_;
    LaunchCfg cfg_;
};

// Host hyper-parameters of the in-bucket optimizer rules, in the argument order of their ops' set_hyper.
struct SgdHyper {
    float lr = 0.01f, momentum = 0.f, dampening = 0.f, weight_decay = 0.f;
    bool nesterov = false;
};
struct AdamHyper {
    float lr = 1e-3f, beta1 = 0.9f, beta2 = 0.999f, eps = 1e-8f, weight_decay = 0.f;
    bool adamw = false;
};
struct LambHyper {
    float lr = 1e-3f, beta1 = 0.9f, beta2 = 0.999f, eps = 1e-6f, weight_decay = 0.01f;
};
struct LarsHyper {
    float lr = 1e-3f, momentum = 0.9f, weight_decay = 0.f, trust_coefficient = 1e-3f;
};
// in double: the kernel's constants are worked out from these and rounded once (lion_params)
struct LionHyper {
    double lr = 1e-4, beta1 = 0.9, beta2 = 0.99, weight_decay = 0.0;
};

// What a rule's kernel receives at the launch that follows `steps` earlier ones.
inline SgdParams device_params(const SgdHyper& h, uint64_t steps) {
    return SgdParams{h.lr, h.momentum, h.dampening, h.weight_decay, h.nesterov ? 1 : 0, steps == 0 ? 1 : 0};
}
inline AdamParams device_params(const AdamHyper& h, uint64_t steps) {
    return adam_params(h.lr, h.beta1, h.beta2, h.eps, h.weight_decay, h.adamw, steps + 1);
}
inline LambParams device_params(const LambHyper& h, uint64_t steps) { return lamb_params(h.lr, h.beta1, h.beta2, h.eps, h.weight_decay, steps + 1); }
inline LarsParams device_params(const LarsHyper& h, uint64_t) { return LarsParams{h.lr, h.momentum, h.weight_decay, h.trust_coefficient}; }
inline LionParams device_params(const LionHyper& h, uint64_t) { return lion_params(h.lr, h.beta1, h.beta2, h.weight_decay); }

// An optimizer op: hyper-parameters published from Python (the forward pre-hook may do so while the comm worker runs the op, hence
// the lock) and the count of launches so far, which checkpoints save and restore. With loss scaling a launch may be a skipped step,
// so the count that matters lives on the device: set_device_step(vote, step) hands the op the {coef, found_inf} pair and the
// effective step counter that LossScaleNormOp maintains; the kernel then takes its gradient coefficient from `vote`, obeys
// found_inf and derives the step-dependent parameters from *step instead of from steps().
template <class Hyper>
class SteppedOp : public CommOp {
public:
    void set_hyper(const Hyper& h) {
        std::lock_guard<std::mutex> lk(mu_);
        hp_ = h;
    }
    uint64_t steps() const { return steps_; }
    void set_steps(uint64_t s) { steps_ = s; }
    void set_device_step(uint64_t vote, uint64_t step) {
        if ((vote == 0) != (step == 0)) throw std::invalid_argument("bagua: an optimizer op takes the vote and the step counter together");
        vote_ = vote, dev_step_ = step;
    }

protected:
    const float* coef_or_vote(uint64_t coef) const { return reinterpret_cast<const float*>(vote_ ? vote_ : coef); }
    const float* vote() const { return reinterpret_cast<const float*>(vote_); }
    const uint32_t* dev_step() const { return reinterpret_cast<const uint32_t*>(dev_step_); }
    auto params() {
        std::lock_guard<std::mutex> lk(mu_);
        return device_params(hp_, steps_);
    }
    uint64_t steps_ = 0;

private:
    uint64_t vote_ = 0, dev_step_ = 0;
    Hyper hp_;
    std::mutex mu_;
};

// The host side of each in-bucket optimizer rule (kernels.h): its hyper-parameters, and whether its kernel arguments are the same at
// every launch that follows `steps` earlier ones.
template <class Rule>
struct RuleHost;
template <>
struct RuleHost<SgdRule> {
    using Hyper = SgdHyper;
    static bool step_invariant(uint64_t steps) { return steps > 0; }  // only the very first launch differs (momentum initialisation)
};
template <>
struct RuleHost<AdamRule> {
    using Hyper = AdamHyper;
    static bool step_invariant(uint64_t) { return false; }  // bias corrections are passed by value
};
template <>
struct RuleHost<LambRule> {
    using Hyper = LambHyper;
    static bool step_invariant(uint64_t) { return false; }  // bias corrections are passed by value
};
template <>
struct RuleHost<LarsRule> {
    using Hyper = LarsHyper;
    static bool step_invariant(uint64_t) { return true; }
};
template <>
struct RuleHost<LionRule> {
    using Hyper = LionHyper;
    static bool step_invariant(uint64_t) { return true; }
};

// reduce-scatter(grads) → the rule on the owned shard → all-gather(weights), one kernel per bucket, during backward (SGD, Adam, Lion).
// `rule` holds the rule's state pointers; each run passes the parameters of its launch.
template <class Rule>
class FusedUpdateOp final : public SteppedOp<typename RuleHost<Rule>::Hyper> {
public:
    FusedUpdateOp(std::shared_ptr<PeerComm> comm, SymmBuf grads, SymmBuf weights, size_t g_off, size_t w_off, size_t bytes, int dtype, Rule rule,
                  float scale, bool zero_grads, bool use_multimem, LaunchCfg cfg)
        : comm_(std::move(comm)), grads_(grads), weights_(weights), g_off_(g_off), w_off_(w_off), bytes_(bytes), dtype_(dtype), rule_(rule),
          scale_(scale), zero_grads_(zero_grads), use_mc_(use_multimem), cfg_(cfg) {}
    const char* kind() const override { return Rule::kFused; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return RuleHost<Rule>::step_invariant(this->steps_); }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf grads_, weights_;
    size_t g_off_, w_off_, bytes_;
    int dtype_;
    Rule rule_;
    const float scale_;
    bool zero_grads_, use_mc_;
    LaunchCfg cfg_;
};


// Intra-node halves of a hierarchical all-reduce (see reduce_scatter_kernel): ReduceScatterOp, then a callback op that
// all-reduces slice `rank` between nodes, then AllGatherOp.
class ReduceScatterOp final : public CommOp {
public:
    ReduceScatterOp(std::shared_ptr<PeerComm> comm, SymmBuf buf, size_t off, size_t bytes, int dtype, float scale, bool use_multimem, LaunchCfg cfg)
        : comm_(std::move(comm)), buf_(buf), off_(off), bytes_(bytes), dtype_(dtype), scale_(scale), use_mc_(use_multimem), cfg_(cfg) {}
    const char* kind() const override { return "reduce_scatter"; }
    void run(Bucket&, StreamHandle stream, int device) override;

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf buf_;
    size_t off_, bytes_;
    int dtype_;
    float scale_;
    bool use_mc_;
    LaunchCfg cfg_;
};

class AllGatherOp final : public CommOp {
public:
    AllGatherOp(std::shared_ptr<PeerComm> comm, SymmBuf buf, size_t off, size_t bytes, int dtype, bool use_multimem, LaunchCfg cfg)
        : comm_(std::move(comm)), buf_(buf), off_(off), bytes_(bytes), dtype_(dtype), use_mc_(use_multimem), cfg_(cfg) {}
    const char* kind() const override { return "all_gather"; }
    void run(Bucket&, StreamHandle stream, int device) override;

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf buf_;
    size_t off_, bytes_;
    int dtype_;
    bool use_mc_;
    LaunchCfg cfg_;
};


// Global-norm clipping of the in-bucket optimizers (see shard_grad_kernel). Phase A, in the bucket program: reduce-scatter of the
// gradients into the fp32 shard of the owned slice, per-CTA fp64 Σx² into `partials` (kMaxCommBlocks doubles), bucket cleared.
// An `accumulate` op sums micro-batches in the shard: its first run after construction or restart() overwrites the shard (the
// kernel of a non-accumulating op), every later run adds to it. run() is called by the comm worker or the inline-issue thread,
// restart() / resume() by the Python thread, hence the atomic.
class ShardGradOp final : public CommOp {
public:
    ShardGradOp(std::shared_ptr<PeerComm> comm, SymmBuf grads, size_t g_off, size_t bytes, int dtype, uint64_t shard, uint64_t partials, float scale,
                bool zero_grads, bool use_multimem, LaunchCfg cfg, bool accumulate = false);
    const char* kind() const override { return "shard_grad_sumsq"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return !accumulate_; }  // overwrite, then add
    void restart() { fresh_.store(true, std::memory_order_release); }
    // the shard holds a sum the next run adds to (a re-bucketing carried it over)
    void resume() { fresh_.store(false, std::memory_order_release); }
    // whether the shard holds a sum that the next run adds to
    bool pending() const { return accumulate_ && !fresh_.load(std::memory_order_acquire); }
    bool accumulate() const { return accumulate_; }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf grads_;
    size_t g_off_, bytes_;
    int dtype_;
    uint64_t shard_, partials_;
    float scale_;
    bool zero_grads_, use_mc_;
    LaunchCfg cfg_;
    const bool accumulate_;
    std::atomic<bool> fresh_{true};
};

// The norm exchange: out = {total, coef} (fp32, device) from the `nslots` partials of this rank plus *extra (fp64, the parameters
// outside the buckets; 0 = none) and the peers' sums. The box is double-buffered by this op's own call counter.
class GradNormOp final : public CommOp {
public:
    GradNormOp(std::shared_ptr<PeerComm> comm, SymmBuf box, size_t box_off, uint64_t partials, int nslots, uint64_t extra, uint64_t out)
        : comm_(std::move(comm)), box_(box), box_off_(box_off), partials_(partials), nslots_(nslots), extra_(extra), out_(out) {}
    const char* kind() const override { return "grad_norm"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // the box half alternates with the call counter
    void set_max_norm(float m) { max_norm_ = m; }
    uint64_t calls() const { return calls_; }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf box_;
    size_t box_off_;
    uint64_t partials_;
    int nslots_;
    uint64_t extra_, out_;
    float max_norm_ = 1.f;
    uint64_t calls_ = 0;
};

// The norm exchange of an optimizer with loss scaling (see loss_scale_norm_kernel): GradNormOp with the loss scale read from device
// memory at `scale` (settable: the scaler's tensor, or a constant 1), out = {total, coef, found_inf} and the effective step count
// `step` (uint32, device) advanced on every step that is not skipped. max_norm = +inf: no clipping.
class LossScaleNormOp final : public CommOp {
public:
    LossScaleNormOp(std::shared_ptr<PeerComm> comm, SymmBuf box, size_t box_off, uint64_t partials, int nslots, uint64_t extra, uint64_t out, uint64_t step)
        : comm_(std::move(comm)), box_(box), box_off_(box_off), partials_(partials), nslots_(nslots), extra_(extra), out_(out), step_(step) {}
    const char* kind() const override { return "loss_scale_norm"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // the box half alternates with the call counter
    void set_max_norm(float m) { max_norm_ = m; }
    void set_scale_ptr(uint64_t scale) { scale_ = scale; }
    uint64_t calls() const { return calls_; }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf box_;
    size_t box_off_;
    uint64_t partials_;
    int nslots_;
    uint64_t extra_, out_, step_;
    uint64_t scale_ = 0;
    float max_norm_ = INFINITY;
    uint64_t calls_ = 0;
};

// Phase B of every rule, run from step(): the rule on the owned shard from the gradient shard·coef, all-gather of the weights (see
// shard_update_kernel). LAMB reads the master instead and no coefficient: its shard and coef are 0. With set_device_step the coef is
// the vote's {coef, found_inf}. Carries the step counter like the fused op (checkpoints see the same interface).
template <class Rule>
class ShardUpdateOp final : public SteppedOp<typename RuleHost<Rule>::Hyper> {
public:
    ShardUpdateOp(std::shared_ptr<PeerComm> comm, SymmBuf weights, size_t w_off, size_t bytes, int dtype, uint64_t shard, uint64_t coef, Rule rule,
                  bool use_multimem, LaunchCfg cfg)
        : comm_(std::move(comm)), weights_(weights), w_off_(w_off), bytes_(bytes), dtype_(dtype), shard_(shard), coef_(coef), rule_(rule),
          use_mc_(use_multimem), cfg_(cfg) {}
    const char* kind() const override { return Rule::kShard; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return RuleHost<Rule>::step_invariant(this->steps_); }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf weights_;
    size_t w_off_, bytes_;
    int dtype_;
    uint64_t shard_, coef_;
    Rule rule_;
    bool use_mc_;
    LaunchCfg cfg_;
};

// In-bucket LAMB, run from step() after phase A (ShardGradOp): LambMomentsOp per bucket (the multi-tensor stage-1 kernel over the
// shard's segment table: fp32 master / gradient shard·*coef / moments, fp64 {Σw², Σu²} per block into `partials`), LambRatioOp once
// per step (the per-parameter exchange), ShardUpdateOp<LambRule> per bucket (apply + all-gather + barrier). The moments and apply ops carry the
// step count (bias corrections) and advance together.
class LambMomentsOp final : public SteppedOp<LambHyper> {
public:
    LambMomentsOp(uint64_t ptrs, uint64_t sizes, uint64_t b2t, uint64_t b2c, int n_tensors, int n_blocks, int chunk, uint64_t coef, uint64_t partials)
        : desc_{reinterpret_cast<const uint64_t*>(ptrs), reinterpret_cast<const int64_t*>(sizes), reinterpret_cast<const int32_t*>(b2t),
                reinterpret_cast<const int32_t*>(b2c), n_tensors, n_blocks, chunk},
          coef_(coef), partials_(partials) {}
    const char* kind() const override { return "lamb_moments"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // bias corrections are passed by value

private:
    TensorListDesc desc_;
    uint64_t coef_, partials_;
};

class LambRatioOp final : public CommOp {
public:
    LambRatioOp(std::shared_ptr<PeerComm> comm, SymmBuf box, size_t box_off, uint64_t seg_ptr, uint64_t seg_nblk, int nparams, uint64_t ratio, uint64_t sums)
        : comm_(std::move(comm)), box_(box), box_off_(box_off), seg_ptr_(seg_ptr), seg_nblk_(seg_nblk), nparams_(nparams), ratio_(ratio), sums_(sums) {}
    const char* kind() const override { return "lamb_ratio"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // the box half alternates with the call counter
    uint64_t calls() const { return calls_; }
    static size_t box_bytes(int nparams) { return 2 * static_cast<size_t>(kMaxPeers) * nparams * 2 * sizeof(double); }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf box_;
    size_t box_off_;
    uint64_t seg_ptr_, seg_nblk_;
    int nparams_;
    uint64_t ratio_, sums_;
    uint64_t calls_ = 0;
};

// In-bucket LARS, run from step() after phase A like LAMB: LarsNormsOp per bucket (the multi-tensor LARS stage 1 over the shard's
// segment table, lists [fp32 master, gradient shard]: fp64 {Σw², Σg̃²} per block into `partials`, g̃ = shard·*coef), the LAMB
// ratio exchange (LambRatioOp) once per step for the per-parameter global sums, ShardUpdateOp<LarsRule> per bucket (momentum + apply from the
// exchanged sums, all-gather, barrier). The rule has no step-dependent parameter; both ops count their launches for checkpoints.
class LarsNormsOp final : public SteppedOp<LarsHyper> {
public:
    LarsNormsOp(uint64_t ptrs, uint64_t sizes, uint64_t b2t, uint64_t b2c, int n_tensors, int n_blocks, int chunk, uint64_t coef, uint64_t partials)
        : desc_{reinterpret_cast<const uint64_t*>(ptrs), reinterpret_cast<const int64_t*>(sizes), reinterpret_cast<const int32_t*>(b2t),
                reinterpret_cast<const int32_t*>(b2c), n_tensors, n_blocks, chunk},
          coef_(coef), partials_(partials) {}
    const char* kind() const override { return "lars_norms"; }
    void run(Bucket&, StreamHandle stream, int device) override;

private:
    TensorListDesc desc_;
    uint64_t coef_, partials_;
};

// Weight EMA of the in-bucket optimizers. EmaOp is local: one multi-tensor launch of e ← e + w·(m − e) over the table's
// [source, ema] pairs (every bucket's master and EMA shards, or the parameters outside the buckets), skipped on the device when the
// vote word (nullable: the loss-scaled step's found_inf) is set. ShardPublishOp all-gathers an fp32 shard, rounded to the bucket's
// dtype, into every rank's weights (see shard_publish_kernel).
class EmaOp final : public CommOp {
public:
    EmaOp(uint64_t ptrs, uint64_t sizes, uint64_t b2t, uint64_t b2c, int n_tensors, int n_blocks, int chunk, float weight, uint64_t vote)
        : desc_{reinterpret_cast<const uint64_t*>(ptrs), reinterpret_cast<const int64_t*>(sizes), reinterpret_cast<const int32_t*>(b2t),
                reinterpret_cast<const int32_t*>(b2c), n_tensors, n_blocks, chunk},
          weight_(weight), vote_(vote) {}
    const char* kind() const override { return "ema"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // the weight is the host's at launch
    void set_weight(float w) { weight_.store(w, std::memory_order_relaxed); }
    float weight() const { return weight_.load(std::memory_order_relaxed); }

private:
    TensorListDesc desc_;
    std::atomic<float> weight_;
    uint64_t vote_;
};

class ShardPublishOp final : public CommOp {
public:
    ShardPublishOp(std::shared_ptr<PeerComm> comm, SymmBuf weights, size_t w_off, size_t bytes, int dtype, uint64_t src, bool use_multimem, LaunchCfg cfg);
    const char* kind() const override { return "shard_publish"; }
    void run(Bucket&, StreamHandle stream, int device) override;

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf weights_;
    size_t w_off_, bytes_;
    int dtype_;
    uint64_t src_;
    bool use_mc_;
    LaunchCfg cfg_;
};

// Decentralized SGD, shift_one pairing (peer formula: comm_ops/decentralized_full_precision_synchronous.rs:81-85).
class PeerAverageOp final : public CommOp {
public:
    PeerAverageOp(std::shared_ptr<PeerComm> comm, SymmBuf weights, size_t off, uint64_t out, size_t bytes, int dtype, LaunchCfg cfg)
        : comm_(std::move(comm)), weights_(weights), off_(off), out_(out), bytes_(bytes), dtype_(dtype), cfg_(cfg) {}
    const char* kind() const override { return "peer_average_shift_one"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }  // the partner rotates with the step
    static int shift_one_peer(int rank, int nranks, int64_t step);
    int64_t step() const { return step_; }

private:
    std::shared_ptr<PeerComm> comm_;
    SymmBuf weights_;
    size_t off_;
    uint64_t out_;
    size_t bytes_;
    int dtype_;
    LaunchCfg cfg_;
    int64_t step_ = 0;
};

class ByteGradOp final : public CommOp {
public:
    ByteGradOp(std::shared_ptr<PeerComm> comm, uint64_t data, size_t numel, int dtype, SymmBuf inbox, size_t inbox_off, SymmBuf outbox,
               size_t outbox_off, bool average, LaunchCfg cfg);
    const char* kind() const override { return grad_ ? "qadam_momentum_bytegrad_fused" : "bytegrad_fused"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    // QAdam compressed stage: the bucket holds the first moment; `grad` (same layout, same dtype) is folded in as
    // m = beta1*m + (1-beta1)*grad inside the kernel's first pass (0 switches it off).
    void set_momentum_source(uint64_t grad, float beta1) { grad_ = grad, beta1_ = beta1; }
    static size_t box_bytes(size_t numel, int nranks) { return static_cast<size_t>(nranks) * minmax_uint8_chunk_bytes(numel / nranks); }

private:
    std::shared_ptr<PeerComm> comm_;
    uint64_t data_;
    size_t numel_;
    int dtype_;
    SymmBuf inbox_, outbox_;
    size_t inbox_off_, outbox_off_;
    bool average_;
    LaunchCfg cfg_;
    std::unique_ptr<QuantScratch> scratch_;
    uint64_t grad_ = 0;
    float beta1_ = 0.f;
};

class LowPrecRingOp final : public CommOp {
public:
    LowPrecRingOp(std::shared_ptr<PeerComm> comm, uint64_t x, uint64_t w, uint64_t l, uint64_t r, size_t numel, int dtype, SymmBuf box,
                  size_t box_off, LaunchCfg cfg);
    const char* kind() const override { return "low_precision_ring_fused"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    static size_t box_bytes(size_t numel) { return 6 * minmax_uint8_chunk_bytes(numel); }

private:
    std::shared_ptr<PeerComm> comm_;
    uint64_t x_, w_, l_, r_;
    size_t numel_;
    int dtype_;
    SymmBuf box_;
    size_t box_off_;
    LaunchCfg cfg_;
    std::unique_ptr<QuantScratch> scratch_;
};

// The device-side weight gate of asynchronous model averaging (see async_average_kernel): a few words in device memory that the
// trainer's stream acquires before a forward pass and releases after the optimizer step, and that the averaging kernel takes for
// its apply phase. Replaces the reference's host mutex + two host synchronisations per iteration.
class WeightGate {
public:
    explicit WeightGate(int device);
    ~WeightGate();
    WeightGate(const WeightGate&) = delete;
    uint32_t* words() const { return words_; }
    void acquire(StreamHandle stream, double timeout_s);  // enqueue on the trainer's stream
    void release(StreamHandle stream);
    uint32_t state();                                      // synchronising read (tests / diagnostics)

private:
    uint32_t* words_ = nullptr;
    int device_;
};

// One round of asynchronous model averaging = one kernel (comm op 5; reference decentralized_full_precision_asynchronous.rs:97-162).
class AsyncAverageOp final : public CommOp {
public:
    AsyncAverageOp(std::shared_ptr<PeerComm> comm, uint64_t weights, SymmBuf snap, size_t snap_off, SymmBuf avg, size_t avg_off, size_t bytes, int dtype,
                   std::shared_ptr<WeightGate> gate, double gate_timeout_s, bool use_multimem, LaunchCfg cfg);
    ~AsyncAverageOp() override;
    const char* kind() const override { return "async_model_average_fused"; }
    void run(Bucket&, StreamHandle stream, int device) override;
    bool step_invariant() const override { return false; }
    void abort() { go_.store(false); }   // this rank votes "stop" from the next round on
    void reset() {
        go_.store(true);
        *status_host_ = 1;
    }
    // Outcome of the last completed round (host-mapped word written by the kernel): 1 averaged, 0 a rank voted stop (all ranks see
    // the same), -1 failed. Valid once the round's ticket has completed.
    int status() const { return __atomic_load_n(status_host_, __ATOMIC_ACQUIRE); }
    uint64_t rounds() const { return seq_; }

private:
    std::shared_ptr<PeerComm> comm_;
    uint64_t w_;
    SymmBuf snap_, avg_;
    size_t snap_off_, avg_off_, bytes_;
    int dtype_;
    std::shared_ptr<WeightGate> gate_;
    double gate_timeout_s_;
    bool use_mc_;
    LaunchCfg cfg_;
    std::atomic<bool> go_{true};
    uint32_t seq_ = 0;
    int* status_host_ = nullptr;
    int* status_dev_ = nullptr;
};

// Plain device-to-device copy on the comm stream (snapshots / copy-back).
class CopyOp final : public CommOp {
public:
    CopyOp(uint64_t dst, uint64_t src, size_t bytes) : dst_(dst), src_(src), bytes_(bytes) {}
    const char* kind() const override { return "copy"; }
    void run(Bucket&, StreamHandle stream, int device) override;

private:
    uint64_t dst_, src_;
    size_t bytes_;
};

}  // namespace bagua
