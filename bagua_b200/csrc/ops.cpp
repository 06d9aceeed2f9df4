#include "ops.h"

#include <cuda_runtime.h>

#include <cstring>

#include <atomic>

namespace bagua {

static std::atomic<uint64_t> g_launches{0};
uint64_t launch_count() { return g_launches.load(std::memory_order_relaxed); }
void count_launch(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

namespace {
inline cudaStream_t S(StreamHandle s) { return reinterpret_cast<cudaStream_t>(s); }
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) BAGUA_CUDA_CHECK(cudaSetDevice(dev));
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};
}  // namespace

PeerComm::PeerComm(int rank, int world, int device, const std::vector<uint64_t>& flag_ptrs, double timeout_s) : device_(device) {
    if (world < 1 || world > kMaxPeers) throw std::invalid_argument("bagua: PeerComm supports 1..8 ranks");
    if (static_cast<int>(flag_ptrs.size()) != world) throw std::invalid_argument("bagua: PeerComm needs one signal pad pointer per rank");
    if (rank < 0 || rank >= world) throw std::invalid_argument("bagua: PeerComm rank out of range");
    DeviceGuard g(device);
    std::memset(&ctx_, 0, sizeof(ctx_));
    for (int p = 0; p < world; ++p) ctx_.flags[p] = reinterpret_cast<uint32_t*>(flag_ptrs[p]);
    BAGUA_CUDA_CHECK(cudaMalloc(&ctx_.epochs, kMaxCommBlocks * sizeof(uint32_t)));
    BAGUA_CUDA_CHECK(cudaMemset(ctx_.epochs, 0, kMaxCommBlocks * sizeof(uint32_t)));
    BAGUA_CUDA_CHECK(cudaMalloc(&ctx_.error, sizeof(int)));
    BAGUA_CUDA_CHECK(cudaMemset(ctx_.error, 0, sizeof(int)));
    BAGUA_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&host_words_), 2 * sizeof(int), cudaHostAllocMapped));
    host_words_[0] = host_words_[1] = 0;
    int* dev_view = nullptr;
    BAGUA_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dev_view), host_words_, 0));
    ctx_.abort = dev_view;
    ctx_.host_error = dev_view + 1;
    ctx_.rank = rank;
    ctx_.world = world;
    set_timeout(timeout_s);
    BAGUA_CUDA_CHECK(cudaDeviceSynchronize());
}

PeerComm::~PeerComm() {
    // Best effort: the context may already be gone at interpreter shutdown.
    if (ctx_.epochs) cudaFree(ctx_.epochs);
    if (ctx_.error) cudaFree(ctx_.error);
    if (host_words_) cudaFreeHost(host_words_);
}

void PeerComm::abort() { __atomic_store_n(host_words_, 1, __ATOMIC_RELEASE); }
void PeerComm::reset_abort() { __atomic_store_n(host_words_, 0, __ATOMIC_RELEASE); }
bool PeerComm::aborted() const { return __atomic_load_n(host_words_, __ATOMIC_ACQUIRE) != 0; }

void PeerComm::check_fatal(const char* what) const {
    const int code = host_error();
    if (code == 0) return;
    static const char* names[] = {"", "timed out waiting for another rank", "was aborted", "timed out in its grid barrier", "saw a peer in a different round"};
    throw std::runtime_error(std::string("bagua: an earlier peer kernel of this communicator ") + (code >= 1 && code <= 4 ? names[code] : "failed") +
                             " (error " + std::to_string(code) + "); the collective was skipped on this rank, replicas may have diverged — refusing to run " + what);
}
void PeerComm::set_timeout(double seconds) { ctx_.timeout_ns = static_cast<unsigned long long>(seconds * 1e9); }

int PeerComm::error_code() {
    DeviceGuard g(device_);
    int v = 0;
    BAGUA_CUDA_CHECK(cudaMemcpy(&v, ctx_.error, sizeof(int), cudaMemcpyDeviceToHost));
    return v;
}
void PeerComm::clear_error() {
    DeviceGuard g(device_);
    BAGUA_CUDA_CHECK(cudaMemset(ctx_.error, 0, sizeof(int)));
    __atomic_store_n(host_words_ + 1, 0, __ATOMIC_RELEASE);
}

SymmBuf::SymmBuf(const std::vector<uint64_t>& ptrs, uint64_t mc, size_t nbytes) : bytes(nbytes) {
    if (ptrs.empty() || ptrs.size() > static_cast<size_t>(kMaxPeers)) throw std::invalid_argument("bagua: SymmBuf needs 1..8 peer pointers");
    std::memset(&buf, 0, sizeof(buf));
    for (size_t p = 0; p < ptrs.size(); ++p) buf.ptr[p] = reinterpret_cast<char*>(ptrs[p]);
    buf.mc = reinterpret_cast<char*>(mc);
}

QuantScratch::QuantScratch(int device, size_t reduced_elems) : device_(device) {
    DeviceGuard g(device);
    const size_t mm_words = 2 * (kMaxPeers + 1) * 2;
    BAGUA_CUDA_CHECK(cudaMalloc(&s_.minmax, mm_words * sizeof(uint32_t)));
    std::vector<uint32_t> init(mm_words);
    for (size_t i = 0; i < mm_words; ++i) init[i] = (i & 1) ? 0u : 0xffffffffu;  // [min-identity, max-identity] pairs
    BAGUA_CUDA_CHECK(cudaMemcpy(s_.minmax, init.data(), mm_words * sizeof(uint32_t), cudaMemcpyHostToDevice));
    BAGUA_CUDA_CHECK(cudaMalloc(&s_.grid_sync, 2 * sizeof(unsigned long long)));
    BAGUA_CUDA_CHECK(cudaMemset(s_.grid_sync, 0, 2 * sizeof(unsigned long long)));
    s_.reduced = nullptr;
    if (reduced_elems) BAGUA_CUDA_CHECK(cudaMalloc(&s_.reduced, reduced_elems * sizeof(float)));
    s_.host_state = host_state_;
}

QuantScratch::~QuantScratch() {
    if (s_.minmax) cudaFree(s_.minmax);
    if (s_.grid_sync) cudaFree(s_.grid_sync);
    if (s_.reduced) cudaFree(s_.reduced);
}

void AllReduceOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("allreduce");
    launch_allreduce(comm_->ctx(), src_.buf, dst_.buf, src_off_, dst_off_, bytes_, dtype_, scale_, variant_, cfg_.nblocks, cfg_.nthreads,
                     S(stream));
}

void AllReduceOneShotOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("allreduce_oneshot");
    launch_allreduce_oneshot(comm_->ctx(), staging_.buf, staging_off_, slot_bytes_, reinterpret_cast<const void*>(in_), reinterpret_cast<void*>(out_),
                             bytes_, dtype_, scale_, cfg_.nblocks, cfg_.nthreads, S(stream), comm_->next_oneshot_parity());
}

void ReduceScatterOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("reduce_scatter");
    launch_reduce_scatter(comm_->ctx(), buf_.buf, off_, bytes_, dtype_, scale_, use_mc_, cfg_.nblocks, cfg_.nthreads, S(stream));
}

void AllGatherOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("all_gather");
    launch_all_gather(comm_->ctx(), buf_.buf, off_, bytes_, dtype_, use_mc_, cfg_.nblocks, cfg_.nthreads, S(stream));
}

ShardGradOp::ShardGradOp(std::shared_ptr<PeerComm> comm, SymmBuf grads, size_t g_off, size_t bytes, int dtype, uint64_t shard, uint64_t partials,
                         float scale, bool zero_grads, bool use_multimem, LaunchCfg cfg, bool accumulate)
    : comm_(std::move(comm)), grads_(grads), g_off_(g_off), bytes_(bytes), dtype_(dtype), shard_(shard), partials_(partials), scale_(scale),
      zero_grads_(zero_grads), use_mc_(use_multimem), cfg_(cfg), accumulate_(accumulate) {
    if (accumulate_) {
        DeviceGuard g(comm_->device());
        preload_shard_grad_accum(dtype_, comm_->world(), use_mc_);
    }
}

void ShardGradOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("shard_grad");
    const bool add = accumulate_ && !fresh_.exchange(false, std::memory_order_acq_rel);
    launch_shard_grad(comm_->ctx(), grads_.buf, g_off_, bytes_, dtype_, reinterpret_cast<float*>(shard_), reinterpret_cast<double*>(partials_), scale_,
                      zero_grads_, use_mc_, cfg_.nblocks, cfg_.nthreads, S(stream), add);
}

void GradNormOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("grad_norm");
    launch_grad_norm(comm_->ctx(), box_.buf, box_off_, reinterpret_cast<const double*>(partials_), nslots_, reinterpret_cast<const double*>(extra_),
                     max_norm_, static_cast<uint32_t>(calls_ & 1u), reinterpret_cast<float*>(out_), S(stream));
    calls_++;
}

void LossScaleNormOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("loss_scale_norm");
    launch_loss_scale_norm(comm_->ctx(), box_.buf, box_off_, reinterpret_cast<const double*>(partials_), nslots_, reinterpret_cast<const double*>(extra_),
                           reinterpret_cast<const float*>(scale_), max_norm_, static_cast<uint32_t>(calls_ & 1u), reinterpret_cast<float*>(out_),
                           reinterpret_cast<uint32_t*>(step_), S(stream));
    calls_++;
}

void LambMomentsOp::run(Bucket&, StreamHandle stream, int) {
    launch_multi_tensor_lamb_stage1(desc_, F32, false, params(), coef_or_vote(coef_), reinterpret_cast<double*>(partials_), false, S(stream), dev_step());
    steps_++;
}

void LambRatioOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("lamb_ratio");
    launch_lamb_ratio(comm_->ctx(), box_.buf, box_off_, reinterpret_cast<const uint64_t*>(seg_ptr_), reinterpret_cast<const int32_t*>(seg_nblk_), nparams_,
                      static_cast<uint32_t>(calls_ & 1u), reinterpret_cast<float*>(ratio_), reinterpret_cast<double*>(sums_), S(stream));
    calls_++;
}

void LarsNormsOp::run(Bucket&, StreamHandle stream, int) {
    launch_multi_tensor_lars_stage1(desc_, F32, false, coef_or_vote(coef_), reinterpret_cast<double*>(partials_), S(stream), vote() != nullptr);
    steps_++;
}

template <class Rule>
void FusedUpdateOp<Rule>::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal(Rule::kFused);
    if (this->vote()) throw std::runtime_error(std::string("bagua: ") + Rule::kFused + " updates during backward and cannot obey a device-side vote or step count");
    launch_fused_update(comm_->ctx(), grads_.buf, weights_.buf, g_off_, w_off_, bytes_, dtype_, rule_, this->params(), scale_, zero_grads_, use_mc_,
                        cfg_.nblocks, cfg_.nthreads, S(stream));
    this->steps_++;
}
template class FusedUpdateOp<SgdRule>;
template class FusedUpdateOp<AdamRule>;
template class FusedUpdateOp<LionRule>;

template <class Rule>
void ShardUpdateOp<Rule>::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal(Rule::kShard);
    launch_shard_update(comm_->ctx(), weights_.buf, w_off_, bytes_, dtype_, reinterpret_cast<const float*>(shard_), this->coef_or_vote(coef_), rule_,
                        this->params(), use_mc_, cfg_.nblocks, cfg_.nthreads, S(stream), this->dev_step());
    this->steps_++;
}
template class ShardUpdateOp<SgdRule>;
template class ShardUpdateOp<AdamRule>;
template class ShardUpdateOp<LionRule>;
template class ShardUpdateOp<LambRule>;
template class ShardUpdateOp<LarsRule>;

void EmaOp::run(Bucket&, StreamHandle stream, int) { launch_multi_tensor_ema(desc_, weight(), reinterpret_cast<const float*>(vote_), S(stream)); }

ShardPublishOp::ShardPublishOp(std::shared_ptr<PeerComm> comm, SymmBuf weights, size_t w_off, size_t bytes, int dtype, uint64_t src, bool use_multimem,
                               LaunchCfg cfg)
    : comm_(std::move(comm)), weights_(weights), w_off_(w_off), bytes_(bytes), dtype_(dtype), src_(src), use_mc_(use_multimem), cfg_(cfg) {
    DeviceGuard g(comm_->device());
    preload_shard_publish(dtype_, comm_->world(), use_mc_);
}

void ShardPublishOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("shard_publish");
    launch_shard_publish(comm_->ctx(), weights_.buf, w_off_, bytes_, dtype_, reinterpret_cast<const float*>(src_), use_mc_, cfg_.nblocks, cfg_.nthreads,
                         S(stream));
}

int PeerAverageOp::shift_one_peer(int rank, int nranks, int64_t step) {
    const int64_t r = rank, n = nranks;
    if (rank < nranks / 2) return static_cast<int>(((step + r) % ((n + 1) / 2)) + (n / 2));
    int64_t v = (r - (n / 2) - step) % (n / 2);
    if (v < 0) v += n / 2;
    return static_cast<int>(v);
}

void PeerAverageOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("peer_average");
    const int n = comm_->world();
    if (n % 2 && n != 1) throw std::runtime_error("bagua: decentralized shift_one needs an even number of ranks, got " + std::to_string(n));
    const int peer = n == 1 ? 0 : shift_one_peer(comm_->rank(), n, step_);  // n == 1: self-peer mode, the partner is this GPU
    launch_peer_average(comm_->ctx(), weights_.buf, off_, peer, reinterpret_cast<void*>(out_), bytes_, dtype_, cfg_.nblocks, cfg_.nthreads,
                        S(stream));
    step_++;
}

ByteGradOp::ByteGradOp(std::shared_ptr<PeerComm> comm, uint64_t data, size_t numel, int dtype, SymmBuf inbox, size_t inbox_off,
                       SymmBuf outbox, size_t outbox_off, bool average, LaunchCfg cfg)
    : comm_(std::move(comm)), data_(data), numel_(numel), dtype_(dtype), inbox_(inbox), outbox_(outbox), inbox_off_(inbox_off),
      outbox_off_(outbox_off), average_(average), cfg_(cfg) {
    const int P = comm_->world();
    if (numel % (static_cast<size_t>(P) * 32)) throw std::invalid_argument("bagua: ByteGrad bucket must be padded to 32*nranks elements");
    cfg_.nblocks = std::max(P, cfg_.nblocks / P * P);
    scratch_ = std::make_unique<QuantScratch>(comm_->device(), numel / P);
}

void ByteGradOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("bytegrad");
    launch_bytegrad(comm_->ctx(), reinterpret_cast<void*>(data_), numel_, dtype_, inbox_.buf, inbox_off_, outbox_.buf, outbox_off_,
                    scratch_->get(), average_, cfg_.nblocks, cfg_.nthreads, S(stream), reinterpret_cast<const void*>(grad_), beta1_);
}

LowPrecRingOp::LowPrecRingOp(std::shared_ptr<PeerComm> comm, uint64_t x, uint64_t w, uint64_t l, uint64_t r, size_t numel, int dtype,
                             SymmBuf box, size_t box_off, LaunchCfg cfg)
    : comm_(std::move(comm)), x_(x), w_(w), l_(l), r_(r), numel_(numel), dtype_(dtype), box_(box), box_off_(box_off), cfg_(cfg) {
    if (numel % 32) throw std::invalid_argument("bagua: low-precision ring bucket must be padded to 32 elements");
    scratch_ = std::make_unique<QuantScratch>(comm_->device(), 0);
}

void LowPrecRingOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("lpdec_ring");
    const int n = comm_->world(), r = comm_->rank();
    launch_lpdec_ring(comm_->ctx(), reinterpret_cast<void*>(x_), reinterpret_cast<void*>(w_), reinterpret_cast<void*>(l_),
                      reinterpret_cast<void*>(r_), numel_, dtype_, box_.buf, box_off_, scratch_->get(), (r + n - 1) % n, (r + 1) % n,
                      cfg_.nblocks, cfg_.nthreads, S(stream));
}

WeightGate::WeightGate(int device) : device_(device) {
    DeviceGuard g(device);
    BAGUA_CUDA_CHECK(cudaMalloc(&words_, 8 * sizeof(uint32_t)));
    BAGUA_CUDA_CHECK(cudaMemset(words_, 0, 8 * sizeof(uint32_t)));
    preload_gate_kernels();
    BAGUA_CUDA_CHECK(cudaDeviceSynchronize());
}
WeightGate::~WeightGate() {
    if (words_) cudaFree(words_);
}
void WeightGate::acquire(StreamHandle stream, double timeout_s) {
    DeviceGuard g(device_);
    launch_gate_acquire(words_, static_cast<unsigned long long>(timeout_s * 1e9), S(stream));
}
void WeightGate::release(StreamHandle stream) {
    DeviceGuard g(device_);
    launch_gate_release(words_, S(stream));
}
uint32_t WeightGate::state() {
    DeviceGuard g(device_);
    uint32_t v = 0;
    BAGUA_CUDA_CHECK(cudaMemcpy(&v, words_, sizeof(v), cudaMemcpyDeviceToHost));
    return v;
}

AsyncAverageOp::AsyncAverageOp(std::shared_ptr<PeerComm> comm, uint64_t weights, SymmBuf snap, size_t snap_off, SymmBuf avg, size_t avg_off, size_t bytes,
                               int dtype, std::shared_ptr<WeightGate> gate, double gate_timeout_s, bool use_multimem, LaunchCfg cfg)
    : comm_(std::move(comm)), w_(weights), snap_(snap), avg_(avg), snap_off_(snap_off), avg_off_(avg_off), bytes_(bytes), dtype_(dtype),
      gate_(std::move(gate)), gate_timeout_s_(gate_timeout_s), use_mc_(use_multimem), cfg_(cfg) {
    DeviceGuard g(comm_->device());
    BAGUA_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&status_host_), sizeof(int), cudaHostAllocMapped));
    *status_host_ = 1;
    BAGUA_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&status_dev_), status_host_, 0));
}
AsyncAverageOp::~AsyncAverageOp() {
    if (status_host_) cudaFreeHost(status_host_);
}
void AsyncAverageOp::run(Bucket&, StreamHandle stream, int) {
    comm_->check_fatal("async_model_average");
    launch_async_average(comm_->ctx(), reinterpret_cast<void*>(w_), snap_.buf, snap_off_, avg_.buf, avg_off_, bytes_, dtype_, seq_ & 0x7fffffffu, go_.load(),
                         gate_ ? gate_->words() : nullptr, static_cast<unsigned long long>(gate_timeout_s_ * 1e9), status_dev_, use_mc_, cfg_.nblocks,
                         cfg_.nthreads, S(stream));
    seq_++;
}

void CopyOp::run(Bucket&, StreamHandle stream, int device) {
    if (device < 0) {  // CPU backend: plain host copy
        std::memcpy(reinterpret_cast<void*>(dst_), reinterpret_cast<const void*>(src_), bytes_);
        return;
    }
    BAGUA_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<void*>(dst_), reinterpret_cast<const void*>(src_), bytes_, cudaMemcpyDeviceToDevice,
                                     S(stream)));
}

}  // namespace bagua
