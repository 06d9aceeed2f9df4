// CommScheduler — the native bucket scheduler of bagua_b200.
//
// Capability parity with the reference's BaguaCommBackend (rust/bagua-core/bagua-core-internal/src/lib.rs:63-338):
// ordered buckets, strictly-in-order scheduling, one background comm worker per backend, a watchdog,
// duplicate detection at registration, waitable completion.
//
// H100-first differences:
//  * the worker never host-synchronises a stream (the reference blocks the worker per bucket with
//    cudaStreamSynchronize, datatypes/mod.rs:1110-1115). Ops are *launched* on the comm stream, a pooled
//    event is recorded behind them, and wait_pending_comm_ops() makes the consumer stream wait on that
//    event — the CPU runs ahead into optimizer.step() while the fused kernels are still in flight.
//  * tensors are raw {ptr, numel, dtype} records cached at registration; no GIL on the worker unless an
//    op is an explicit python callback.
//  * one event per *bucket* (recorded when its last tensor is marked) instead of one per tensor.
#pragma once
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "common.h"

// Forward declarations so this header does not need cuda_runtime.h.
struct CUstream_st;
struct CUevent_st;

namespace bagua {

using StreamHandle = CUstream_st*;
using EventHandle = CUevent_st*;

class Tensor {
public:
    Tensor(std::string name, uint64_t ptr, int64_t numel, int dtype, int device)
        : name_(std::move(name)), ptr_(ptr), numel_(numel), dtype_(dtype), device_(device) {}
    const std::string& name() const { return name_; }
    uint64_t data_ptr() const { return ptr_; }
    int64_t numel() const { return numel_; }
    int dtype() const { return dtype_; }
    int device() const { return device_; }
    size_t bytes() const { return static_cast<size_t>(numel_) * dtype_size(dtype_); }
    // Re-point the record (used when a bucket is re-flattened into another arena slice).
    void reset_ptr(uint64_t ptr) { ptr_ = ptr; }
    bool ready() const { return ready_.load(std::memory_order_acquire); }

private:
    friend class Bucket;
    friend class Backend;
    std::string name_;
    uint64_t ptr_;
    int64_t numel_;
    int dtype_;
    int device_;
    std::atomic<bool> ready_{false};
    EventHandle ready_event_ = nullptr;  // optional user-supplied event (reference-style API)
    bool always_ready_ = false;          // padding tensors
};

class Bucket;

// One step of a bucket's communication program.
class CommOp {
public:
    virtual ~CommOp() = default;
    virtual const char* kind() const = 0;
    // Launch (never host-block on GPU work) on `stream`. device < 0 ⇒ CPU mode.
    virtual void run(Bucket& bucket, StreamHandle stream, int device) = 0;
    // True for ops that may block the calling thread or need the GIL (python callbacks): never issued inline.
    virtual bool host_blocking() const { return false; }
    // False for ops whose launch arguments change from step to step (step counters, rotating peers): a CUDA graph would
    // freeze them, so such a bucket program must not be captured.
    virtual bool step_invariant() const { return true; }
};

class CallbackOp final : public CommOp {
public:
    using Fn = std::function<void(const std::string& bucket_name)>;
    explicit CallbackOp(Fn fn, std::string label = "python") : fn_(std::move(fn)), label_(std::move(label)) {}
    const char* kind() const override { return label_.c_str(); }
    void run(Bucket& bucket, StreamHandle, int) override;
    bool host_blocking() const override { return true; }

private:
    Fn fn_;
    std::string label_;
};

class Bucket {
public:
    Bucket(std::string name, std::vector<std::shared_ptr<Tensor>> tensors);
    const std::string& name() const { return name_; }
    const std::vector<std::shared_ptr<Tensor>>& tensors() const { return tensors_; }
    void append_op(std::shared_ptr<CommOp> op) { ops_.push_back(std::move(op)); }
    void clear_ops() { ops_.clear(); }
    const std::vector<std::shared_ptr<CommOp>>& ops() const { return ops_; }
    std::string describe_ops() const;
    bool ready_for_comm() const;
    void reset_comm_ready();
    // Contiguity: tensors laid out back to back (in order) in one allocation.
    bool contiguous() const { return contiguous_; }
    uint64_t flat_ptr() const { return flat_ptr_; }
    size_t bytes() const { return bytes_; }
    int64_t numel() const { return numel_; }
    int dtype() const { return dtype_; }
    int device() const { return device_; }
    void mark_padding(size_t index) { tensors_.at(index)->always_ready_ = true; }
    void recompute_layout();

private:
    friend class Backend;
    std::string name_;
    std::vector<std::shared_ptr<Tensor>> tensors_;
    std::vector<std::shared_ptr<CommOp>> ops_;
    bool contiguous_ = false;
    uint64_t flat_ptr_ = 0;
    size_t bytes_ = 0;
    int64_t numel_ = 0;
    int dtype_ = F32;
    int device_ = -1;
    // scheduling state (guarded by Backend::mu_)
    size_t pending_ = 0;
    StreamHandle producer_stream_ = nullptr;
    bool producer_stream_set_ = false;
    std::vector<EventHandle> user_events_;
};

// Per-bucket communication statistics (opt-in, Backend::set_profile): device time of the bucket's op list measured with
// a pair of timing events on the comm stream (host time on the CPU backend), plus the host-side queueing delay between
// "last tensor marked" and "ops issued". The reference has no equivalent (its speed metric is one number per iteration,
// data_parallel/bagua_distributed.py:113-131); these feed the per-bucket GB/s report and the autotuner.
struct BucketStat {
    std::string name;
    std::string ops;
    size_t bytes = 0;
    uint64_t count = 0;
    double total_ms = 0.0;
    double max_ms = 0.0;
    double queue_ms = 0.0;  // sum of (issue time − schedule time) on the host
};

// One execution of one bucket's op list on the communication stream (opt-in, Backend::set_timeline): when the host issued it
// (steady clock), when it began on the device relative to the moment the timeline was switched on, how long it ran there and
// how long it had waited in the host queue. This is the per-bucket timeline that says which bucket's communication is exposed
// after backward has ended (bagua_b200.utils.trace.export_chrome_trace puts it next to the tensor-ready marks).
struct BucketSample {
    std::string name;
    uint64_t iteration = 0;
    int64_t issue_ns = 0;      // steady clock, ns
    double start_ms = 0.0;     // device timeline (GPU backend) or host timeline (CPU backend), 0 = set_timeline(true)
    double device_ms = 0.0;
    double queue_ms = 0.0;
};

struct ReadySpan {
    std::string tensor_name;
    int64_t t_ns;     // steady clock, ns
    uint64_t iteration;
};

class Backend {
public:
    // channel_cap mirrors the reference's bounded channel (lib.rs:177). device_id < 0 ⇒ CPU backend.
    Backend(size_t channel_cap, int device_id, StreamHandle comm_stream, double watchdog_timeout_s = 300.0);
    ~Backend();
    Backend(const Backend&) = delete;

    void register_ordered_buckets(std::vector<std::shared_ptr<Bucket>> buckets);
    // Reference-style mark: optional raw event recorded by the caller on the producing stream.
    void mark_communication_ready(const std::shared_ptr<Tensor>& t, EventHandle ready_event);
    // Fast path: the backend records one pooled event on `producer` when the bucket completes.
    void mark_ready_on_stream(const std::shared_ptr<Tensor>& t, StreamHandle producer);
    // Host-waits until every scheduled bucket has been *issued*; then makes `consumer` wait for the
    // device-side completion (consumer == nullptr ⇒ host-synchronise, the reference behaviour).
    // Returns the number of buckets waited for. Rethrows worker errors.
    size_t wait_pending_comm_ops(StreamHandle consumer, bool host_sync);
    size_t pending_count();

    void set_watchdog_fatal(bool fatal) { watchdog_fatal_ = fatal; }
    std::string watchdog_error();
    std::vector<ReadySpan> pop_ready_spans();
    void set_record_spans(bool on) { record_spans_ = on; }
    void set_profile(bool on) { profile_ = on; }
    // Keep every resolved profile sample (bounded) for pop_bucket_timeline(); implies set_profile(on). On the GPU backend a
    // reference event is recorded on the comm stream so that every sample gets a device-time offset.
    void set_timeline(bool on);
    std::vector<BucketSample> pop_bucket_timeline();
    // Device time (ms) between the timeline's reference event and a caller's CUDA event (e.g. "backward ended" recorded on the
    // compute stream); -1 when the timeline is off, the event has not completed yet or this is the CPU backend.
    double timeline_ms_of_event(uint64_t cuda_event_ptr);
    int64_t timeline_ref_ns() const { return timeline_ref_ns_; }
    // Inline issue: a bucket whose program consists of native (asynchronously launching) ops only is issued by the thread
    // that marks its last tensor ready instead of being handed to the worker thread — no thread hand-off on the critical
    // path, and every CUDA call happens on the marking thread, which is what a stream capture (CUDA graph) needs. Order is
    // preserved: a bucket is issued inline only while the worker has nothing queued or in flight.
    void set_inline(bool on) { inline_ = on; }
    bool inline_mode() const { return inline_.load(); }
    // Every registered bucket consists of native ops with step-invariant launch arguments (or has no ops at all).
    bool graph_capturable();
    uint64_t inline_total() const { return inline_total_.load(); }
    // Folds every finished measurement into the table and returns it (non-blocking: kernels still running stay pending).
    std::vector<BucketStat> bucket_stats(bool reset = false);
    uint64_t scheduled_total() const { return scheduled_total_.load(); }
    int device_id() const { return device_; }
    StreamHandle comm_stream() const { return stream_; }
    void set_comm_stream(StreamHandle s) { stream_ = s; }
    void shutdown();

private:
    struct Ticket {
        std::shared_ptr<Bucket> bucket;
        std::vector<EventHandle> wait_events;   // comm stream waits on these before the ops
        std::vector<EventHandle> pooled_waits;  // subset of wait_events owned by the pool
        EventHandle done_event = nullptr;       // recorded on comm stream after the ops
        bool issued = false;
        bool failed = false;
        std::string error;
        std::chrono::steady_clock::time_point t_sched;
        uint64_t iteration = 0;                 // training iteration the bucket belongs to (copied under mu_)
    };

    void schedule_locked(std::unique_lock<std::mutex>& lk);
    void on_tensor_ready_locked(const std::shared_ptr<Tensor>& t, std::unique_lock<std::mutex>& lk);
    void worker_loop();
    void issue_ticket(const std::shared_ptr<Ticket>& tk);  // waits, ops, done event; never touches mu_
    void watchdog_loop();
    EventHandle acquire_event();
    void release_event(EventHandle e);

    size_t cap_;
    int device_;
    StreamHandle stream_;
    double timeout_s_;
    std::atomic<bool> watchdog_fatal_{true};
    std::atomic<bool> record_spans_{false};
    std::atomic<bool> profile_{false};
    std::atomic<bool> inline_{false};
    std::atomic<uint64_t> inline_total_{0};
    struct ProfSample {
        std::string name;
        EventHandle start = nullptr, stop = nullptr;  // GPU backend
        double host_ms = -1.0;                        // CPU backend
        double queue_ms = 0.0;
        int64_t issue_ns = 0;
        uint64_t iteration = 0;
    };
    std::atomic<bool> timeline_{false};
    bool profile_before_timeline_ = false;
    EventHandle timeline_ref_ = nullptr;              // GPU backend: recorded on the comm stream by set_timeline(true)
    int64_t timeline_ref_ns_ = 0;
    std::vector<BucketSample> timeline_samples_;      // guarded by prof_mu_, capped at kTimelineCap entries
    static constexpr size_t kTimelineCap = 1 << 16;
    std::mutex prof_mu_;
    std::deque<ProfSample> prof_pending_;
    std::vector<EventHandle> timing_pool_;
    std::unordered_map<std::string, BucketStat> prof_stats_;
    std::vector<std::string> prof_order_;
    EventHandle acquire_timing_event();

    std::mutex mu_;
    std::condition_variable cv_worker_;   // queue not empty / stop
    std::condition_variable cv_space_;    // queue has space
    std::condition_variable cv_done_;     // a ticket was issued
    std::condition_variable cv_watch_;    // watchdog tick / stop
    std::deque<std::shared_ptr<Bucket>> ordered_;
    std::unordered_map<const Tensor*, std::shared_ptr<Bucket>> owner_;
    std::deque<std::shared_ptr<Ticket>> queue_;
    std::deque<std::shared_ptr<Ticket>> not_waited_;
    std::shared_ptr<Ticket> in_flight_;
    std::vector<EventHandle> event_pool_;
    std::mutex pool_mu_;
    std::vector<ReadySpan> spans_;
    std::string watchdog_error_;
    std::atomic<uint64_t> scheduled_total_{0};
    uint64_t iteration_ = 0;            // complete passes over the registered bucket order (tags ready spans and timeline samples)
    const Bucket* first_bucket_ = nullptr;  // head of the registered order: the deque is back at it when a pass is complete
    bool stop_ = false;
    std::thread worker_;
    std::thread watchdog_;
};

}  // namespace bagua
