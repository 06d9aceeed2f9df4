// pybind11 face of the native core: module `bagua_b200._C`.
// Capability parity with the reference's PyO3 module bagua_core (rust/bagua-core/bagua-core-py/src/lib.rs:17-568):
// backend / tensor / bucket / communicator classes + direct kernel entry points. The GIL is released around every
// call that may block or take the scheduler lock (reference: lib.rs:374,388,396).
#include <pybind11/functional.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cuda_runtime.h>

#include "kernels.h"
#include "log.h"
#include "ops.h"
#include "scheduler.h"

namespace py = pybind11;
using namespace bagua;

namespace {
inline cudaStream_t S(uint64_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline StreamHandle SH(uint64_t s) { return reinterpret_cast<StreamHandle>(s); }
inline EventHandle EH(uint64_t e) { return reinterpret_cast<EventHandle>(e); }

// A python callable that can be destroyed from any thread.
std::shared_ptr<py::object> hold(py::object o) {
    return std::shared_ptr<py::object>(new py::object(std::move(o)), [](py::object* p) {
        if (Py_IsInitialized()) {
            py::gil_scoped_acquire g;
            delete p;
        }  // else: leak at interpreter teardown
    });
}

SgdParams make_sgd(float lr, float momentum, float dampening, float weight_decay, bool nesterov, bool first_step) {
    return SgdParams{lr, momentum, dampening, weight_decay, nesterov ? 1 : 0, first_step ? 1 : 0};
}
AdamParams make_adam(float lr, float b1, float b2, float eps, float wd, int step, bool adamw) {
    AdamParams p;
    p.lr = lr, p.beta1 = b1, p.beta2 = b2, p.eps = eps, p.weight_decay = wd;
    p.bias_correction1 = 1.f - std::pow(b1, static_cast<float>(step));
    p.bias_correction2 = 1.f - std::pow(b2, static_cast<float>(step));
    p.adamw = adamw ? 1 : 0;
    p.amsgrad = 0;
    return p;
}
}  // namespace

// Entry point for the optional torch extension (csrc/torch_hooks): marks a tensor ready without going through Python.
extern "C" __attribute__((visibility("default"))) void bagua_native_mark_ready(void* backend, void* tensor_handle, uint64_t stream) {
    auto* b = static_cast<bagua::Backend*>(backend);
    auto* t = static_cast<std::shared_ptr<bagua::Tensor>*>(tensor_handle);
    b->mark_ready_on_stream(*t, reinterpret_cast<bagua::StreamHandle>(stream));
}

PYBIND11_MODULE(_C, m) {
    m.doc() = "bagua_b200 native core (sm_90a)";
    m.def("nhwc_api_ptr", [] { return reinterpret_cast<uint64_t>(bagua_nhwc_api()); });
    m.def("native_mark_ready_fn", [] { return reinterpret_cast<uint64_t>(&bagua_native_mark_ready); });
    m.def("backend_raw_ptr", [](Backend& b) { return reinterpret_cast<uint64_t>(&b); });
    m.def("tensor_handle_new", [](std::shared_ptr<Tensor> t) { return reinterpret_cast<uint64_t>(new std::shared_ptr<Tensor>(std::move(t))); });
    m.def("tensor_handle_free", [](uint64_t h) { delete reinterpret_cast<std::shared_ptr<Tensor>*>(h); });
    m.def("log_level", [] { return std::string(bagua::log::name(bagua::log::threshold())); });
    m.def("set_log_level", [](const std::string& lvl) { bagua::log::threshold() = bagua::log::parse_level(lvl.c_str()); });
    m.attr("MAX_PEERS") = kMaxPeers;
    m.attr("MAX_COMM_BLOCKS") = kMaxCommBlocks;
    m.attr("AR_ONE_SHOT") = static_cast<int>(AR_ONE_SHOT);
    m.attr("AR_TWO_SHOT") = static_cast<int>(AR_TWO_SHOT);
    m.attr("AR_MULTIMEM") = static_cast<int>(AR_MULTIMEM);
    m.def("show_version", [] {
        int rt = 0;
        cudaRuntimeGetVersion(&rt);
        return std::string("bagua_b200 native core; target sm_90a; cuda runtime ") + std::to_string(rt);
    });
    m.def("launch_count", &launch_count);
    m.def("signal_pad_bytes", &PeerComm::signal_pad_bytes);
    m.def("minmax_uint8_chunk_bytes", &minmax_uint8_chunk_bytes);
    m.def("dtype_size", &dtype_size);

    py::class_<Tensor, std::shared_ptr<Tensor>>(m, "Tensor")
        .def(py::init<std::string, uint64_t, int64_t, int, int>(), py::arg("name"), py::arg("data_ptr"), py::arg("numel"), py::arg("dtype"),
             py::arg("device"))
        .def("name", &Tensor::name)
        .def("data_ptr", &Tensor::data_ptr)
        .def("num_elements", &Tensor::numel)
        .def("dtype", &Tensor::dtype)
        .def("device_id", &Tensor::device)
        .def("bytes", &Tensor::bytes)
        .def("ready", &Tensor::ready)
        .def("reset_ptr", &Tensor::reset_ptr);

    py::class_<CommOp, std::shared_ptr<CommOp>>(m, "CommOp").def("kind", [](CommOp& o) { return std::string(o.kind()); });

    py::class_<Bucket, std::shared_ptr<Bucket>>(m, "Bucket")
        .def(py::init<std::string, std::vector<std::shared_ptr<Tensor>>>(), py::arg("name"), py::arg("tensors"))
        .def("name", &Bucket::name)
        .def("tensors", &Bucket::tensors)
        .def("append_op", &Bucket::append_op)
        .def("append_python_op",
             [](Bucket& b, py::object fn, const std::string& label) {
                 auto held = hold(std::move(fn));
                 b.append_op(std::make_shared<CallbackOp>(
                     [held](const std::string& name) {
                         py::gil_scoped_acquire g;
                         (*held)(name);
                     },
                     label));
             },
             py::arg("fn"), py::arg("label") = "python")
        .def("clear_ops", &Bucket::clear_ops)
        .def("print_ops", &Bucket::describe_ops)
        .def("num_ops", [](Bucket& b) { return b.ops().size(); })
        .def("ready_for_comm", &Bucket::ready_for_comm)
        .def("reset_comm_ready", &Bucket::reset_comm_ready)
        .def("contiguous", &Bucket::contiguous)
        .def("flat_ptr", &Bucket::flat_ptr)
        .def("bytes", &Bucket::bytes)
        .def("numel", &Bucket::numel)
        .def("dtype", &Bucket::dtype)
        .def("mark_padding", &Bucket::mark_padding)
        .def("recompute_layout", &Bucket::recompute_layout);

    py::class_<Backend, std::shared_ptr<Backend>>(m, "Backend")
        .def(py::init([](size_t cap, int device, uint64_t stream, double timeout) {
                 return std::make_shared<Backend>(cap, device, SH(stream), timeout);
             }),
             py::arg("channel_cap") = 100, py::arg("device_id") = -1, py::arg("comm_stream") = 0, py::arg("watchdog_timeout_s") = 300.0)
        .def("register_ordered_buckets", &Backend::register_ordered_buckets, py::call_guard<py::gil_scoped_release>())
        .def("mark_communication_ready",
             [](Backend& b, const std::shared_ptr<Tensor>& t, uint64_t ev) { b.mark_communication_ready(t, EH(ev)); },
             py::arg("tensor"), py::arg("ready_event") = 0, py::call_guard<py::gil_scoped_release>())
        .def("mark_ready_on_stream",
             [](Backend& b, const std::shared_ptr<Tensor>& t, uint64_t stream) { b.mark_ready_on_stream(t, SH(stream)); },
             py::call_guard<py::gil_scoped_release>())
        .def("wait_pending_comm_ops",
             [](Backend& b, uint64_t consumer, bool host_sync) { return b.wait_pending_comm_ops(SH(consumer), host_sync); },
             py::arg("consumer_stream") = 0, py::arg("host_sync") = false, py::call_guard<py::gil_scoped_release>())
        .def("pending_count", &Backend::pending_count)
        .def("set_watchdog_fatal", &Backend::set_watchdog_fatal)
        .def("watchdog_error", &Backend::watchdog_error)
        .def("set_record_spans", &Backend::set_record_spans)
        .def("set_profile", &Backend::set_profile)
        .def("set_inline", &Backend::set_inline)
        .def("inline_mode", &Backend::inline_mode)
        .def("graph_capturable", &Backend::graph_capturable)
        .def("inline_total", &Backend::inline_total)
        .def("bucket_stats",
             [](Backend& b, bool reset) {
                 py::list out;
                 for (auto& s : b.bucket_stats(reset)) {
                     py::dict d;
                     d["name"] = s.name, d["ops"] = s.ops, d["bytes"] = s.bytes, d["count"] = s.count, d["total_ms"] = s.total_ms, d["max_ms"] = s.max_ms,
                     d["queue_ms"] = s.queue_ms;
                     out.append(d);
                 }
                 return out;
             },
             py::arg("reset") = false)
        .def("set_timeline", &Backend::set_timeline)
        .def("timeline_ms_of_event", &Backend::timeline_ms_of_event)
        .def("timeline_ref_ns", &Backend::timeline_ref_ns)
        .def("pop_bucket_timeline",
             [](Backend& b) {
                 py::list out;
                 for (auto& s : b.pop_bucket_timeline()) {
                     py::dict d;
                     d["bucket"] = s.name;
                     d["iteration"] = s.iteration;
                     d["issue_ns"] = s.issue_ns;
                     d["start_ms"] = s.start_ms;
                     d["device_ms"] = s.device_ms;
                     d["queue_ms"] = s.queue_ms;
                     out.append(d);
                 }
                 return out;
             })
        .def("pop_ready_spans",
             [](Backend& b) {
                 py::list out;
                 for (auto& s : b.pop_ready_spans()) out.append(py::make_tuple(s.tensor_name, s.t_ns, s.iteration));
                 return out;
             })
        .def("scheduled_total", &Backend::scheduled_total)
        .def("device_id", &Backend::device_id)
        .def("set_comm_stream", [](Backend& b, uint64_t s) { b.set_comm_stream(SH(s)); })
        .def("shutdown", &Backend::shutdown, py::call_guard<py::gil_scoped_release>());

    py::class_<PeerComm, std::shared_ptr<PeerComm>>(m, "PeerComm")
        .def(py::init<int, int, int, const std::vector<uint64_t>&, double>(), py::arg("rank"), py::arg("world"), py::arg("device"),
             py::arg("flag_ptrs"), py::arg("timeout_s") = 300.0)
        .def("rank", &PeerComm::rank)
        .def("nranks", &PeerComm::world)
        .def("device_id", &PeerComm::device)
        .def("abort", &PeerComm::abort)
        .def("reset_abort", &PeerComm::reset_abort)
        .def("check_abort", &PeerComm::aborted)
        .def("error_code", &PeerComm::error_code)
        .def("host_error", &PeerComm::host_error)
        .def("check_fatal", [](PeerComm& c, const std::string& what) { c.check_fatal(what.c_str()); }, py::arg("what") = "the next collective")
        .def("clear_error", &PeerComm::clear_error)
        .def("set_timeout", &PeerComm::set_timeout)
        .def("barrier", [](PeerComm& c, uint64_t stream) { launch_peer_barrier(c.ctx(), S(stream)); });

    py::class_<SymmBuf>(m, "SymmBuf")
        .def(py::init<const std::vector<uint64_t>&, uint64_t, size_t>(), py::arg("ptrs"), py::arg("multicast_ptr") = 0, py::arg("bytes") = 0)
        .def("has_multicast", &SymmBuf::has_multicast)
        .def_readonly("bytes", &SymmBuf::bytes);

    py::class_<LaunchCfg>(m, "LaunchCfg")
        .def(py::init([](int nb, int nt) {
                 LaunchCfg c;
                 c.nblocks = nb, c.nthreads = nt;
                 return c;
             }),
             py::arg("nblocks") = 32, py::arg("nthreads") = 512)
        .def_readwrite("nblocks", &LaunchCfg::nblocks)
        .def_readwrite("nthreads", &LaunchCfg::nthreads);

    py::class_<AllReduceOp, CommOp, std::shared_ptr<AllReduceOp>>(m, "AllReduceOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, SymmBuf, size_t, size_t, size_t, int, float, int, LaunchCfg>(), py::arg("comm"),
             py::arg("src"), py::arg("dst"), py::arg("src_off"), py::arg("dst_off"), py::arg("bytes"), py::arg("dtype"), py::arg("scale"),
             py::arg("variant"), py::arg("cfg"))
        .def("set_variant", &AllReduceOp::set_variant);
    py::class_<AllReduceOneShotOp, CommOp, std::shared_ptr<AllReduceOneShotOp>>(m, "AllReduceOneShotOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, size_t, size_t, uint64_t, uint64_t, size_t, int, float, LaunchCfg>(), py::arg("comm"),
             py::arg("staging"), py::arg("staging_off"), py::arg("slot_bytes"), py::arg("in_ptr"), py::arg("out_ptr"), py::arg("bytes"), py::arg("dtype"),
             py::arg("scale"), py::arg("cfg"));
    py::class_<AllReduceSgdOp, CommOp, std::shared_ptr<AllReduceSgdOp>>(m, "AllReduceSgdOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, SymmBuf, size_t, size_t, size_t, int, uint64_t, uint64_t, float, bool, bool,
                      LaunchCfg>(),
             py::arg("comm"), py::arg("grads"), py::arg("weights"), py::arg("g_off"), py::arg("w_off"), py::arg("bytes"), py::arg("dtype"),
             py::arg("master_ptr"), py::arg("momentum_ptr"), py::arg("scale"), py::arg("zero_grads"), py::arg("use_multimem"), py::arg("cfg"))
        .def("set_hyper", &AllReduceSgdOp::set_hyper)
        .def("set_grad_scale", &AllReduceSgdOp::set_grad_scale)
        .def("steps", &AllReduceSgdOp::steps)
        .def("set_steps", &AllReduceSgdOp::set_steps);
    py::class_<ReduceScatterOp, CommOp, std::shared_ptr<ReduceScatterOp>>(m, "ReduceScatterOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, size_t, size_t, int, float, bool, LaunchCfg>(), py::arg("comm"), py::arg("buf"), py::arg("off"),
             py::arg("bytes"), py::arg("dtype"), py::arg("scale"), py::arg("use_multimem"), py::arg("cfg"));
    py::class_<AllGatherOp, CommOp, std::shared_ptr<AllGatherOp>>(m, "AllGatherOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, size_t, size_t, int, bool, LaunchCfg>(), py::arg("comm"), py::arg("buf"), py::arg("off"),
             py::arg("bytes"), py::arg("dtype"), py::arg("use_multimem"), py::arg("cfg"));
    py::class_<AllReduceAdamOp, CommOp, std::shared_ptr<AllReduceAdamOp>>(m, "AllReduceAdamOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, SymmBuf, size_t, size_t, size_t, int, uint64_t, uint64_t, uint64_t, float, bool, bool,
                      LaunchCfg>(),
             py::arg("comm"), py::arg("grads"), py::arg("weights"), py::arg("g_off"), py::arg("w_off"), py::arg("bytes"), py::arg("dtype"),
             py::arg("master_ptr"), py::arg("exp_avg_ptr"), py::arg("exp_avg_sq_ptr"), py::arg("scale"), py::arg("zero_grads"), py::arg("use_multimem"),
             py::arg("cfg"))
        .def("set_hyper", &AllReduceAdamOp::set_hyper)
        .def("set_grad_scale", &AllReduceAdamOp::set_grad_scale)
        .def("steps", &AllReduceAdamOp::steps)
        .def("set_steps", &AllReduceAdamOp::set_steps);
    py::class_<PeerAverageOp, CommOp, std::shared_ptr<PeerAverageOp>>(m, "PeerAverageOp")
        .def(py::init<std::shared_ptr<PeerComm>, SymmBuf, size_t, uint64_t, size_t, int, LaunchCfg>(), py::arg("comm"), py::arg("weights"),
             py::arg("off"), py::arg("out_ptr"), py::arg("bytes"), py::arg("dtype"), py::arg("cfg"))
        .def("step", &PeerAverageOp::step)
        .def_static("shift_one_peer", &PeerAverageOp::shift_one_peer);
    py::class_<ByteGradOp, CommOp, std::shared_ptr<ByteGradOp>>(m, "ByteGradOp")
        .def(py::init<std::shared_ptr<PeerComm>, uint64_t, size_t, int, SymmBuf, size_t, SymmBuf, size_t, bool, LaunchCfg>(), py::arg("comm"),
             py::arg("data_ptr"), py::arg("numel"), py::arg("dtype"), py::arg("inbox"), py::arg("inbox_off"), py::arg("outbox"),
             py::arg("outbox_off"), py::arg("average"), py::arg("cfg"))
        .def("set_momentum_source", &ByteGradOp::set_momentum_source, py::arg("grad_ptr"), py::arg("beta1"))
        .def_static("box_bytes", &ByteGradOp::box_bytes);
    py::class_<WeightGate, std::shared_ptr<WeightGate>>(m, "WeightGate")
        .def(py::init<int>(), py::arg("device"))
        .def("acquire", [](WeightGate& g, uint64_t stream, double timeout_s) { g.acquire(SH(stream), timeout_s); }, py::arg("stream"), py::arg("timeout_s") = 10.0)
        .def("release", [](WeightGate& g, uint64_t stream) { g.release(SH(stream)); })
        .def("state", &WeightGate::state);
    py::class_<AsyncAverageOp, CommOp, std::shared_ptr<AsyncAverageOp>>(m, "AsyncAverageOp")
        .def(py::init<std::shared_ptr<PeerComm>, uint64_t, SymmBuf, size_t, SymmBuf, size_t, size_t, int, std::shared_ptr<WeightGate>, double, bool, LaunchCfg>(),
             py::arg("comm"), py::arg("weights_ptr"), py::arg("snap"), py::arg("snap_off"), py::arg("avg"), py::arg("avg_off"), py::arg("bytes"), py::arg("dtype"),
             py::arg("gate"), py::arg("gate_timeout_s"), py::arg("use_multimem"), py::arg("cfg"))
        .def("abort", &AsyncAverageOp::abort)
        .def("reset", &AsyncAverageOp::reset)
        .def("status", &AsyncAverageOp::status)
        .def("rounds", &AsyncAverageOp::rounds);
    py::class_<LowPrecRingOp, CommOp, std::shared_ptr<LowPrecRingOp>>(m, "LowPrecRingOp")
        .def(py::init<std::shared_ptr<PeerComm>, uint64_t, uint64_t, uint64_t, uint64_t, size_t, int, SymmBuf, size_t, LaunchCfg>(),
             py::arg("comm"), py::arg("x_ptr"), py::arg("w_ptr"), py::arg("l_ptr"), py::arg("r_ptr"), py::arg("numel"), py::arg("dtype"),
             py::arg("box"), py::arg("box_off"), py::arg("cfg"))
        .def_static("box_bytes", &LowPrecRingOp::box_bytes);
    py::class_<CopyOp, CommOp, std::shared_ptr<CopyOp>>(m, "CopyOp").def(py::init<uint64_t, uint64_t, size_t>());

    // Run a native op immediately on a stream (no scheduler) — used by blocking collectives and tests.
    m.def(
        "run_op",
        [](std::shared_ptr<CommOp> op, uint64_t stream, int device) {
            static auto dummy_tensor = std::make_shared<Tensor>("__run_op__", 0, 0, F32, -1);
            static Bucket dummy("__run_op__", {dummy_tensor});
            op->run(dummy, SH(stream), device);
        },
        py::arg("op"), py::arg("stream"), py::arg("device"), py::call_guard<py::gil_scoped_release>());

    // ---- direct kernel entry points (raw pointers; callers keep the tensors alive) ----------------------------
    m.def("flat_sgd",
          [](uint64_t param, int pdt, uint64_t grad, int gdt, uint64_t mom, uint64_t model, int mdt, size_t n, float lr, float momentum,
             float dampening, float wd, bool nesterov, bool first_step, float grad_scale, bool zero_grad, uint64_t stream) {
              launch_flat_sgd(reinterpret_cast<void*>(param), pdt, reinterpret_cast<const void*>(grad), gdt, reinterpret_cast<float*>(mom),
                              reinterpret_cast<void*>(model), mdt, n, make_sgd(lr, momentum, dampening, wd, nesterov, first_step),
                              grad_scale, zero_grad, S(stream));
          });
    m.def("flat_adam",
          [](uint64_t param, int pdt, uint64_t grad, int gdt, uint64_t m1, uint64_t m2, uint64_t model, int mdt, size_t n, float lr, float b1,
             float b2, float eps, float wd, int step, bool adamw, float grad_scale, bool zero_grad, uint64_t stream) {
              launch_flat_adam(reinterpret_cast<void*>(param), pdt, reinterpret_cast<const void*>(grad), gdt, reinterpret_cast<float*>(m1),
                               reinterpret_cast<float*>(m2), reinterpret_cast<void*>(model), mdt, n, make_adam(lr, b1, b2, eps, wd, step, adamw),
                               grad_scale, zero_grad, S(stream));
          });
    m.def("multi_tensor_sgd",
          [](uint64_t ptrs, uint64_t sizes, uint64_t b2t, uint64_t b2c, int n_tensors, int n_blocks, int chunk, int dtype, bool has_mom,
             float lr, float momentum, float dampening, float wd, bool nesterov, bool first_step, float grad_scale, uint64_t stream) {
              TensorListDesc d{reinterpret_cast<const uint64_t*>(ptrs), reinterpret_cast<const int64_t*>(sizes),
                               reinterpret_cast<const int32_t*>(b2t), reinterpret_cast<const int32_t*>(b2c), n_tensors, n_blocks, chunk};
              launch_multi_tensor_sgd(d, dtype, has_mom, make_sgd(lr, momentum, dampening, wd, nesterov, first_step), grad_scale, S(stream));
          });
    m.def("multi_tensor_adam",
          [](uint64_t ptrs, uint64_t sizes, uint64_t b2t, uint64_t b2c, int n_tensors, int n_blocks, int chunk, int dtype, float lr, float b1,
             float b2, float eps, float wd, int step, bool adamw, float grad_scale, uint64_t stream) {
              TensorListDesc d{reinterpret_cast<const uint64_t*>(ptrs), reinterpret_cast<const int64_t*>(sizes),
                               reinterpret_cast<const int32_t*>(b2t), reinterpret_cast<const int32_t*>(b2c), n_tensors, n_blocks, chunk};
              launch_multi_tensor_adam(d, dtype, make_adam(lr, b1, b2, eps, wd, step, adamw), grad_scale, S(stream));
          });
    m.def("multi_tensor_adam_mp",
          [](uint64_t ptrs, uint64_t sizes, uint64_t b2t, uint64_t b2c, int n_tensors, int n_blocks, int chunk, int dtype, float lr, float b1,
             float b2, float eps, float wd, int step, bool adamw, float grad_scale, uint64_t stream) {
              TensorListDesc d{reinterpret_cast<const uint64_t*>(ptrs), reinterpret_cast<const int64_t*>(sizes),
                               reinterpret_cast<const int32_t*>(b2t), reinterpret_cast<const int32_t*>(b2c), n_tensors, n_blocks, chunk};
              launch_multi_tensor_adam_mp(d, dtype, make_adam(lr, b1, b2, eps, wd, step, adamw), grad_scale, S(stream));
          });
    m.def("qadam_momentum", [](uint64_t m1, uint64_t grad, int gdt, size_t n, float beta1, uint64_t stream) {
        launch_qadam_momentum(reinterpret_cast<float*>(m1), reinterpret_cast<const void*>(grad), gdt, n, beta1, S(stream));
    });
    m.def("bias_relu_nhwc_fwd", [](uint64_t y, uint64_t bias, size_t rows, int C, int dtype, uint64_t stream) {
        launch_bias_relu_nhwc_fwd(reinterpret_cast<void*>(y), reinterpret_cast<const void*>(bias), rows, C, dtype, S(stream));
    });
    m.def("bias_relu_nhwc_bwd", [](uint64_t g, uint64_t y, uint64_t gout, uint64_t bias_grad, size_t rows, int C, int dtype, uint64_t stream) {
        launch_bias_relu_nhwc_bwd(reinterpret_cast<const void*>(g), reinterpret_cast<const void*>(y), reinterpret_cast<void*>(gout),
                                  reinterpret_cast<float*>(bias_grad), rows, C, dtype, S(stream));
    });
    m.def("bias_relu_nhwc_bwd_fin",
          [](uint64_t g, uint64_t y, uint64_t gout, uint64_t ws, uint64_t bias_grad_out, uint64_t ticket, size_t rows, int C, int dtype, uint64_t stream) {
              launch_bias_relu_nhwc_bwd(reinterpret_cast<const void*>(g), reinterpret_cast<const void*>(y), reinterpret_cast<void*>(gout),
                                        reinterpret_cast<float*>(ws), rows, C, dtype, S(stream), reinterpret_cast<void*>(bias_grad_out),
                                        reinterpret_cast<unsigned int*>(ticket));
          });
    m.def("bias_relu_pool_nhwc_bwd_fin",
          [](uint64_t g, uint64_t out, uint64_t idx, uint64_t gin, uint64_t ws, uint64_t bias_grad_out, uint64_t ticket, int N, int H, int W, int C, int dtype,
             uint64_t stream) {
              launch_bias_relu_pool_nhwc_bwd(reinterpret_cast<const void*>(g), reinterpret_cast<const void*>(out), reinterpret_cast<const uint8_t*>(idx),
                                             reinterpret_cast<void*>(gin), reinterpret_cast<float*>(ws), N, H, W, C, dtype, S(stream),
                                             reinterpret_cast<void*>(bias_grad_out), reinterpret_cast<unsigned int*>(ticket));
          });
    m.def("bias_relu_pool_nhwc_fwd", [](uint64_t x, uint64_t bias, uint64_t out, uint64_t idx, int N, int H, int W, int C, int dtype, uint64_t stream) {
        launch_bias_relu_pool_nhwc_fwd(reinterpret_cast<const void*>(x), reinterpret_cast<const void*>(bias), reinterpret_cast<void*>(out),
                                       reinterpret_cast<uint8_t*>(idx), N, H, W, C, dtype, S(stream));
    });
    m.def("bias_relu_pool_nhwc_bwd",
          [](uint64_t g, uint64_t out, uint64_t idx, uint64_t gin, uint64_t bias_grad, int N, int H, int W, int C, int dtype, uint64_t stream) {
              launch_bias_relu_pool_nhwc_bwd(reinterpret_cast<const void*>(g), reinterpret_cast<const void*>(out), reinterpret_cast<const uint8_t*>(idx),
                                             reinterpret_cast<void*>(gin), reinterpret_cast<float*>(bias_grad), N, H, W, C, dtype, S(stream));
          });
    m.def("grouped_gemm_supported", &grouped_gemm_supported);
    m.def("grouped_gemm_tn", [](uint64_t A, uint64_t B, uint64_t C, uint64_t bias, int G, int M, int N, int K, int act, uint64_t stream) {
        launch_grouped_gemm_tn(reinterpret_cast<const void*>(A), reinterpret_cast<const void*>(B), reinterpret_cast<void*>(C),
                               reinterpret_cast<const float*>(bias), G, M, N, K, act, S(stream));
    });
    m.def("grouped_gemm_tn_push",
          [](uint64_t A, uint64_t B, uint64_t bias, int G, int N, int K, int act, std::shared_ptr<PeerComm> comm, SymmBuf out, size_t out_off, int cap,
             uint64_t stream) {
              launch_grouped_gemm_tn_push(reinterpret_cast<const void*>(A), reinterpret_cast<const void*>(B), reinterpret_cast<const float*>(bias), G, N, K,
                                          act, comm->ctx(), out.buf, out_off, cap, S(stream));
          });
    m.def("moe_scatter",
          [](std::shared_ptr<PeerComm> comm, SymmBuf dst, size_t dst_off, uint64_t rows, uint64_t eidx, uint64_t sidx, uint64_t scale, int n_tok, int K,
             int M, int E_local, int C, int dtype, int nblocks, uint64_t stream) {
              launch_moe_scatter(comm->ctx(), dst.buf, dst_off, reinterpret_cast<const void*>(rows), reinterpret_cast<const int64_t*>(eidx),
                                 reinterpret_cast<const int64_t*>(sidx), reinterpret_cast<const float*>(scale), n_tok, K, M, E_local, C, dtype, nblocks,
                                 S(stream));
          });
    m.def("moe_gather",
          [](std::shared_ptr<PeerComm> comm, SymmBuf src, size_t src_off, uint64_t out, uint64_t eidx, uint64_t sidx, uint64_t weights, uint64_t picked,
             int n_tok, int K, int M, int E_local, int C, int dtype, int nblocks, uint64_t stream, bool local_layout) {
              launch_moe_gather(comm->ctx(), src.buf, src_off, reinterpret_cast<void*>(out), reinterpret_cast<const int64_t*>(eidx),
                                reinterpret_cast<const int64_t*>(sidx), reinterpret_cast<const float*>(weights), reinterpret_cast<void*>(picked), n_tok, K, M,
                                E_local, C, dtype, nblocks, S(stream), local_layout);
          },
          py::arg("comm"), py::arg("src"), py::arg("src_off"), py::arg("out"), py::arg("eidx"), py::arg("sidx"), py::arg("weights"), py::arg("picked"),
          py::arg("n_tok"), py::arg("K"), py::arg("M"), py::arg("E_local"), py::arg("C"), py::arg("dtype"), py::arg("nblocks"), py::arg("stream"),
          py::arg("local_layout") = false);
    m.def("minmax_uint8_compress",
          [](uint64_t in, size_t numel, int dtype, int n_chunks, int target_chunk, uint64_t out, uint64_t scratch, uint64_t stream) {
              launch_minmax_uint8_compress(reinterpret_cast<const void*>(in), numel, dtype, n_chunks, target_chunk,
                                           reinterpret_cast<uint8_t*>(out), reinterpret_cast<float*>(scratch), S(stream));
          });
    m.def("minmax_uint8_decompress", [](uint64_t in, size_t numel, int dtype, int n_chunks, uint64_t out, uint64_t stream) {
        launch_minmax_uint8_decompress(reinterpret_cast<const uint8_t*>(in), numel, dtype, n_chunks, reinterpret_cast<void*>(out), S(stream));
    });
    m.def("async_apply", [](uint64_t w, uint64_t red, uint64_t snap, size_t n, int dtype, float inv_p, uint64_t stream) {
        launch_async_apply(reinterpret_cast<void*>(w), reinterpret_cast<const void*>(red), reinterpret_cast<const void*>(snap), n, dtype, inv_p,
                           S(stream));
    });
    m.def("reduce_chunks", [](uint64_t data, size_t chunk, int n_chunks, int target, int dtype, bool average, uint64_t stream) {
        launch_reduce_chunks(reinterpret_cast<void*>(data), chunk, n_chunks, target, dtype, average, S(stream));
    });
    m.def("axpby", [](uint64_t x, uint64_t y, size_t n, int dtype, float a, float b, uint64_t stream) {
        launch_axpby(reinterpret_cast<void*>(x), reinterpret_cast<const void*>(y), n, dtype, a, b, S(stream));
    });
    m.def("scale", [](uint64_t x, size_t n, int dtype, float a, uint64_t stream) {
        launch_scale(reinterpret_cast<void*>(x), n, dtype, a, S(stream));
    });
    m.def("cast", [](uint64_t in, int idt, uint64_t out, int odt, size_t n, uint64_t stream) {
        launch_cast(reinterpret_cast<const void*>(in), idt, reinterpret_cast<void*>(out), odt, n, S(stream));
    });
}
