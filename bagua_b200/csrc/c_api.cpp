#include "c_api.h"

#include <memory>
#include <string>
#include <vector>

#include "ops.h"
#include "scheduler.h"

using namespace bagua;

struct BaguaTensorC {
    std::shared_ptr<Tensor> inner;
};
struct BaguaBucketC {
    std::shared_ptr<Bucket> inner;
};
struct BaguaBackendC {
    std::shared_ptr<Backend> inner;
};
struct BaguaPeerCommC {
    std::shared_ptr<PeerComm> inner;
};

namespace {
thread_local std::string g_last_error;
template <typename F>
int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& e) {
        g_last_error = e.what();
        return -1;
    } catch (...) {
        g_last_error = "unknown error";
        return -2;
    }
}
}  // namespace

extern "C" {

const char* bagua_last_error(void) { return g_last_error.c_str(); }
const char* bagua_version(void) { return "bagua_b200 native core (sm_90a)"; }

BaguaTensorC* bagua_tensor_c_create(const char* name, uint64_t data_ptr, int64_t num_elements, int dtype, int device_id) {
    BaguaTensorC* out = nullptr;
    guarded([&] {
        dtype_size(dtype);  // validates the code
        out = new BaguaTensorC{std::make_shared<Tensor>(name ? name : "", data_ptr, num_elements, dtype, device_id)};
    });
    return out;
}
void bagua_tensor_c_destroy(BaguaTensorC** t) {
    if (t && *t) {
        delete *t;
        *t = nullptr;
    }
}

BaguaBucketC* bagua_bucket_c_create(BaguaTensorC* const* tensors, size_t n, const char* name) {
    BaguaBucketC* out = nullptr;
    guarded([&] {
        std::vector<std::shared_ptr<Tensor>> v;
        for (size_t i = 0; i < n; ++i) v.push_back(tensors[i]->inner);
        out = new BaguaBucketC{std::make_shared<Bucket>(name ? name : "", std::move(v))};
    });
    return out;
}
void bagua_bucket_c_destroy(BaguaBucketC** b) {
    if (b && *b) {
        delete *b;
        *b = nullptr;
    }
}
int bagua_bucket_c_append_callback_op(BaguaBucketC* bucket, bagua_callback_t fn, void* user_data) {
    return guarded([&] {
        bucket->inner->append_op(std::make_shared<CallbackOp>([fn, user_data](const std::string& name) { fn(name.c_str(), user_data); }, "c_callback"));
    });
}
int bagua_bucket_c_clear_ops(BaguaBucketC* bucket) {
    return guarded([&] { bucket->inner->clear_ops(); });
}

BaguaPeerCommC* bagua_peer_comm_c_create(int rank, int nranks, int device_id, const uint64_t* flag_ptrs, double timeout_s) {
    BaguaPeerCommC* out = nullptr;
    guarded([&] {
        std::vector<uint64_t> flags(flag_ptrs, flag_ptrs + nranks);
        out = new BaguaPeerCommC{std::make_shared<PeerComm>(rank, nranks, device_id, flags, timeout_s)};
    });
    return out;
}
void bagua_peer_comm_c_destroy(BaguaPeerCommC** c) {
    if (c && *c) {
        delete *c;
        *c = nullptr;
    }
}
int bagua_peer_comm_c_abort(BaguaPeerCommC* comm) {
    return guarded([&] { comm->inner->abort(); });
}
size_t bagua_peer_comm_c_signal_pad_bytes(void) { return PeerComm::signal_pad_bytes(); }

int bagua_bucket_c_append_centralized_synchronous_op(BaguaBucketC* bucket, BaguaPeerCommC* comm, const uint64_t* peer_ptrs, uint64_t mc_ptr, size_t offset,
                                                     size_t bytes, int dtype, int average, int variant, int nblocks) {
    return guarded([&] {
        const int n = comm->inner->world();
        SymmBuf buf(std::vector<uint64_t>(peer_ptrs, peer_ptrs + n), mc_ptr, offset + bytes);
        LaunchCfg cfg;
        cfg.nblocks = nblocks > 0 ? nblocks : 32;
        bucket->inner->append_op(
            std::make_shared<AllReduceOp>(comm->inner, buf, buf, offset, offset, bytes, dtype, average ? 1.0f / n : 1.0f, variant, cfg));
    });
}

BaguaBackendC* bagua_comm_backend_c_create(size_t cap, int device_id, uint64_t comm_stream, double timeout_s) {
    BaguaBackendC* out = nullptr;
    guarded([&] { out = new BaguaBackendC{std::make_shared<Backend>(cap, device_id, reinterpret_cast<StreamHandle>(comm_stream), timeout_s)}; });
    return out;
}
void bagua_comm_backend_c_destroy(BaguaBackendC** b) {
    if (b && *b) {
        (*b)->inner->shutdown();
        delete *b;
        *b = nullptr;
    }
}
int bagua_comm_backend_c_register_ordered_buckets(BaguaBackendC* backend, BaguaBucketC* const* buckets, size_t n) {
    return guarded([&] {
        std::vector<std::shared_ptr<Bucket>> v;
        for (size_t i = 0; i < n; ++i) v.push_back(buckets[i]->inner);
        backend->inner->register_ordered_buckets(std::move(v));
    });
}
int bagua_comm_backend_c_mark_communication_ready(BaguaBackendC* backend, BaguaTensorC* tensor, uint64_t ready_cuda_event) {
    return guarded([&] { backend->inner->mark_communication_ready(tensor->inner, reinterpret_cast<EventHandle>(ready_cuda_event)); });
}
int bagua_comm_backend_c_wait_pending_comm_ops(BaguaBackendC* backend, uint64_t consumer_stream, int host_sync) {
    return guarded([&] { backend->inner->wait_pending_comm_ops(reinterpret_cast<StreamHandle>(consumer_stream), host_sync != 0); });
}

}  // extern "C"
