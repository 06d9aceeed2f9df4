// bagua_b200 native core — shared definitions.
//
// Torch-free on purpose: the runtime sees raw device pointers, element counts, dtype codes and
// raw CUDA stream/event handles. Python (or the C ABI) caches them once at registration time, so
// the comm worker never needs the GIL to look at a tensor (the reference re-enters Python for every
// data_ptr()/numel() call from its worker thread, rust/bagua-core/bagua-core-internal/src/datatypes/mod.rs:603-676).
#pragma once
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

namespace bagua {

// dtype codes shared with python (bagua_b200/define.py). bf16 is new w.r.t. the reference
// (rust/bagua-core/bagua-core-internal/src/datatypes/mod.rs:42-48 only knows f32/f16/u8/i64).
enum DType : int { F32 = 0, F16 = 1, U8 = 2, I64 = 3, BF16 = 4 };

inline size_t dtype_size(int dt) {
    switch (dt) {
        case F32: return 4;
        case F16: return 2;
        case U8: return 1;
        case I64: return 8;
        case BF16: return 2;
        default: throw std::runtime_error("bagua: unknown dtype code " + std::to_string(dt));
    }
}

// Reduction op codes — same numbering as the reference's ReduceOp (bagua/torch_api/communication.py:64-75).
enum RedOp : int { SUM = 0, PRODUCT = 1, MIN = 2, MAX = 3, BOR = 7, BAND = 8, BXOR = 9, AVG = 10 };

constexpr int kMaxPeers = 8;        // one NVSwitch domain (HGX H100 = 8 GPUs)
constexpr int kMaxCommBlocks = 256;  // upper bound on CTAs of any peer kernel (flag slots per block)
constexpr int kFlagStride = kMaxPeers;
// Behind the barrier flags every signal pad carries a small "vote" area: slot [s] is written by rank s (all of its CTAs write
// the same word) just before a barrier and read by the owner just after it — an all-to-all of one word riding on the barrier
// (used by async_average_kernel to agree on abort without a separate collective).
constexpr int kVoteWordOffset = kMaxCommBlocks * kMaxPeers;  // in uint32 words from the start of the pad
constexpr int kVoteWords = 64;

// Everything a peer kernel needs to talk to the other GPUs of its group.
// flags[p] points at rank p's signal pad: uint32 [kMaxCommBlocks][kMaxPeers]; slot [b][s] is written
// only by block b of rank s, with monotonically increasing epochs, so it never needs a reset.
struct PeerCtx {
    uint32_t* flags[kMaxPeers];
    uint32_t* epochs;        // local, private: uint32 [kMaxCommBlocks] — last epoch used by block b
    volatile int* abort;     // host-mapped flag; non-zero → spinning kernels bail out
    int* error;              // local device int; set to non-zero by a kernel that timed out / aborted
    volatile int* host_error;  // the same code mirrored into host-mapped memory: the host polls it without synchronising
    unsigned long long timeout_ns;
    int rank;
    int world;
};

// A symmetric buffer: the same allocation mapped from every peer (+ optional NVLS multicast alias).
struct PeerBuf {
    char* ptr[kMaxPeers];
    char* mc;  // multicast (NVLS) address of the same pages or nullptr
};

// Number of kernels this library has launched in the current process (benchmarks report it as `gpu_launches`).
uint64_t launch_count();
void count_launch(int n = 1);

#define BAGUA_CUDA_CHECK(expr)                                                                         \
    do {                                                                                               \
        cudaError_t _e = (expr);                                                                       \
        if (_e != cudaSuccess) {                                                                       \
            throw std::runtime_error(std::string("bagua CUDA error: ") + cudaGetErrorString(_e) +     \
                                     " at " + __FILE__ + ":" + std::to_string(__LINE__));            \
        }                                                                                              \
    } while (0)

}  // namespace bagua
