// Host-side helpers shared by the kernel launchers: turn a runtime dtype code, world size or multicast flag into a compile-time
// template argument, and check a launch.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>
#include <type_traits>

#include "common.h"

namespace bagua {

// f(T{}) with T = float, __half or __nv_bfloat16. `family` names the kernels in the error message.
template <typename F>
void dispatch_float(int dtype, const char* family, F&& f) {
    switch (dtype) {
        case F32: f(float{}); break;
        case F16: f(__half{}); break;
        case BF16: f(__nv_bfloat16{}); break;
        default: throw std::runtime_error(std::string("bagua: ") + family + " need f32/f16/bf16, got dtype code " + std::to_string(dtype));
    }
}

// f(std::integral_constant<int, world>{}) for the world sizes of one NVSwitch domain.
template <typename F>
void dispatch_world(int world, F&& f) {
    switch (world) {
        case 1: f(std::integral_constant<int, 1>{}); break;
        case 2: f(std::integral_constant<int, 2>{}); break;
        case 3: f(std::integral_constant<int, 3>{}); break;
        case 4: f(std::integral_constant<int, 4>{}); break;
        case 5: f(std::integral_constant<int, 5>{}); break;
        case 6: f(std::integral_constant<int, 6>{}); break;
        case 7: f(std::integral_constant<int, 7>{}); break;
        case 8: f(std::integral_constant<int, 8>{}); break;
        default: throw std::runtime_error("bagua: peer kernels support 1..8 ranks, got " + std::to_string(world));
    }
}

// f(std::bool_constant<use_multimem>{}): selects the NVLS multicast or the peer-pointer flavour of a peer kernel.
template <typename F>
void dispatch_mc(bool use_multimem, F&& f) {
    if (use_multimem)
        f(std::true_type{});
    else
        f(std::false_type{});
}

// f(std::bool_constant<on>{}) for any other compile-time switch of a kernel.
template <typename F>
void dispatch_flag(bool on, F&& f) {
    dispatch_mc(on, f);
}

inline void check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of ") + what + " failed: " + cudaGetErrorString(e));
    count_launch();
}

}  // namespace bagua
