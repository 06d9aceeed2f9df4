// Host test double of the kernel table behind the C++ NHWC autograd Functions (csrc/torch_hooks/nhwc_functions.cpp): lets the
// CPU suite exercise the Function plumbing (saved tensors, in-place output, shapes, memory format, dtype of the bias gradient,
// workspace / ticket handling) without a GPU. bf16 only; arithmetic in float. Same NaN rule as the kernels: relu(NaN) = NaN, the
// gradient is kept where !(y <= 0), and the pool's argmax is the first maximum in scan order or else the last NaN of the window.
#include <cstdint>
#include <cstring>
#include <vector>

namespace {
float bf2f(uint16_t v) {
    uint32_t u = static_cast<uint32_t>(v) << 16;
    float f;
    std::memcpy(&f, &u, 4);
    return f;
}
uint16_t f2bf(float f) {
    uint32_t u;
    std::memcpy(&u, &f, 4);
    u += 0x7FFFu + ((u >> 16) & 1u);  // round to nearest even
    return static_cast<uint16_t>(u >> 16);
}
float relu(float v) { return v <= 0.f ? 0.f : v; }
int calls[4] = {0, 0, 0, 0};

int bias_relu_fwd(void* y, const void* bias, size_t rows, int C, int, void*) {
    auto* p = static_cast<uint16_t*>(y);
    auto* b = static_cast<const uint16_t*>(bias);
    for (size_t r = 0; r < rows; ++r)
        for (int c = 0; c < C; ++c) {
            float v = bf2f(p[r * C + c]) + bf2f(b[c]);
            p[r * C + c] = f2bf(relu(v));
        }
    ++calls[0];
    return 0;
}
void finish(float* sums, int C, void* out, unsigned int* ticket) {
    if (!out) return;
    auto* o = static_cast<uint16_t*>(out);
    for (int c = 0; c < C; ++c) o[c] = f2bf(sums[c]), sums[c] = 0.f;
    *ticket = 0;
}
int bias_relu_bwd(const void* g, const void* y, void* gout, float* bias_grad, size_t rows, int C, int, void*, void* bias_grad_out, unsigned int* ticket) {
    auto* pg = static_cast<const uint16_t*>(g);
    auto* py = static_cast<const uint16_t*>(y);
    auto* po = static_cast<uint16_t*>(gout);
    for (size_t r = 0; r < rows; ++r)
        for (int c = 0; c < C; ++c) {
            float v = bf2f(py[r * C + c]) <= 0.f ? 0.f : bf2f(pg[r * C + c]);
            po[r * C + c] = f2bf(v);
            bias_grad[c] += v;
        }
    finish(bias_grad, C, bias_grad_out, ticket);
    ++calls[1];
    return 0;
}
int pool_fwd(const void* x, const void* bias, void* out, uint8_t* idx, int N, int H, int W, int C, int, void*) {
    auto* px = static_cast<const uint16_t*>(x);
    auto* b = static_cast<const uint16_t*>(bias);
    auto* po = static_cast<uint16_t*>(out);
    const int Ho = H / 2, Wo = W / 2;
    for (int n = 0; n < N; ++n)
        for (int ho = 0; ho < Ho; ++ho)
            for (int wo = 0; wo < Wo; ++wo)
                for (int c = 0; c < C; ++c) {
                    float best = 0.f;
                    int arg = 0;
                    for (int q = 0; q < 4; ++q) {
                        const int h = 2 * ho + q / 2, w = 2 * wo + q % 2;
                        const float v = bf2f(px[((static_cast<size_t>(n) * H + h) * W + w) * C + c]);
                        if (q == 0 || v > best || v != v) best = v, arg = q;
                    }
                    const size_t o = ((static_cast<size_t>(n) * Ho + ho) * Wo + wo) * C + c;
                    const float v = best + bf2f(b[c]);
                    po[o] = f2bf(relu(v));
                    idx[o] = static_cast<uint8_t>(arg);
                }
    ++calls[2];
    return 0;
}
int pool_bwd(const void* g, const void* out, const uint8_t* idx, void* gin, float* bias_grad, int N, int H, int W, int C, int, void*, void* bias_grad_out,
             unsigned int* ticket) {
    auto* pg = static_cast<const uint16_t*>(g);
    auto* po = static_cast<const uint16_t*>(out);
    auto* pi = static_cast<uint16_t*>(gin);
    const int Ho = H / 2, Wo = W / 2;
    std::memset(pi, 0, static_cast<size_t>(N) * H * W * C * 2);
    for (int n = 0; n < N; ++n)
        for (int ho = 0; ho < Ho; ++ho)
            for (int wo = 0; wo < Wo; ++wo)
                for (int c = 0; c < C; ++c) {
                    const size_t o = ((static_cast<size_t>(n) * Ho + ho) * Wo + wo) * C + c;
                    const float v = bf2f(po[o]) <= 0.f ? 0.f : bf2f(pg[o]);
                    const int q = idx[o], h = 2 * ho + q / 2, w = 2 * wo + q % 2;
                    pi[((static_cast<size_t>(n) * H + h) * W + w) * C + c] = f2bf(v);
                    bias_grad[c] += v;
                }
    finish(bias_grad, C, bias_grad_out, ticket);
    ++calls[3];
    return 0;
}
const char* last_error() { return "fake"; }

struct Api {
    decltype(&bias_relu_fwd) a;
    decltype(&bias_relu_bwd) b;
    decltype(&pool_fwd) c;
    decltype(&pool_bwd) d;
    decltype(&last_error) e;
};
const Api api = {bias_relu_fwd, bias_relu_bwd, pool_fwd, pool_bwd, last_error};
}  // namespace

extern "C" const void* fake_nhwc_api() { return &api; }
extern "C" int fake_nhwc_calls(int i) { return calls[i]; }
