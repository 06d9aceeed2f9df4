// Grouped bf16 GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier), hand-written for sm_90a.
//
//   C[g] = act( A[g] · B[g]^T + bias[g] ),   A: [G, M, K]  B: [G, N, K]  (both K-contiguous),  C: [G, M, N]  bf16, fp32 accumulate
//
// This is the MoE expert FFN (the one GEMM-shaped hot op of the framework; the reference runs a python loop of cuBLAS
// linears, bagua/torch_api/model_parallel/moe/experts.py:31-41). Persistent kernel, one CTA per SM walking 128 x BN
// output tiles (BN = 256, or 128 when N is not a multiple of 256), three warpgroups:
//   warpgroup 0    : TMA producer — one thread issues cp.async.bulk.tensor (128B-swizzled 128x64 / BNx64 tiles of A and B)
//                                    into a 4/6-stage smem ring; the warpgroup gives its registers to the consumers (setmaxnreg)
//   warpgroups 1,2 : consumers    — each owns 64 rows of the tile and issues wgmma.mma_async m64nBNk16 straight from the
//                                    smem descriptors, accumulating in registers (BN/2 fp32 per thread); one wgmma group stays
//                                    in flight while the previous stage is released. Epilogue from registers: + bias, GELU,
//                                    bf16, stores — to local memory, or (PEER variant) straight into the symmetric buffer
//                                    of the GPU that owns the token (the MoE "combine" all-to-all happens in the epilogue,
//                                    tile by tile, while the producer already streams the next tile's operands)
// Synchronisation is mbarrier-only (full/empty per stage). All waits are bounded: a wedged pipeline traps instead of
// hanging the GPU.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>

#include "kernels.h"

namespace bagua {

namespace {

constexpr int BM = 128, BK = 64;
constexpr int WGMMA_K = 16;
constexpr int kGemmThreads = 384;  // producer warpgroup + two consumer warpgroups
constexpr uint32_t kStageBytesA = BM * BK * 2;

// Tile BM x BN with BN in {128, 256}. At BN = 256 each consumer's m64n256k16 reads 2 KB of A + 8 KB of B per 256 tensor
// cycles, well inside the shared-memory bandwidth; at BN = 128 operand traffic per FLOP is 1.5x higher, so it is kept for N
// that 256 does not divide. 4 (BN = 256) or 6 (BN = 128) stages of 48/32 KB fill 192 KB of the 227 KB a block may use.
template <int BN>
struct GemmCfg {
    static constexpr int STAGES = BN == 256 ? 4 : 6;
    static constexpr uint32_t kStageBytesB = BN * BK * 2;
};

template <int BN>
struct __align__(1024) GemmSmem {
    uint8_t a[GemmCfg<BN>::STAGES][kStageBytesA];
    uint8_t b[GemmCfg<BN>::STAGES][GemmCfg<BN>::kStageBytesB];
    uint64_t full[GemmCfg<BN>::STAGES];
    uint64_t empty[GemmCfg<BN>::STAGES];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();  // seconds of waiting: the pipeline is wedged — fail loudly, never hang
    }
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// K-major operand tile in smem with the 128-byte swizzle written by TMA: rows of 128 B, 8-row atoms of 1024 B.
// (wgmma matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major) | SBO>>4 [32,46) | SWIZZLE_128B=1 [62,64))
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    return static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (static_cast<uint64_t>(1024 >> 4) << 32) | (1ull << 62);
}

// D[64 x N] (+)= A[64 x 16] · B[N x 16]^T, both operands K-major in shared memory, D in registers
template <int N>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_bf16<256>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads/writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ float gelu_tanh(float x) {
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    const float u = k0 * (x + k1 * x * x * x);
    return 0.5f * x * (1.f + tanhf(u));
}

// tile id → (group, m block, n block): consecutive ids (= concurrently running CTAs) share the B tile and walk along M
struct TileCoord {
    int g, m0, n0;
};
__device__ __forceinline__ TileCoord tile_coord(int tile, int tiles_m, int tiles_n, int BN) {
    TileCoord c;
    c.m0 = (tile % tiles_m) * BM;
    const int r = tile / tiles_m;
    c.n0 = (r % tiles_n) * BN;
    c.g = r / tiles_n;
    return c;
}

// PEER variant: where the epilogue stores go. Rows of A are ordered [source rank][capacity slot]; the tile of rows
// [m0, m0+128) of expert g belongs to source rank m0 / cap and lands in THAT rank's buffer, laid out
// [owner rank][expert][slot][N] so the receiver finds "what expert e on rank r produced for my slot c".
struct GemmPeerOut {
    char* ptr[kMaxPeers];
    size_t off;
    int rank;    // this (owner) rank
    int cap;     // capacity slots per (source rank, expert); multiple of BM
    int groups;  // local experts
};

template <int BN, bool PEER>
__global__ void __launch_bounds__(kGemmThreads, 1)
    grouped_gemm_tn_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, __nv_bfloat16* __restrict__ C,
                           const float* __restrict__ bias, int M, int N, int K, int num_tiles, int tiles_m, int tiles_n, int act,
                           const GemmPeerOut peer) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int R = BN / 2;  // accumulator registers per consumer thread
    extern __shared__ uint8_t smem_raw[];
    GemmSmem<BN>& sm = *reinterpret_cast<GemmSmem<BN>*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int wg = threadIdx.x >> 7;
    const int num_kb = K / BK;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_a)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_b)) : "memory");
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&sm.full[s], 1);
            mbar_init(&sm.empty[s], 2);  // one arrival per consumer warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {  // ===== TMA producer =====
            uint32_t it = 0;  // running stage counter across tiles
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord(tile, tiles_m, tiles_n, BN);
                for (int kb = 0; kb < num_kb; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&sm.empty[s], ((it / STAGES) & 1) ^ 1);  // fresh barrier: waiting on parity 1 passes immediately
                    mbar_expect_tx(&sm.full[s], kStageBytesA + Cfg::kStageBytesB);
                    tma_load_3d(sm.a[s], &tm_a, &sm.full[s], kb * BK, tc.m0, tc.g);
                    tma_load_3d(sm.b[s], &tm_b, &sm.full[s], kb * BK, tc.n0, tc.g);
                }
            }
        }
        return;
    }

    // ===== consumer warpgroups 1, 2: rows [64 (wg-1), +64) of every tile =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const uint32_t a_off = static_cast<uint32_t>(wg - 1) * 64 * 128;  // 64 rows of 128 B: a whole number of 1024-B swizzle atoms
    float acc[R];
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(tile, tiles_m, tiles_n, BN);
        int prev = -1;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % STAGES;
            mbar_wait(&sm.full[s], (it / STAGES) & 1);
            const uint64_t da = make_smem_desc(smem_u32(sm.a[s]) + a_off), db = make_smem_desc(smem_u32(sm.b[s]));
            fence_regs<R>(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / WGMMA_K; ++k) {
                // advance 32 bytes (16 bf16) along K inside the 128-byte swizzle atom: +2 in the (addr >> 4) field
                wgmma_bf16<BN>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), (kb | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            fence_regs<R>(acc);
            wgmma_wait<1>();  // the previous stage's MMAs are done: hand that stage back to the producer
            if (prev >= 0 && t == 0) mbar_arrive(&sm.empty[prev]);
            prev = s;
        }
        wgmma_wait<0>();
        fence_regs<R>(acc);
        if (t == 0) mbar_arrive(&sm.empty[prev]);

        // epilogue: accumulator fragment of m64nBN — d[4j + h] is row 16 warp + lane/4 + 8 (h/2), column 8 j + 2 (lane%4) + h%2
        const int r0 = (wg - 1) * 64 + warp * 16 + (lane >> 2);
        __nv_bfloat16* crow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if constexpr (PEER) {
                const int src = tc.m0 / peer.cap, c0 = tc.m0 - src * peer.cap;
                crow[h] = reinterpret_cast<__nv_bfloat16*>(peer.ptr[src] + peer.off) +
                          ((static_cast<size_t>(peer.rank) * peer.groups + tc.g) * peer.cap + (c0 + row)) * N + tc.n0;
            } else {
                crow[h] = C + (static_cast<size_t>(tc.g) * M + (tc.m0 + row)) * N + tc.n0;
            }
        }
        const float* brow = bias ? bias + static_cast<size_t>(tc.g) * N + tc.n0 : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            float b0 = 0.f, b1 = 0.f;
            if (brow) b0 = __ldg(brow + col), b1 = __ldg(brow + col + 1);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
                if (act == 1) v0 = gelu_tanh(v0), v1 = gelu_tanh(v1);
                *reinterpret_cast<__nv_bfloat162*>(crow[h] + col) = __floats2bfloat162_rn(v0, v1);
            }
        }
    }
}

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) throw std::runtime_error("bagua: cuTensorMapEncodeTiled is not available from the driver");
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// [G, rows, K] bf16, K contiguous → box (BK x box_rows x 1), 128-byte swizzle
CUtensorMap make_map(const void* ptr, int G, int rows, int K, int box_rows) {
    CUtensorMap m;
    cuuint64_t dims[3] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(G)};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(K) * 2, static_cast<cuuint64_t>(rows) * K * 2};
    cuuint32_t box[3] = {BK, static_cast<cuuint32_t>(box_rows), 1};  // ≤ 256 rows per box
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw std::runtime_error("bagua: cuTensorMapEncodeTiled failed with code " + std::to_string(static_cast<int>(r)));
    return m;
}

}  // namespace

bool grouped_gemm_supported(int M, int N, int K) { return M > 0 && N > 0 && K > 0 && M % BM == 0 && N % 128 == 0 && K % BK == 0; }

namespace {
template <int BN, bool PEER>
void launch_bn(const void* A, const void* B, void* C, const float* bias, int G, int M, int N, int K, int act, const GemmPeerOut& peer,
               cudaStream_t stream) {
    const CUtensorMap ta = make_map(A, G, M, K, BM), tb = make_map(B, G, N, K, BN);
    const size_t smem = sizeof(GemmSmem<BN>) + 1024;
    static bool configured = false;
    static int num_sms = 0;
    if (!configured) {
        BAGUA_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_tn_kernel<BN, PEER>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        int dev = 0;
        BAGUA_CUDA_CHECK(cudaGetDevice(&dev));
        BAGUA_CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        configured = true;
    }
    const int tiles_m = M / BM, tiles_n = N / BN;
    const int num_tiles = tiles_m * tiles_n * G;
    const int grid = num_tiles < num_sms ? num_tiles : num_sms;  // persistent: one CTA per SM
    grouped_gemm_tn_kernel<BN, PEER><<<grid, kGemmThreads, smem, stream>>>(ta, tb, static_cast<__nv_bfloat16*>(C), bias, M, N, K, num_tiles, tiles_m,
                                                                            tiles_n, act, peer);
}
}  // namespace

void launch_grouped_gemm_tn(const void* A, const void* B, void* C, const float* bias, int G, int M, int N, int K, int act, cudaStream_t stream) {
    if (!grouped_gemm_supported(M, N, K)) throw std::runtime_error("bagua: grouped_gemm_tn needs M%128==0, N%128==0, K%64==0");
    if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C)) & 15u)
        throw std::runtime_error("bagua: grouped_gemm_tn needs 16-byte aligned operands");
    const GemmPeerOut none{};
    if (N % 256 == 0)
        launch_bn<256, false>(A, B, C, bias, G, M, N, K, act, none, stream);
    else
        launch_bn<128, false>(A, B, C, bias, G, M, N, K, act, none, stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of grouped_gemm_tn failed: ") + cudaGetErrorString(e));
    count_launch();
}

// GEMM whose epilogue IS the MoE combine all-to-all: A [G, world*cap, K] (rows ordered [source rank][slot]), B [G, N, K];
// the 128-row tiles of source rank s are stored into rank s's symmetric buffer at [this rank][g][slot][N].
// No cross-GPU synchronisation inside: the consumer kernel (moe_gather, local layout) starts with the peer barrier that
// makes the pushes of every owner visible, and ends with the one that lets the owners reuse the buffer.
void launch_grouped_gemm_tn_push(const void* A, const void* B, const float* bias, int G, int N, int K, int act, const PeerCtx& ctx, const PeerBuf& out,
                                 size_t out_off, int cap, cudaStream_t stream) {
    const int M = ctx.world * cap;
    if (!grouped_gemm_supported(M, N, K) || cap % BM != 0) throw std::runtime_error("bagua: grouped_gemm_tn_push needs cap%128==0, N%128==0, K%64==0");
    if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | out_off) & 15u)
        throw std::runtime_error("bagua: grouped_gemm_tn_push needs 16-byte aligned operands");
    GemmPeerOut peer{};
    for (int p = 0; p < ctx.world; ++p) peer.ptr[p] = out.ptr[p];
    peer.off = out_off;
    peer.rank = ctx.rank;
    peer.cap = cap;
    peer.groups = G;
    if (N % 256 == 0)
        launch_bn<256, true>(A, B, nullptr, bias, G, M, N, K, act, peer, stream);
    else
        launch_bn<128, true>(A, B, nullptr, bias, G, M, N, K, act, peer, stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("bagua: launch of grouped_gemm_tn_push failed: ") + cudaGetErrorString(e));
    count_launch();
}

}  // namespace bagua
