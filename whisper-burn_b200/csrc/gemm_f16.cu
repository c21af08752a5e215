// Tensor-core GEMM of the encoder: Hopper wgmma (fp16 operands, fp32 accumulate) fed by TMA through an mbarrier ring.
// (reference ops: burn nn::Linear / Conv1d at src/model/mod.rs:243-244, :376-382, :429-435, :484-485)
//
//   C[g][m][n] = epi( sum_k A[g][m][k] * B[n][k] )      same contract and epilogues as gemm.cu
//
// Precision: the parity bar is identical greedy tokens (encoder output within 2e-5 of scale), so a single fp16 / bf16 pass is
// not acceptable.  B (the weights) is exact in fp16; the fp32 activations travel between the encoder kernels as a PAIR of fp16
// planes A = A_hi + A_lo / 2048 (the hi/lo split of prims.cuh), written by the producing kernel (LayerNorm, attention, the GELU
// epilogue below).  The two planes accumulate into TWO register accumulators that the epilogue combines as hi + lo / 2048.
// Against a TF32 hi/lo formulation: half the bytes per k-block through shared memory, the weight tile loaded once instead of
// twice, and twice the MMA rate.
//
// Kernel shape (one 128 x BN output tile per CTA, 288 threads, one CTA per SM):
//   warps 0-7   two consumer warpgroups; warpgroup w owns rows [64 w, 64 w + 64) of the tile: per k-block 4 + 4
//               wgmma.m64nBNk16 (hi and lo planes against the same B tile), one k-block kept in flight, then the epilogue
//               straight from the accumulator registers -> bias / GELU / q,k scale / pos-emb / residual -> fp32 rows and / or
//               fp16 hi/lo planes for the next kernel
//   warp 8      TMA producer: cp.async.bulk.tensor (3-D maps: k, row, window) of A_hi, A_lo (128 x 64 halves each) and B
//               (BN x 64) into a 4-stage 128B-swizzled ring, mbarrier expect_tx / complete_tx; a slot is released when both
//               warpgroups' MMAs that read it have completed
// The conv stems use the same kernel: their A rows are overlapping windows of a token-major buffer, expressed as a tensor map
// whose row stride is smaller than the row length.
//
// Token scoring (score.cu) runs the same main loop over the tied token embedding (logits = x E^T, mod.rs:154-156) with a
// statistics epilogue (LogitArgs) instead of writing the P x V logits: per (row, column tile) the tile max, the sum of
// exp(x - tile max), the tile arg-max (lowest id on ties) and, in the tile that holds it, the row's target logit.  Columns
// past V (zero-filled by TMA) and special ids of masked rows are excluded.
#include <cuda.h>
#include <cuda_fp16.h>

#include <climits>
#include <cstring>
#include <mutex>
#include <type_traits>

#include "prims.cuh"
#include "wb_internal.h"
#include "wgmma.cuh"

namespace wb {

namespace {

constexpr int F_BM = 128, F_BK = 64, F_STAGES = 4;   // 4 stages x 48 KB (BN = 128): the accumulators of a 128 x 128 tile take
                                                     // 128 registers per consumer thread, so one CTA per SM and a deeper ring
constexpr int F_CONSUMERS = 256;                     // two warpgroups
constexpr int F_THREADS = F_CONSUMERS + 32;          // + the TMA producer warp

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)), "l"(map),
                 "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)), "l"(map),
                 "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t desc_a, uint64_t desc_b) {
    if constexpr (BN == 128) wgmma_m64n128k16(d, desc_a, desc_b);
    else wgmma_m64n64k16(d, desc_a, desc_b);
}

struct F16Args {
    float* C;                 // fp32 result rows (may be null when only planes are wanted)
    __half *P_hi, *P_lo;      // fp16 hi / lo planes of the result (may be null); same row geometry as C
    const float* bias;
    const float* residual;
    const float* pos;
    const GemmGroup* groups;  // device array or null
    GemmGroup single;
    int64_t ldc;
    int N, K;
    int act;
    float scale;
    int scale_cols;
};
struct LogitArgs : F16Args {
    const int* target;          // [rows] id whose logit is gathered
    const uint8_t* row_mask;    // [rows] 1: the row excludes special ids (null: no row does)
    const uint8_t* is_special;  // [V]
    int V, n_tiles;             // n_tiles = gridDim.x: the stride of the per-row tile statistics
    float *tile_m, *tile_s, *tgt_logit;
    int* tile_i;
};

// Statistics epilogue of the logits GEMM: the 4 lanes of a quad hold one row's BN / 4 columns per accumulator half
template <int BN>
__device__ __forceinline__ void logit_stats_epilogue(const float (&acc_h)[BN / 2], const float (&acc_l)[BN / 2], const LogitArgs& g, int rows,
                                                     int m_base, int n0, int lane) {
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
        const int m = m_base + 8 * hrow;
        const bool live = m < rows;   // quad-uniform; every lane stays for the shuffles
        const int mr = live ? m : 0;
        const bool masked = g.row_mask != nullptr && g.row_mask[mr] != 0;
        const int tgt = g.target[mr];
        float mx = -INFINITY;
        int ai = INT_MAX;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = n0 + 8 * j + 2 * (lane & 3) + e;
                const float x = hl_join(acc_h[4 * j + 2 * hrow + e], acc_l[4 * j + 2 * hrow + e]);
                if (live && n == tgt) g.tgt_logit[m] = x;
                const bool ok = n < g.V && !(masked && __ldg(g.is_special + n));
                if (ok && x > mx) { mx = x; ai = n; }   // ascending n: the lowest id of a tie stays
            }
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, mx, o);
            const int oi = __shfl_xor_sync(0xffffffffu, ai, o);
            if (om > mx || (om == mx && oi < ai)) { mx = om; ai = oi; }
        }
        float s = 0.0f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = n0 + 8 * j + 2 * (lane & 3) + e;
                const float x = hl_join(acc_h[4 * j + 2 * hrow + e], acc_l[4 * j + 2 * hrow + e]);
                if (n < g.V && !(masked && __ldg(g.is_special + n))) s += expf(x - mx);
            }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if (live && (lane & 3) == 0) {
            const int64_t o = (int64_t)m * g.n_tiles + blockIdx.x;
            g.tile_m[o] = mx;
            g.tile_s[o] = s;
            g.tile_i[o] = ai;
        }
    }
}

template <int BN, typename Args>
__global__ void __launch_bounds__(F_THREADS, 1)
gemm_f16_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                   const __grid_constant__ CUtensorMap map_b, const Args g) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    constexpr int A_BYTES = F_BM * F_BK * 2;   // 16 KB per plane
    constexpr int B_BYTES = BN * F_BK * 2;
    constexpr int STAGE = 2 * A_BYTES + B_BYTES;
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(base + F_STAGES * STAGE);
    uint64_t* empty = full + F_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const GemmGroup grp = g.groups ? g.groups[blockIdx.z] : g.single;
    const int m0 = blockIdx.y * F_BM;
    if (m0 >= grp.rows) return;   // uniform per CTA
    const int n0 = blockIdx.x * BN;
    const int nkb = (g.K + F_BK - 1) / F_BK;

    if (threadIdx.x == F_CONSUMERS) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        for (int s = 0; s < F_STAGES; ++s) {
            mbar_init(full + s, 1);
            mbar_init(empty + s, 2);   // one arrival per consumer warpgroup
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (threadIdx.x >= F_CONSUMERS) {
        if (lane == 0) {
            // ===== TMA producer
            for (int i = 0; i < nkb; ++i) {
                const int s = i % F_STAGES;
                const uint32_t ph = (i / F_STAGES) & 1;
                mbar_wait(empty + s, ph ^ 1);
                mbar_expect_tx(full + s, STAGE);
                uint8_t* st = base + s * STAGE;
                tma_load_3d(st, &map_a_hi, full + s, i * F_BK, m0, blockIdx.z);
                tma_load_3d(st + A_BYTES, &map_a_lo, full + s, i * F_BK, m0, blockIdx.z);
                tma_load_2d(st + 2 * A_BYTES, &map_b, full + s, i * F_BK, n0);
            }
        }
        return;
    }
    // ===== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of the tile
    const int wg = warp >> 2;
    float acc_h[BN / 2], acc_l[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) { acc_h[j] = 0.0f; acc_l[j] = 0.0f; }
    wgmma_fence_regs(acc_h);
    wgmma_fence_regs(acc_l);
#pragma unroll 1
    for (int i = 0; i < nkb; ++i) {
        const int s = i % F_STAGES;
        mbar_wait(full + s, (i / F_STAGES) & 1);
        const uint32_t st = smem_u32(base + s * STAGE);
        // a warpgroup's 64 rows are 8 swizzle atoms of 1024 bytes into the 128-row A tiles
        const uint64_t dah = wgmma_desc(st + wg * 8192), dal = wgmma_desc(st + A_BYTES + wg * 8192), db = wgmma_desc(st + 2 * A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < F_BK / 16; ++k) {   // K step = 16 halves = 32 bytes -> +2 in the (>> 4) address field
            wgmma_tile<BN>(acc_h, dah + 2 * k, db + 2 * k);
            wgmma_tile<BN>(acc_l, dal + 2 * k, db + 2 * k);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have read their stage
        if (i > 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty + (i - 1) % F_STAGES);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc_h);
    wgmma_fence_regs(acc_l);

    if constexpr (std::is_same<Args, LogitArgs>::value) {
        logit_stats_epilogue<BN>(acc_h, acc_l, g, grp.rows, m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), n0, lane);
    } else {
        // ===== epilogue.  Accumulator fragment of a m64nBN wgmma: register 4j + e of thread (warp w, lane) holds row
        // 16 w + lane / 4 (+ 8 for e >= 2), column 8 j + 2 (lane % 4) + (e & 1).
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hrow;
            if (m >= grp.rows) continue;
            const int64_t crow = grp.c_off + (int64_t)m * g.ldc;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = n0 + 8 * j + 2 * (lane & 3);
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float t = hl_join(acc_h[4 * j + 2 * hrow + e], acc_l[4 * j + 2 * hrow + e]);
                    if (g.bias) t = __fadd_rn(t, __ldg(g.bias + n + e));
                    if (g.act == ACT_GELU) t = gelu_erf(t);
                    if (n + e < g.scale_cols) t = __fmul_rn(t, g.scale);
                    v[e] = t;
                }
                if (g.pos) {
                    const float2 p2 = __ldg(reinterpret_cast<const float2*>(g.pos + (int64_t)m * g.N + n));
                    v[0] = __fadd_rn(v[0], p2.x); v[1] = __fadd_rn(v[1], p2.y);
                }
                if (g.residual) {
                    const float2 r2 = *reinterpret_cast<const float2*>(g.residual + crow + n);
                    v[0] = __fadd_rn(r2.x, v[0]); v[1] = __fadd_rn(r2.y, v[1]);
                }
                if (g.C) *reinterpret_cast<float2*>(g.C + crow + n) = make_float2(v[0], v[1]);
                if (g.P_hi) {
                    __half2 h, l;
                    hl_split_pair(v[0], v[1], h, l);
                    *reinterpret_cast<__half2*>(g.P_hi + crow + n) = h;
                    *reinterpret_cast<__half2*>(g.P_lo + crow + n) = l;
                }
            }
        }
    }
}

// fp32 -> (hi, lo) fp16 planes
__global__ void split_f16_kernel(const float4* __restrict__ src, uint2* __restrict__ hi, uint2* __restrict__ lo, int64_t n4) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
        hl_split4(src[i], hi[i], lo[i]);
}

// ---- host: tensor maps ----------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static std::once_flag once;
    static EncodeTiledFn fn = nullptr;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
    });
    if (!fn) fail(WB_ERR_CUDA, "cuTensorMapEncodeTiled not available");
    return fn;
}

// fp16 tensor [dim2][dim1][dim0] with element strides (1, s1, s2); box (b0, b1, 1); 128B swizzle
CUtensorMap make_map(const __half* base, uint64_t dim0, uint64_t dim1, uint64_t dim2, uint64_t s1, uint64_t s2, uint32_t b0, uint32_t b1, int rank) {
    CUtensorMap m;
    std::memset(&m, 0, sizeof(m));
    cuuint64_t dims[3] = {dim0, dim1, dim2};
    cuuint64_t strides[2] = {s1 * sizeof(__half), s2 * sizeof(__half)};
    cuuint32_t box[3] = {b0, b1, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) fail(WB_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
    return m;
}

template <int BN, typename Args>
void launch_f16_t(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& b, const Args& a, dim3 grid, cudaStream_t st) {
    constexpr size_t smem = 1024 + (size_t)F_STAGES * (2 * F_BM * F_BK * 2 + BN * F_BK * 2) + 2 * F_STAGES * sizeof(uint64_t);
    static std::mutex mu;
    static bool configured[16] = {};   // per device ordinal
    int dev = 0;
    WB_CUDA(cudaGetDevice(&dev));
    {
        std::lock_guard<std::mutex> lock(mu);
        if (dev >= 0 && dev < 16 && !configured[dev]) {
            WB_CUDA(cudaFuncSetAttribute(gemm_f16_tc_kernel<BN, Args>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            configured[dev] = true;
        }
    }
    gemm_f16_tc_kernel<BN, Args><<<grid, F_THREADS, smem, st>>>(ah, al, b, a);
    WB_LAUNCH_CHECK();
}

}  // namespace

void launch_split_f16(const float* src, __half* hi, __half* lo, int64_t n, cudaStream_t st) {
    WB_REQUIRE(n % 4 == 0, "split: length must be a multiple of 4");
    const int64_t n4 = n / 4;
    if (n4 == 0) return;
    const int blocks = (int)std::min<int64_t>((n4 + 255) / 256, 132 * 8);
    split_f16_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<uint2*>(hi), reinterpret_cast<uint2*>(lo), n4);
    WB_LAUNCH_CHECK();
}

bool gemm_f16_supported(const GemmF16Params& p) { return p.N % 64 == 0 && p.K % 8 == 0 && p.lda % 8 == 0 && p.ldc % 4 == 0; }

// Tensor maps depend only on (pointers, shapes): a plan is built once per GEMM site and geometry and reused by every launch.
struct GemmF16Plan::Impl {
    CUtensorMap ah, al, b;
    F16Args args;
    dim3 grid;
    int BN;
};
GemmF16Plan::GemmF16Plan() = default;
GemmF16Plan::~GemmF16Plan() { delete impl; }

void GemmF16Plan::build(const GemmF16Params& p, int64_t a_group_stride, int a_rows_total_per_group) {
    WB_REQUIRE(gemm_f16_supported(p), "gemm_f16: unsupported shape");
    delete impl;
    impl = new Impl();
    const int ng = p.groups ? p.n_groups : 1;
    const uint64_t rows = (uint64_t)a_rows_total_per_group;
    const uint64_t gstride = ng > 1 ? (uint64_t)a_group_stride : (uint64_t)p.lda * rows;
    impl->ah = make_map(p.A_hi, (uint64_t)p.K, rows, (uint64_t)ng, (uint64_t)p.lda, gstride, F_BK, F_BM, 3);
    impl->al = make_map(p.A_lo, (uint64_t)p.K, rows, (uint64_t)ng, (uint64_t)p.lda, gstride, F_BK, F_BM, 3);
    impl->BN = (p.N % 128 == 0 && (int64_t)(p.N / 128) * ((p.max_rows + F_BM - 1) / F_BM) * ng >= 96) ? 128 : 64;
    impl->b = make_map(p.B, (uint64_t)p.K, (uint64_t)p.N, 1, (uint64_t)p.K, (uint64_t)p.K * p.N, F_BK, (uint32_t)impl->BN, 2);
    F16Args& a = impl->args;
    a.C = p.C; a.P_hi = p.P_hi; a.P_lo = p.P_lo; a.bias = p.bias; a.residual = p.residual; a.pos = p.pos; a.groups = p.groups;
    a.single = GemmGroup{0, 0, p.max_rows};
    a.ldc = p.ldc; a.N = p.N; a.K = p.K; a.act = p.act; a.scale = p.scale; a.scale_cols = p.scale_cols;
    impl->grid = dim3(p.N / impl->BN, (p.max_rows + F_BM - 1) / F_BM, ng);
    key_rows = p.max_rows;
    key_groups = ng;
}

void GemmF16Plan::launch(cudaStream_t st) const {
    if (!impl || impl->args.single.rows <= 0 || impl->grid.y == 0) return;
    if (impl->BN == 128) launch_f16_t<128>(impl->ah, impl->al, impl->b, impl->args, impl->grid, st);
    else launch_f16_t<64>(impl->ah, impl->al, impl->b, impl->args, impl->grid, st);
}

int logit_stats_tiles(int V) { return (V + 127) / 128; }

void launch_logit_stats(const LogitStatsParams& p, cudaStream_t st) {
    WB_REQUIRE(p.rows >= 1 && p.K % 8 == 0 && p.V >= 1, "logit_stats: unsupported shape");
    constexpr int BN = 128;
    const CUtensorMap ah = make_map(p.A_hi, (uint64_t)p.K, (uint64_t)p.rows, 1, (uint64_t)p.K, (uint64_t)p.K * p.rows, F_BK, F_BM, 3);
    const CUtensorMap al = make_map(p.A_lo, (uint64_t)p.K, (uint64_t)p.rows, 1, (uint64_t)p.K, (uint64_t)p.K * p.rows, F_BK, F_BM, 3);
    const CUtensorMap b = make_map(p.E, (uint64_t)p.K, (uint64_t)p.V, 1, (uint64_t)p.K, (uint64_t)p.K * p.V, F_BK, BN, 2);   // rows past V read 0
    LogitArgs a{};
    a.single = GemmGroup{0, 0, p.rows};
    a.K = p.K;
    a.target = p.target; a.row_mask = p.row_mask; a.is_special = p.is_special;
    a.V = p.V; a.n_tiles = logit_stats_tiles(p.V);
    a.tile_m = p.tile_m; a.tile_s = p.tile_s; a.tile_i = p.tile_i; a.tgt_logit = p.tgt_logit;
    launch_f16_t<BN>(ah, al, b, a, dim3(a.n_tiles, (p.rows + F_BM - 1) / F_BM, 1), st);
}

}  // namespace wb
