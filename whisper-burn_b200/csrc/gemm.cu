// fp32 GEMM with fused epilogues for the encoder (reference ops: burn nn::Linear / Conv1d used at
// src/model/mod.rs:243-244 (conv stems as sliding-window GEMMs), :376-382 (MLP), :429-435 (attention
// projections), :484-485 (cross K/V)).
//
//   C[g][m][n] = epi( sum_k A[g][m*lda + k] * B[n][k] )        A, B, C fp32, fp32 accumulate
//   epi(v) = act(v + bias[n]) * (n < scale_cols ? scale : 1) + pos[m][n] + residual[g][m][n]
//
// v1 data path: 128x64x16 tiles, 256 threads, 8x4 register tile per thread, operands staged
// transposed in shared memory (k-major) so the inner loop reads two float4 of A and one of B per
// 32 FMAs.  fp32 CUDA-core FMA keeps the reference's f32 numerics exactly (up to summation order);
// the tensor-core path (gemm_f16.cu, wgmma over fp16 hi/lo planes) replaces this kernel for the large GEMMs.
#include "prims.cuh"
#include "wb_internal.h"

namespace wb {

namespace {

constexpr int BM = 128, BN = 64, BK = 16;
constexpr int GEMM_THREADS = 256;
constexpr int AS_STRIDE = BM + 4;
constexpr int BS_STRIDE = BN + 4;

struct GemmArgs {
    const float* A;
    const float* B;
    float* C;
    const float* bias;
    const float* residual;
    const float* pos;
    const GemmGroup* groups;
    int64_t lda, ldc;
    int N, K;
    int act;
    float scale;
    int scale_cols;
    GemmGroup single;   // used when groups == nullptr
};

__global__ void __launch_bounds__(GEMM_THREADS)
gemm_f32_kernel(const GemmArgs g) {
    __shared__ __align__(16) float As[2][BK][AS_STRIDE];
    __shared__ __align__(16) float Bs[2][BK][BS_STRIDE];

    const GemmGroup grp = g.groups ? g.groups[blockIdx.z] : g.single;
    const int m0 = blockIdx.y * BM;
    if (m0 >= grp.rows) return;
    const int n0 = blockIdx.x * BN;
    const int tid = threadIdx.x;
    const float* A = g.A + grp.a_off;

    // global->smem mapping: A tile 128x16 = 512 float4 (2 per thread), B tile 64x16 = 256 float4
    const int a_row = tid >> 2, a_kq = tid & 3;      // rows a_row and a_row+64
    const int b_row = tid >> 2, b_kq = tid & 3;
    const bool a_ok0 = m0 + a_row < grp.rows, a_ok1 = m0 + a_row + 64 < grp.rows;
    const bool b_ok = n0 + b_row < g.N;
    const float* a_ptr0 = A + (int64_t)(m0 + a_row) * g.lda + a_kq * 4;
    const float* a_ptr1 = A + (int64_t)(m0 + a_row + 64) * g.lda + a_kq * 4;
    const float* b_ptr = g.B + (int64_t)(n0 + b_row) * g.K + b_kq * 4;

    const int ty = tid >> 4, tx = tid & 15;   // 16 x 16 threads, 8 rows x 4 cols each
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 ra0 = a_ok0 ? __ldg(reinterpret_cast<const float4*>(a_ptr0)) : z4;
    float4 ra1 = a_ok1 ? __ldg(reinterpret_cast<const float4*>(a_ptr1)) : z4;
    float4 rb = b_ok ? __ldg(reinterpret_cast<const float4*>(b_ptr)) : z4;

    const int n_kt = g.K / BK;
    for (int kt = 0; kt < n_kt; ++kt) {
        const int buf = kt & 1;
        As[buf][a_kq * 4 + 0][a_row] = ra0.x; As[buf][a_kq * 4 + 1][a_row] = ra0.y;
        As[buf][a_kq * 4 + 2][a_row] = ra0.z; As[buf][a_kq * 4 + 3][a_row] = ra0.w;
        As[buf][a_kq * 4 + 0][a_row + 64] = ra1.x; As[buf][a_kq * 4 + 1][a_row + 64] = ra1.y;
        As[buf][a_kq * 4 + 2][a_row + 64] = ra1.z; As[buf][a_kq * 4 + 3][a_row + 64] = ra1.w;
        Bs[buf][b_kq * 4 + 0][b_row] = rb.x; Bs[buf][b_kq * 4 + 1][b_row] = rb.y;
        Bs[buf][b_kq * 4 + 2][b_row] = rb.z; Bs[buf][b_kq * 4 + 3][b_row] = rb.w;
        __syncthreads();
        if (kt + 1 < n_kt) {
            const int ko = (kt + 1) * BK;
            ra0 = a_ok0 ? __ldg(reinterpret_cast<const float4*>(a_ptr0 + ko)) : z4;
            ra1 = a_ok1 ? __ldg(reinterpret_cast<const float4*>(a_ptr1 + ko)) : z4;
            rb = b_ok ? __ldg(reinterpret_cast<const float4*>(b_ptr + ko)) : z4;
        }
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        // the next iteration writes the other buffer; one barrier per k-tile is enough because a
        // thread can only be one tile ahead of the slowest (it must pass the barrier above first)
    }

    // ---- epilogue
    const int n = n0 + tx * 4;
    if (n >= g.N) return;
    float bias[4] = {0.f, 0.f, 0.f, 0.f};
    if (g.bias) {
#pragma unroll
        for (int j = 0; j < 4; ++j) bias[j] = __ldg(g.bias + n + j);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + ty * 8 + i;
        if (m >= grp.rows) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float t = g.bias ? __fadd_rn(acc[i][j], bias[j]) : acc[i][j];
            if (g.act == ACT_GELU) t = gelu_erf(t);
            if (n + j < g.scale_cols) t = __fmul_rn(t, g.scale);
            v[j] = t;
        }
        if (g.pos) {
            const float4 p4 = __ldg(reinterpret_cast<const float4*>(g.pos + (int64_t)m * g.N + n));
            v[0] = __fadd_rn(v[0], p4.x); v[1] = __fadd_rn(v[1], p4.y);
            v[2] = __fadd_rn(v[2], p4.z); v[3] = __fadd_rn(v[3], p4.w);
        }
        const int64_t co = grp.c_off + (int64_t)m * g.ldc + n;
        if (g.residual) {
            const float4 r4 = *reinterpret_cast<const float4*>(g.residual + co);
            v[0] = __fadd_rn(r4.x, v[0]); v[1] = __fadd_rn(r4.y, v[1]);
            v[2] = __fadd_rn(r4.z, v[2]); v[3] = __fadd_rn(r4.w, v[3]);
        }
        *reinterpret_cast<float4*>(g.C + co) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

}  // namespace

void launch_gemm(const GemmParams& p, cudaStream_t st) {
    WB_REQUIRE(p.K % BK == 0 && p.N % 4 == 0 && p.lda % 4 == 0 && p.ldc % 4 == 0, "gemm: unsupported shape");
    GemmArgs a;
    a.A = p.A; a.B = p.B; a.C = p.C; a.bias = p.bias; a.residual = p.residual; a.pos = p.pos;
    a.groups = p.groups; a.lda = p.lda; a.ldc = p.ldc; a.N = p.N; a.K = p.K; a.act = p.act;
    a.scale = p.scale; a.scale_cols = p.scale_cols;
    a.single = GemmGroup{0, 0, p.max_rows};
    if (p.max_rows <= 0) return;
    dim3 grid((p.N + BN - 1) / BN, (p.max_rows + BM - 1) / BM, p.groups ? p.n_groups : 1);
    gemm_f32_kernel<<<grid, GEMM_THREADS, 0, st>>>(a);
    WB_LAUNCH_CHECK();
}

}  // namespace wb
