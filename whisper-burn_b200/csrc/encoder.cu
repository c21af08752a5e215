// Encoder-side kernels other than the GEMMs: LayerNorm and non-causal multi-head attention
// (reference: burn nn::LayerNorm used at src/model/mod.rs:300-301,259; qkv_attention mod.rs:493-533).
#include <cuda_fp16.h>
#include "prims.cuh"
#include "wb_internal.h"

namespace wb {

namespace {

constexpr int LN_MAX_PER_LANE = 40;   // d <= 1280

// Where a LayerNorm row goes: fp32 rows y, or fp16 hi / lo planes (x = hi + lo / 2048, prims.cuh) for the tensor-core GEMM
// that consumes the row, with the fp32 rows as well when y is non-null (ln_post: the encoder output returned through the ABI).
struct LnPlanes {
    float* y;
    __half* hi;
    __half* lo;
};
__device__ __forceinline__ void ln_store(float* y, int64_t i, float o) { y[i] = o; }
__device__ __forceinline__ void ln_store(const LnPlanes& p, int64_t i, float o) {
    if (p.y) p.y[i] = o;
    hl_split(o, p.hi[i], p.lo[i]);
}

// One warp per row: burn 0.9 LayerNorm (prims.cuh) of x into out (float* or LnPlanes).  The two instances replace the former
// layernorm_kernel (fp32 rows) and layernorm_f16_kernel (planes), the names the LayerNorm-eps tests still use.
template <typename Out>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, Out out, const float* __restrict__ g, const float* __restrict__ b, float eps,
                 int eps_outside, int rows, int d) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float* xr = x + (int64_t)row * d;
    float v[LN_MAX_PER_LANE];
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE; ++i) {
        const int c = i * 32 + lane;
        v[i] = c < d ? xr[c] : 0.0f;
        s += v[i];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = __fdiv_rn(s, (float)d);
    float q = 0.0f;
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE; ++i) {
        const int c = i * 32 + lane;
        const float dv = __fsub_rn(v[i], mean);
        v[i] = dv;
        if (c < d) q = ln_sq_add(q, dv);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float var = __fdiv_rn(q, (float)d);
    const float den = LN_DEN(var, eps, eps_outside);
#pragma unroll
    for (int i = 0; i < LN_MAX_PER_LANE; ++i) {
        const int c = i * 32 + lane;
        if (c < d) {
            ln_store(out, (int64_t)row * d + c, ln_norm(v[i], den, g, b, c));
        }
    }
}

// ---- flash-style fp32 attention, head dim 64 -----------------------------------------------------
constexpr int AQ = 64, AKV = 64, DH = 64, AST = 68;   // tiles and padded smem stride
constexpr int ATT_THREADS = 256;
constexpr size_t ATT_SMEM = (size_t)4 * 64 * AST * sizeof(float);

__global__ void __launch_bounds__(ATT_THREADS)
enc_attention_kernel(const float* __restrict__ qkv, float* __restrict__ out, const AttnWindow* __restrict__ wins, int d) {
    extern __shared__ __align__(16) float sm[];
    float* Qt = sm;                  // [c][q]
    float* Kt = sm + 64 * AST;       // [c][k]
    float* Vs = sm + 2 * 64 * AST;   // [k][c]
    float* Ps = sm + 3 * 64 * AST;   // [q][k]

    const AttnWindow win = wins[blockIdx.z];
    const int q0 = blockIdx.x * AQ;
    if (q0 >= win.T) return;
    const int h = blockIdx.y;
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    const int64_t ld = 3 * (int64_t)d;
    const float* base = qkv + win.row_off * ld + h * DH;

    // Q tile, transposed
    for (int i = tid; i < AQ * 16; i += ATT_THREADS) {
        const int q = i & 63, c4 = i >> 6;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q0 + q < win.T) v = __ldg(reinterpret_cast<const float4*>(base + (int64_t)(q0 + q) * ld + c4 * 4));
        Qt[(c4 * 4 + 0) * AST + q] = v.x; Qt[(c4 * 4 + 1) * AST + q] = v.y;
        Qt[(c4 * 4 + 2) * AST + q] = v.z; Qt[(c4 * 4 + 3) * AST + q] = v.w;
    }
    float o[4][4], mrow[4], lrow[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        mrow[i] = -INFINITY;
        lrow[i] = 0.0f;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.0f;
    }

    for (int k0 = 0; k0 < win.T; k0 += AKV) {
        __syncthreads();
        for (int i = tid; i < AKV * 16; i += ATT_THREADS) {
            const int k = i & 63, c4 = i >> 6;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k0 + k < win.T) v = __ldg(reinterpret_cast<const float4*>(base + d + (int64_t)(k0 + k) * ld + c4 * 4));
            Kt[(c4 * 4 + 0) * AST + k] = v.x; Kt[(c4 * 4 + 1) * AST + k] = v.y;
            Kt[(c4 * 4 + 2) * AST + k] = v.z; Kt[(c4 * 4 + 3) * AST + k] = v.w;
        }
        for (int i = tid; i < AKV * 16; i += ATT_THREADS) {
            const int k = i >> 4, c4 = i & 15;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k0 + k < win.T) v = __ldg(reinterpret_cast<const float4*>(base + 2 * d + (int64_t)(k0 + k) * ld + c4 * 4));
            *reinterpret_cast<float4*>(Vs + k * AST + c4 * 4) = v;
        }
        __syncthreads();
        // S = Q K^T  (q, k already carry the dh^-0.25 factors, mod.rs:503-514)
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.0f;
#pragma unroll 8
        for (int c = 0; c < DH; ++c) {
            const float4 q4 = *reinterpret_cast<const float4*>(Qt + c * AST + ty * 4);
            const float4 k4 = *reinterpret_cast<const float4*>(Kt + c * AST + tx * 4);
            const float qv[4] = {q4.x, q4.y, q4.z, q4.w};
            const float kv[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (k0 + tx * 4 + j >= win.T) {
#pragma unroll
                for (int i = 0; i < 4; ++i) s[i][j] = -INFINITY;
            }
        // online softmax: exp(x - max) / sum  (burn activation::softmax)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float mx = fmaxf(fmaxf(s[i][0], s[i][1]), fmaxf(s[i][2], s[i][3]));
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float mnew = fmaxf(mrow[i], mx);
            const float corr = expf(mrow[i] - mnew);
            float ps = 0.0f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s[i][j] = expf(s[i][j] - mnew);
                ps += s[i][j];
            }
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
            lrow[i] = lrow[i] * corr + ps;
            mrow[i] = mnew;
#pragma unroll
            for (int j = 0; j < 4; ++j) o[i][j] *= corr;
            *reinterpret_cast<float4*>(Ps + (ty * 4 + i) * AST + tx * 4) = make_float4(s[i][0], s[i][1], s[i][2], s[i][3]);
        }
        __syncthreads();
        // O += P V
#pragma unroll 4
        for (int k = 0; k < AKV; k += 4) {
            float pv[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 p4 = *reinterpret_cast<const float4*>(Ps + (ty * 4 + i) * AST + k);
                pv[i][0] = p4.x; pv[i][1] = p4.y; pv[i][2] = p4.z; pv[i][3] = p4.w;
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float4 v4 = *reinterpret_cast<const float4*>(Vs + (k + kk) * AST + tx * 4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    o[i][0] = fmaf(pv[i][kk], v4.x, o[i][0]);
                    o[i][1] = fmaf(pv[i][kk], v4.y, o[i][1]);
                    o[i][2] = fmaf(pv[i][kk], v4.z, o[i][2]);
                    o[i][3] = fmaf(pv[i][kk], v4.w, o[i][3]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int q = q0 + ty * 4 + i;
        if (q >= win.T) continue;
        const float inv = lrow[i];
        float r[4] = {__fdiv_rn(o[i][0], inv), __fdiv_rn(o[i][1], inv), __fdiv_rn(o[i][2], inv), __fdiv_rn(o[i][3], inv)};
        const int64_t oo = (win.row_off + q) * (int64_t)d + h * DH + tx * 4;
        *reinterpret_cast<float4*>(out + oo) = make_float4(r[0], r[1], r[2], r[3]);
    }
}

}  // namespace

void launch_layernorm(const float* x, float* y, __half* y_hi, __half* y_lo, const LayerNormW& ln, int rows, int d, int eps_outside,
                      cudaStream_t st) {
    WB_REQUIRE(d <= 32 * LN_MAX_PER_LANE, "layernorm: d too large");
    WB_REQUIRE((y_hi == nullptr) == (y_lo == nullptr), "layernorm: hi and lo planes go together");
    if (rows <= 0) return;
    if (y_hi)
        layernorm_kernel<<<(rows + 7) / 8, 256, 0, st>>>(x, LnPlanes{y, y_hi, y_lo}, ln.g, ln.b, ln.eps, eps_outside, rows, d);
    else
        layernorm_kernel<<<(rows + 7) / 8, 256, 0, st>>>(x, y, ln.g, ln.b, ln.eps, eps_outside, rows, d);
    WB_LAUNCH_CHECK();
}

void launch_encoder_attention(const float* qkv, float* out, const AttnWindow* win_dev, int n_windows, int max_T, int d, int n_head,
                              cudaStream_t st) {
    WB_REQUIRE(d == n_head * DH, "attention: head dim must be 64");
    WB_CUDA(cudaFuncSetAttribute(enc_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM));   // per device, cheap: the fp32 path is the fallback
    dim3 grid((max_T + AQ - 1) / AQ, n_head, n_windows);
    enc_attention_kernel<<<grid, ATT_THREADS, ATT_SMEM, st>>>(qkv, out, win_dev, d);
    WB_LAUNCH_CHECK();
}


// ---- cross K/V re-layout -------------------------------------------------------------------------------
// The cross-attention K|V projection (C[M][2d], row = encoder position, written by the GEMM) is re-laid out
// HEAD-MAJOR for the decoders: window w (rows [off_w, off_w + T_w)) keeps its byte range, inside it head h owns the
// contiguous block [T_w][128] = per position 64 key dims then 64 value dims (16-byte chunks XOR-4 swizzled on odd positions).  A decoder (row, head) unit then
// streams ONE contiguous T_w * 512-byte (fp32) block instead of 256-byte pieces at a 2d stride: full DRAM pages,
// and a key batch is a single bulk copy.  Also the place where the fp16 cache is rounded (round-to-nearest).
namespace {
template <typename OT>
__global__ void ckv_relayout_kernel(const float* __restrict__ src, OT* __restrict__ dst, const int64_t* __restrict__ win_row_off,
                                    const int* __restrict__ win_T, int n_windows, int64_t M, int d) {
    const int64_t n4 = M * (2 * d / 4);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / (2 * d / 4);
        const int c = (int)(i % (2 * d / 4)) * 4;
        int lo = 0, hi = n_windows - 1;   // last window whose first row is <= m
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (win_row_off[mid] <= m) lo = mid; else hi = mid - 1;
        }
        const int64_t off = win_row_off[lo];
        const int T = win_T[lo];
        const int which = c / d, cc = c % d, h = cc >> 6, e = cc & 63;
        const float4 v = *reinterpret_cast<const float4*>(src + m * 2 * d + c);
        // XOR-4 swizzle of the 16-byte chunks on odd positions: two consecutive positions staged in shared memory at a
        // 512 / 256-byte pitch then never share a bank group (conflict-free 16-byte reads of 8 keys x 4 lanes)
        constexpr int CH = 16 / (int)sizeof(OT);
        const int j = (int)(m - off);
        const int e_phys = (((e / CH) ^ (4 * (j & 1))) * CH) + e % CH;
        OT* o = dst + off * 2 * d + (int64_t)h * T * 128 + (int64_t)j * 128 + which * 64 + e_phys;
        if constexpr (sizeof(OT) == 4) {
            *reinterpret_cast<float4*>(o) = v;
        } else {
            const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
            uint2 u;
            u.x = *reinterpret_cast<const uint32_t*>(&a);
            u.y = *reinterpret_cast<const uint32_t*>(&b);
            *reinterpret_cast<uint2*>(o) = u;
        }
    }
}
}  // namespace

void launch_ckv_relayout(const float* src, void* dst, bool dst_half, const int64_t* win_row_off, const int* win_T, int n_windows,
                         int64_t M, int d, cudaStream_t st) {
    const int64_t n4 = M * (2 * d / 4);
    const int blocks = (int)std::min<int64_t>((n4 + 255) / 256, 132 * 16);
    if (dst_half) ckv_relayout_kernel<__half><<<blocks, 256, 0, st>>>(src, reinterpret_cast<__half*>(dst), win_row_off, win_T, n_windows, M, d);
    else ckv_relayout_kernel<float><<<blocks, 256, 0, st>>>(src, reinterpret_cast<float*>(dst), win_row_off, win_T, n_windows, M, d);
    WB_LAUNCH_CHECK();
}

}  // namespace wb
