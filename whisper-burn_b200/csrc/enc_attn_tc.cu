// Encoder self-attention on the tensor cores (reference op: qkv_attention, src/model/mod.rs:493-533, non-causal, head dim 64).
//
// Flash-attention structure (one CTA = 64 queries of one (window, head), 4 warps x 16 query rows, key/value tiles of 64
// positions streamed through a double-buffered cp.async ring), but at fp32-class accuracy: the reference computes in f32 and the
// parity bar is 2e-5 of scale, so every operand is a PAIR of fp16 planes  x = hi + lo / 2048  (the hi/lo split of prims.cuh)
// and every product is three mma.sync.m16n8k16 terms
//     Q.K^T = Qh.Kh + (Qh.Kl + Ql.Kh) / 2048          P.V = Ph.Vh + (Ph.Vl + Pl.Vh) / 2048
// (the dropped lo.lo term is 2^-22 relative) with fp32 accumulation in two accumulators (main / correction) and the softmax in
// fp32 exactly as burn's activation::softmax composes it (exp(x - max) / sum, online over the key tiles).
// q | k | v arrive as fp16 planes [rows][3d] written by the QKV GEMM epilogue (q and k already carry dh^-0.25, mod.rs:503-514);
// the output leaves as the fp16 planes [rows][d] the out-projection GEMM consumes.
//
// The same CTA body serves the sequence-parallel decoder pass of token scoring (score.cu):
//   * causal self attention (attn_decoder_mask, mod.rs:139): key tiles past the query tile are skipped, keys j > i of the
//     diagonal tile get -inf before the running max;
//   * fp16 K/V (WB_KV_F16 sessions): only the hi planes of K and V enter, hi = fp16(x) being exactly the rounding the persistent
//     decoders apply where K/V enter their fp16 cache; the products lose their K / V correction terms;
//   * cross attention (mod.rs:482-490): the queries are one sequence's rows, the keys and values its window's head block of the
//     session's head-major, XOR-swizzled cross K/V (encoder.cu ckv_relayout_kernel), the same bytes the decoders stream;
//     fp32 K/V are split hi/lo as they are staged.
#include <cuda_fp16.h>

#include "attn_tile.cuh"
#include "wb_internal.h"

namespace wb {

namespace {

constexpr int AT_THREADS = 128;
constexpr size_t AT_SMEM = 2 * TILE_B + 2 * 4 * TILE_B;   // Q hi/lo + 2 stages x (K hi, K lo, V hi, V lo) = 80 KB

// One CTA: the 64 queries [q0, q0 + 64) of one head.  load_q(sQ) stages the Q tile (hi, lo); load_kv(stage_base, k0) stages
// K hi, K lo, V hi, V lo of keys [k0, k0 + 64) (zero rows past Tk; the lo tiles are not read with KV16); o_hi / o_lo: the
// head's output column of query row 0, rows ldo apart.
template <bool CAUSAL, bool KV16, typename LoadQ, typename LoadKV>
__device__ __forceinline__ void attn_cta_tc(uint8_t* sm, int q0, int Tq, int Tk, LoadQ&& load_q, LoadKV&& load_kv, __half* o_hi,
                                            __half* o_lo, int64_t ldo) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const uint32_t sQ = smem_u32(sm), sKV = sQ + 2 * TILE_B;
    load_q(sQ);
    load_kv(sKV, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");

    float o_m[8][4], o_c[8][4], m_row[2] = {-INFINITY, -INFINITY}, l_row[2] = {0.0f, 0.0f};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { o_m[i][j] = 0.0f; o_c[i][j] = 0.0f; }
    uint32_t qh[4][4], ql[4][4];

    int n_tiles = (Tk + TK - 1) / TK;
    if constexpr (CAUSAL) n_tiles = min(n_tiles, q0 / TK + 1);   // TQ == TK: the query tile is the last key tile it sees
    for (int it = 0; it < n_tiles; ++it) {
        if (it + 1 < n_tiles) load_kv(sKV + ((it + 1) & 1) * 4 * TILE_B, (it + 1) * TK);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();
        if (it == 0) {   // A fragments of this warp's 16 query rows, all four 16-dim k-steps
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const int r = warp * 16 + (lane & 15), c = ks * 2 + (lane >> 4);
                ldsm4(sQ + tile_off(r, c), qh[ks][0], qh[ks][1], qh[ks][2], qh[ks][3]);
                ldsm4(sQ + TILE_B + tile_off(r, c), ql[ks][0], ql[ks][1], ql[ks][2], ql[ks][3]);
            }
        }
        const uint32_t sK = sKV + (it & 1) * 4 * TILE_B, sV = sK + 2 * TILE_B;
        // ---- S = Q K^T for 16 rows x 64 keys: main and correction accumulators
        float s_m[8][4], s_c[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) { s_m[i][j] = 0.0f; s_c[i][j] = 0.0f; }
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {   // two 8-key n-tiles per ldmatrix.x4
                // B fragment (k = dim, n = key) from K[key][dim]: matrices (keys 0-7, dims 0-7), (keys 0-7, dims 8-15), (keys 8-15, ...)
                const int r = np * 16 + (lane & 7) + ((lane >> 4) << 3), c = ks * 2 + ((lane >> 3) & 1);
                uint32_t kh0, kh1, kh2, kh3;
                ldsm4(sK + tile_off(r, c), kh0, kh1, kh2, kh3);
                mma(s_m[2 * np], qh[ks], kh0, kh1);
                mma(s_m[2 * np + 1], qh[ks], kh2, kh3);
                if constexpr (!KV16) {
                    uint32_t kl0, kl1, kl2, kl3;
                    ldsm4(sK + TILE_B + tile_off(r, c), kl0, kl1, kl2, kl3);
                    mma(s_c[2 * np], qh[ks], kl0, kl1);
                    mma(s_c[2 * np + 1], qh[ks], kl2, kl3);
                }
                mma(s_c[2 * np], ql[ks], kh0, kh1);
                mma(s_c[2 * np + 1], ql[ks], kh2, kh3);
            }
        }
        // ---- online softmax over the tile (rows g and g + 8 of the warp's 16; a row lives in the 4 lanes of a quad)
        const int k0 = it * TK;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float v = hl_join(s_m[i][j], s_c[i][j]);
                const int key = k0 + i * 8 + 2 * t + (j & 1);
                if (key >= Tk) v = -INFINITY;
                if constexpr (CAUSAL)
                    if (key > q0 + warp * 16 + g + 8 * (j >> 1)) v = -INFINITY;
                s_m[i][j] = v;
                mx[j >> 1] = fmaxf(mx[j >> 1], v);
            }
        float corr[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
            mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
            const float mn = fmaxf(m_row[e], mx[e]);
            corr[e] = expf(m_row[e] - mn);
            m_row[e] = mn;
        }
        float ps[2] = {0.0f, 0.0f};
        uint32_t ph[4][4], pl[4][4];   // P as A fragments of the P.V product: k-step = 16 keys = S n-tiles 2ks, 2ks + 1
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float p0 = expf(s_m[i][0] - m_row[0]), p1 = expf(s_m[i][1] - m_row[0]);
            const float p2 = expf(s_m[i][2] - m_row[1]), p3 = expf(s_m[i][3] - m_row[1]);
            ps[0] += p0 + p1;
            ps[1] += p2 + p3;
            // A fragment: a0 = (row g, k 2t..), a1 = (row g+8, k 2t..), a2 = (row g, k 2t+8..), a3 = (row g+8, k 2t+8..)
            const int ks = i >> 1, hi_half = i & 1;
            split2(p0, p1, ph[ks][hi_half * 2], pl[ks][hi_half * 2]);
            split2(p2, p3, ph[ks][hi_half * 2 + 1], pl[ks][hi_half * 2 + 1]);
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            ps[e] += __shfl_xor_sync(0xffffffffu, ps[e], 1);
            ps[e] += __shfl_xor_sync(0xffffffffu, ps[e], 2);
            l_row[e] = l_row[e] * corr[e] + ps[e];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            o_m[i][0] *= corr[0]; o_m[i][1] *= corr[0]; o_m[i][2] *= corr[1]; o_m[i][3] *= corr[1];
            o_c[i][0] *= corr[0]; o_c[i][1] *= corr[0]; o_c[i][2] *= corr[1]; o_c[i][3] *= corr[1];
        }
        // ---- O += P V
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {   // two 8-dim n-tiles per ldmatrix.x4.trans
                // B fragment (k = key, n = dim) from V[key][dim] through the transposing load:
                // matrices (keys 0-7, dims 0-7), (keys 8-15, dims 0-7), (keys 0-7, dims 8-15), (keys 8-15, dims 8-15)
                const int r = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), c = np * 2 + (lane >> 4);
                uint32_t vh0, vh1, vh2, vh3;
                ldsm4t(sV + tile_off(r, c), vh0, vh1, vh2, vh3);
                mma(o_m[2 * np], ph[ks], vh0, vh1);
                mma(o_m[2 * np + 1], ph[ks], vh2, vh3);
                if constexpr (!KV16) {
                    uint32_t vl0, vl1, vl2, vl3;
                    ldsm4t(sV + TILE_B + tile_off(r, c), vl0, vl1, vl2, vl3);
                    mma(o_c[2 * np], ph[ks], vl0, vl1);
                    mma(o_c[2 * np + 1], ph[ks], vl2, vl3);
                }
                mma(o_c[2 * np], pl[ks], vh0, vh1);
                mma(o_c[2 * np + 1], pl[ks], vh2, vh3);
            }
        }
        __syncthreads();   // every warp is done with this stage before the next prefetch overwrites it
    }
    // ---- normalise (softmax denominator) and write the fp16 planes of the out-projection's input
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int q = q0 + warp * 16 + g + 8 * e;
        if (q >= Tq) continue;
        const float inv = l_row[e];
        __half* oh = o_hi + q * ldo;
        __half* ol = o_lo + q * ldo;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float a = __fdiv_rn(hl_join(o_m[i][2 * e], o_c[i][2 * e]), inv);
            const float b = __fdiv_rn(hl_join(o_m[i][2 * e + 1], o_c[i][2 * e + 1]), inv);
            uint32_t hi, lo;
            split2(a, b, hi, lo);
            *reinterpret_cast<uint32_t*>(oh + i * 8 + 2 * t) = hi;
            *reinterpret_cast<uint32_t*>(ol + i * 8 + 2 * t) = lo;
        }
    }
}

// Self attention over the packed rows of each window (encoder: non-causal, hi/lo K/V) or sequence (scoring: causal, hi/lo or
// fp16 K/V): q | k | v planes [rows][3d]
template <bool CAUSAL, bool KV16>
__global__ void __launch_bounds__(AT_THREADS)
enc_attn_tc_kernel(const __half* __restrict__ qkv_hi, const __half* __restrict__ qkv_lo, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                   const AttnWindow* __restrict__ wins, int d) {
    extern __shared__ __align__(128) uint8_t sm[];
    const AttnWindow win = wins[blockIdx.z];
    const int q0 = blockIdx.x * TQ;
    if (q0 >= win.T) return;
    const int h = blockIdx.y, T = win.T, tid = threadIdx.x;
    const int64_t ld = 3 * (int64_t)d;
    const __half* bh = qkv_hi + win.row_off * ld + h * HD;
    const __half* bl = qkv_lo + win.row_off * ld + h * HD;
    auto load_tile = [&](uint32_t dst, const __half* src, int row0) {   // [64][64] halves from rows row0.. of a [.][3d] plane
        for (int i = tid; i < 64 * 8; i += AT_THREADS) {
            const int r = i >> 3, c = i & 7;
            const bool ok = row0 + r < T;
            cp16(dst + tile_off(r, c), src + (int64_t)(ok ? row0 + r : 0) * ld + c * 8, ok);
        }
    };
    auto load_q = [&](uint32_t sQ) {
        load_tile(sQ, bh, q0);
        load_tile(sQ + TILE_B, bl, q0);
    };
    auto load_kv = [&](uint32_t base, int k0) {
        load_tile(base, bh + d, k0);
        if constexpr (!KV16) load_tile(base + TILE_B, bl + d, k0);
        load_tile(base + 2 * TILE_B, bh + 2 * d, k0);
        if constexpr (!KV16) load_tile(base + 3 * TILE_B, bl + 2 * d, k0);
    };
    attn_cta_tc<CAUSAL, KV16>(sm, q0, T, T, load_q, load_kv, out_hi + win.row_off * (int64_t)d + h * HD,
                              out_lo + win.row_off * (int64_t)d + h * HD, d);
}

// Cross attention of sequence z (rows seqs[z], cross-query planes [rows][d]) over window seq_win[z] of one layer's head-major
// cross K/V: head h of window w is the block [T_w][128] at ckv + win_row_off[w] * 2d + h * T_w * 128, position j holding 64
// key then 64 value elements whose 16-byte chunks are XOR-4 swizzled on odd j.
template <typename KVT>
__global__ void __launch_bounds__(AT_THREADS)
cross_attn_tc_kernel(const __half* __restrict__ q_hi, const __half* __restrict__ q_lo, const KVT* __restrict__ ckv, __half* __restrict__ out_hi,
                     __half* __restrict__ out_lo, const AttnWindow* __restrict__ seqs, const int* __restrict__ seq_win,
                     const int64_t* __restrict__ win_row_off, const int* __restrict__ win_T, int d) {
    extern __shared__ __align__(128) uint8_t sm[];
    constexpr bool KV16 = sizeof(KVT) == 2;
    const AttnWindow sq = seqs[blockIdx.z];
    const int q0 = blockIdx.x * TQ;
    if (q0 >= sq.T) return;
    const int h = blockIdx.y, tid = threadIdx.x, w = seq_win[blockIdx.z], Tk = win_T[w];
    const KVT* blk = ckv + win_row_off[w] * 2 * (int64_t)d + (int64_t)h * Tk * 128;
    auto load_q = [&](uint32_t sQ) {
        for (int i = tid; i < 64 * 8; i += AT_THREADS) {
            const int r = i >> 3, c = i & 7;
            const bool ok = q0 + r < sq.T;
            const int64_t off = (sq.row_off + (ok ? q0 + r : 0)) * (int64_t)d + h * HD + c * 8;
            cp16(sQ + tile_off(r, c), q_hi + off, ok);
            cp16(sQ + TILE_B + tile_off(r, c), q_lo + off, ok);
        }
    };
    auto load_kv = [&](uint32_t base, int k0) {   // which = 0: K, 1: V
        for (int i = tid; i < 2 * 64 * 8; i += AT_THREADS) {
            const int which = i >> 9, r = (i >> 3) & 63, c = i & 7, j = k0 + r;
            const bool ok = j < Tk;
            const uint32_t dst = base + which * 2 * TILE_B + tile_off(r, c);
            const KVT* row = blk + (int64_t)(ok ? j : 0) * 128 + which * 64;
            if constexpr (KV16) {
                cp16(dst, row + ((c ^ (4 * (j & 1))) << 3), ok);   // 8-half chunks
            } else {   // the 8 floats of half-chunk c: float4 chunks 2c, 2c + 1, adjacent after the swizzle
                uint2 h0 = make_uint2(0, 0), l0 = h0, h1 = h0, l1 = h0;
                if (ok) {
                    const float4* src = reinterpret_cast<const float4*>(row) + ((2 * c) ^ (4 * (j & 1)));
                    hl_split4(__ldg(src), h0, l0);
                    hl_split4(__ldg(src + 1), h1, l1);
                }
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(h0.x), "r"(h0.y), "r"(h1.x), "r"(h1.y) : "memory");
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst + TILE_B), "r"(l0.x), "r"(l0.y), "r"(l1.x), "r"(l1.y) : "memory");
            }
        }
    };
    attn_cta_tc<false, KV16>(sm, q0, sq.T, Tk, load_q, load_kv, out_hi + sq.row_off * (int64_t)d + h * HD,
                             out_lo + sq.row_off * (int64_t)d + h * HD, d);
}

template <auto* kernel>
void set_smem_once() {
    static bool attr_set[16] = {};   // per kernel and device ordinal
    int dev = 0;
    WB_CUDA(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 16 && !attr_set[dev]) {
        WB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AT_SMEM));
        attr_set[dev] = true;
    }
}

}  // namespace

void launch_encoder_attention_tc(const __half* qkv_hi, const __half* qkv_lo, __half* out_hi, __half* out_lo, const AttnWindow* win_dev,
                                 int n_windows, int max_T, int d, int n_head, cudaStream_t st) {
    WB_REQUIRE(d == n_head * HD, "attention: head dim must be 64");
    set_smem_once<enc_attn_tc_kernel<false, false>>();
    dim3 grid((max_T + TQ - 1) / TQ, n_head, n_windows);
    enc_attn_tc_kernel<false, false><<<grid, AT_THREADS, AT_SMEM, st>>>(qkv_hi, qkv_lo, out_hi, out_lo, win_dev, d);
    WB_LAUNCH_CHECK();
}

void launch_causal_attention_tc(const __half* qkv_hi, const __half* qkv_lo, __half* out_hi, __half* out_lo, const AttnWindow* seq_dev,
                                int n_seqs, int max_T, int d, int n_head, bool kv_f16, cudaStream_t st) {
    WB_REQUIRE(d == n_head * HD, "attention: head dim must be 64");
    dim3 grid((max_T + TQ - 1) / TQ, n_head, n_seqs);
    if (kv_f16) {
        set_smem_once<enc_attn_tc_kernel<true, true>>();
        enc_attn_tc_kernel<true, true><<<grid, AT_THREADS, AT_SMEM, st>>>(qkv_hi, qkv_lo, out_hi, out_lo, seq_dev, d);
    } else {
        set_smem_once<enc_attn_tc_kernel<true, false>>();
        enc_attn_tc_kernel<true, false><<<grid, AT_THREADS, AT_SMEM, st>>>(qkv_hi, qkv_lo, out_hi, out_lo, seq_dev, d);
    }
    WB_LAUNCH_CHECK();
}

void launch_cross_attention_tc(const __half* q_hi, const __half* q_lo, const void* ckv_layer, bool kv_f16, __half* out_hi, __half* out_lo,
                               const AttnWindow* seq_dev, const int* seq_win_dev, const int64_t* win_row_off_dev, const int* win_T_dev,
                               int n_seqs, int max_T, int d, int n_head, cudaStream_t st) {
    WB_REQUIRE(d == n_head * HD, "attention: head dim must be 64");
    dim3 grid((max_T + TQ - 1) / TQ, n_head, n_seqs);
    if (kv_f16) {
        set_smem_once<cross_attn_tc_kernel<__half>>();
        cross_attn_tc_kernel<__half><<<grid, AT_THREADS, AT_SMEM, st>>>(q_hi, q_lo, static_cast<const __half*>(ckv_layer), out_hi, out_lo, seq_dev,
                                                                          seq_win_dev, win_row_off_dev, win_T_dev, d);
    } else {
        set_smem_once<cross_attn_tc_kernel<float>>();
        cross_attn_tc_kernel<float><<<grid, AT_THREADS, AT_SMEM, st>>>(q_hi, q_lo, static_cast<const float*>(ckv_layer), out_hi, out_lo, seq_dev,
                                                                         seq_win_dev, win_row_off_dev, win_T_dev, d);
    }
    WB_LAUNCH_CHECK();
}

}  // namespace wb
