// Batched persistent decoder on the tensor cores (up to 32 rows per launch: small.en / medium / large batches and beams).
//
// Same single-launch structure, stage list and reference math as decoder3.cu (TextDecoder::forward
// src/model/mod.rs:131-157, blocks :345-350, attention :428-533, MLP :376-382, search closure
// src/transcribe.rs:253-307), but every linear layer is a swap-AB tensor-core product instead of a per-row
// FMA GEMV, so the weights are streamed ONCE per step for all rows:
//   * a warp owns a 16-feature tile of W[N][K] (fp16, exact) and multiplies it with ALL rows of the batch:
//     mma.sync.m16n8k16 with M = 16 output features, N = 8 batch rows per n-tile (up to 4 n-tiles), K = 16;
//   * the fp32 activations are split into fp16 hi + fp16 (lo * 2^11) planes (22 mantissa bits; products with
//     the fp16 weights are exact, accumulation is fp32) held in FRAGMENT ORDER, so a B fragment is one
//     conflict-free 16-byte shared load.  Attention outputs, LayerNorm outputs and the MLP hidden layer are WRITTEN in
//     that layout by their producers (global planes), so staging them is a plain cp.async copy; a LayerNorm is its own
//     stage: row r is normalised ONCE, by all 256 threads of CTA r (every CTA recomputing all rows cost 12-18 us per
//     stage in L2 -> SM bandwidth, a single warp per row ~3 us of dependent arithmetic, the block-wide version 1.5 us);
//   * the A fragments come straight from global memory as 16-byte loads (a K permutation inside each
//     32-column chunk makes 8 consecutive halves of a weight row the a0..a3 registers of two MMAs) and are
//     prefetched BEFORE the grid barrier that precedes the stage: weights do not depend on activations;
//   * the 8 warps of a CTA split K; partial tiles are reduced through shared memory in a fixed order;
//   * MLP2 (K = 4d) is split over CTAs into K slabs (3 x 4d/3 when that keeps the 8-warp split, else 4 x d): the
//     partial sums are folded into x, in a fixed order, by the LayerNorm stage that consumes x next (only CTA r
//     touches row r there, so the fold is in place).  The d x d projections (out, cross query, cross out) run the same way
//     as d/256 slabs of 256 columns when that still fits one round of the grid (small.en: 144 items instead of 48, a third of
//     the staging per CTA); the cross query's partials are folded where the attention stage loads q (dec5_build_tables builds the
//     descriptors; the producers of the staged planes write them slab-major);
//   * cross attention streams the unit's contiguous head-major K/V block (encoder.cu ckv_relayout_kernel) with 4 KB bulk
//     copies (8 fp32 / 16 fp16 keys) into a per-warp mbarrier ring that aliases the (then dead) activation planes;
//   * logits: E[V][d] is streamed once through the same MMA path into an L2-resident [R][V] buffer (vocabulary tiles dealt per
//     CTA first, then per warp: every SM streams the same number); a second stage turns it into per-slice (max, sum-exp, top
//     candidates) records (compact code for greedy: this part runs once per step from a cold instruction cache), then one
//     warp per row finishes.
// Code size matters: the layer loop must stay inside the instruction cache, so every building block (staging,
// MMA tile, emit, attention) exists ONCE and the stages are driven by small descriptors (the first version
// inlined six copies and ran 3x slower than its memory traffic explains).
// Requirements: fp16-exact weights, d % 256 == 0, d <= 1280, R <= 32 per launch (launch_dec5 runs larger batches -- beams of many
// windows -- as row groups of 32, one launch each, a.kv_row0 = first cache row of the group).  Everything else falls back to decoder3.cu.
#include <cooperative_groups.h>
#include <cuda_fp16.h>

#include "dec_common.cuh"

namespace wb {

namespace {

constexpr int RED_LD = 20;    // padded feature stride of the cross-warp reduction buffer (conflict-free fragment stores)
constexpr int MAXCH = 5;      // 32-column chunks per warp and slab: slab = d <= 1280 -> d / 256 <= 5
constexpr int GC = 4;         // logits: chunks per prefetch group
constexpr int PL_ROWS = 32;   // rows of the global activation planes
constexpr int RING_W = 16384; // attention: bytes of the per-warp K/V ring (aliases the activation planes, which are dead during attention)
constexpr int DEC5_KC = 8;    // top candidates kept per (row, slice) record

enum { ST_LN_EMB = D5_ST_LN_EMB, ST_LN_FOLD = D5_ST_LN_FOLD, ST_LN_FOLD_NOPUB = D5_ST_LN_FOLD_NOPUB, ST_LN_X = D5_ST_LN_X,
       ST_PLANES = D5_ST_PLANES, ST_CROSS = D5_ST_CROSS };
enum { EM_QKV = D5_EM_QKV, EM_RESID = D5_EM_RESID, EM_CQ = D5_EM_CQ, EM_HID = D5_EM_HID, EM_PART = D5_EM_PART, EM_LOGITS = D5_EM_LOGITS };

// widest K slab staged in shared memory: d, or 4d/3 when MLP2 splits into 3 slabs (session.cu)
#define PLANE_COLS_MAX(d_) ((((4 * (d_)) % 3 == 0) && ((4 * (d_) / 3) % 256 == 0) && (4 * (d_) / 3 <= 1280)) ? 4 * (d_) / 3 : (d_))

using GemmDesc = Dec5Desc;   // host-built stage descriptors (decoder.h): no switch in the kernel, so the compiler cannot clone the stage body per case

__device__ __forceinline__ void bar_named(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

__device__ __forceinline__ void store_plane_elem(uint4* phi, uint4* plo, int nchunks, int row, int col, float v) {
    __half h, l;
    hl_split(v, h, l);
    const int idx = plane_idx(nchunks, row, col);
    reinterpret_cast<__half*>(phi + idx)[col & 7] = h;
    reinterpret_cast<__half*>(plo + idx)[col & 7] = l;
}

// A fragments of one (16-feature tile, K slice of this warp): feature rows g and g+8, MAXCH chunks of 32 columns
struct AFrag {
    uint4 r0[MAXCH], r8[MAXCH];
    float bias;
};
// item = slab * n_tiles + tile; this warp's slice of the slab (= D.ks columns) is [warp * ks / 8, +ks / 8)
__device__ __forceinline__ void load_afrag(const GemmDesc& D, int d, int item, AFrag& f) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int n_tiles = D.N >> 4, tile = item % n_tiles, slab = item / n_tiles;
    const int ks = D.ks, K = D.n_slabs * ks, nch = ks >> 8;
    const int k0 = slab * ks + warp * (ks >> 3) + t * 8;
    const __half* Wh = reinterpret_cast<const __half*>(D.W);
    const uint4* p0 = reinterpret_cast<const uint4*>(Wh + (int64_t)(tile * 16 + g) * K + k0);
    const uint4* p1 = reinterpret_cast<const uint4*>(Wh + (int64_t)(tile * 16 + g + 8) * K + k0);
#pragma unroll
    for (int c = 0; c < MAXCH; ++c) {
        if (c < nch) {
            f.r0[c] = __ldg(p0 + c * 4);
            f.r8[c] = __ldg(p1 + c * 4);
        }
    }
    f.bias = (D.bias != nullptr && slab == 0) ? __ldg(D.bias + tile * 16 + (threadIdx.x & 15)) : 0.0f;
}

// =====================================================================================================
// Stage slots of one layer (descriptor a.d5[l * 16 + slot]); the logits use a.d5[L * 16 + {11, 12}].
enum { SL_LN1 = 0, SL_QKV, SL_SELF, SL_OUT, SL_LN2, SL_CQ, SL_CROSS, SL_COUT, SL_LN3, SL_MLP1, SL_MLP2, SL_LNF, SL_LOGITS, SL_COUNT };

template <int NT8, typename KVT>
__global__ void __launch_bounds__(NT, 1)
dec5_kernel(const DecArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int d = a.d, H = a.H, L = a.L, V = a.V, R = a.R, t_max = a.t_max;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    constexpr int RP = NT8 * 8;
    constexpr int KC = DEC5_KC;
    constexpr int NE = (16 * RP + NT - 1) / NT;
    const int nchunks = d >> 5, nch = d >> 8, nv = d >> 2;
    uint4* xhi = reinterpret_cast<uint4*>(sm);            // [NT8][d/32][32] fragment-order fp16 hi plane
    uint4* xlo = xhi + NT8 * (PLANE_COLS_MAX(d) >> 5) * 32;   // same, residual * 2^11 (planes sized for the widest K slab)
    float* red = reinterpret_cast<float*>(reinterpret_cast<char*>(sm) + max(2 * NT8 * (PLANE_COLS_MAX(d) >> 5) * 32 * 16, NW * RING_W));   // [NW][RP][RED_LD]; also cross-merge weights
    float* qs = red + NW * RP * RED_LD;                   // [2][64] query of the attention unit of each 4-warp group
    float* wm = qs + 128;                                 // [NW]
    float* wl = wm + NW;                                  // [NW]
    float* wo = wl + NW;                                  // [NW][64]
    GemmDesc* ds = reinterpret_cast<GemmDesc*>(wo + NW * 64);   // [L * 16 + 16] stage descriptors: a global load per stage would be a dependent round trip
    for (int i = tid; i < (L * 16 + 16) * (int)(sizeof(GemmDesc) / 16); i += NT) reinterpret_cast<uint4*>(ds)[i] = __ldg(reinterpret_cast<const uint4*>(a.d5) + i);
    uint64_t* kv_bar = reinterpret_cast<uint64_t*>(ds + L * 16 + 16);   // [NW][KV_STG] cross-attention K/V ring: one mbarrier per stage
    constexpr int KV_STG = RING_W / AttnBulkGeom<KVT>::STGB;               // 4 stages of 4 KB: 8 fp32 keys or 16 fp16 keys each
    if (lane == 0) {
        for (int j = 0; j < KV_STG; ++j) mbar_init(kv_bar + warp * KV_STG + j, 1);
        mbar_fence_init();
    }
    unsigned int kv_count = 0;   // batches this warp has pushed through its K/V ring
    __syncthreads();
    unsigned int gen = 0;
    int tr_n = 0;
    WB_TRACE();
    const float scale = a.qk_scale;
    const int S = a.n_splits;
    const float* yp = a.ypart;                            // [4][R][d] MLP2 partial sums of the previous layer
    const int64_t yps = (int64_t)R * d;
    const int64_t pl_plane = (int64_t)PL_ROWS * d / 8;    // uint4 per global plane (one slab)
    uint4* att_hi = reinterpret_cast<uint4*>(a.att_pl);   // attention output planes: hi, lo
    uint4* att_lo = att_hi + pl_plane;
    uint4* xn_hi = att_lo + pl_plane;                     // LayerNorm output planes: hi, lo
    uint4* xn_lo = xn_hi + pl_plane;
    uint4* hid_hi = reinterpret_cast<uint4*>(a.hid_pl);   // [slabs] hi planes, then [slabs] lo planes (slab width hks columns: 4d in 4 or 3 slabs)
    uint4* hid_lo = hid_hi + 4 * pl_plane;
    const int hks = ds[SL_MLP2].ks;                       // K slab width of MLP2 = column width of the hidden-layer planes
    const int aks = ds[SL_OUT].ks;                        // K slab width of the out projections = column width of the attention-output planes (d: unsplit)
    const int cq_parts = ds[SL_CQ].emit == EM_PART ? ds[SL_CQ].n_slabs : 0;   // cross query delivered as K-slab partial sums (folded where it is read)
    float* x = a.x;

    AFrag pf;
    bool pf_valid = false;
    for (int step = 0; step < a.n_steps; ++step) {
        const int p = a.pos0 + step;
        const bool want_logits = p >= a.logits_from;
        for (int l = 0; l < L; ++l) {
            KVT* kcl = reinterpret_cast<KVT*>(a.kc) + (size_t)l * a.Rmax * t_max * d;
            KVT* vcl = reinterpret_cast<KVT*>(a.vc) + (size_t)l * a.Rmax * t_max * d;
            const int n_slots = (l == L - 1 && want_logits) ? SL_COUNT : SL_LNF;
#pragma unroll 1
            for (int slot = 0; slot < n_slots; ++slot) {
                const GemmDesc& D = ds[(slot >= SL_LNF ? L : l) * 16 + slot];
                if (D.kind == D5_KIND_LN) {
                    // ================= LayerNorm (burn 0.9 form, prims.cuh) of row blockIdx.x by ONE warp of ONE CTA,
                    // written as fragment-order hi/lo planes for the next linear stage (every CTA copies them after the barrier).
                    // EMB: x = tok_emb[token] + pos_emb[p] (mod.rs:141-146); FOLD: x += the four MLP2 partial sums of the
                    // previous layer (fixed order); both publish the fp32 row for the residual adds of this layer.
                    // The whole CTA works on the row (thread t owns the float4 columns t and t + 256): a single warp would spend ~2 us
                    // in dependent arithmetic; two block reductions through shared memory instead.
                    const int r = blockIdx.x;
                    if (r < R) {
                        constexpr int PT = 2;   // float4 per thread: d <= 1280 -> d / 4 <= 320 <= 2 * 256
                        const int n_part = D.n_fold;   // K-slab partial sums of the producing linear stage (MLP2, or a split out projection)
                        float4 v[PT], g4[PT], b4[PT];
                        int tok = 0;
                        if (D.stage == ST_LN_EMB) tok = a.use_cur_tok ? __ldcg(a.cur_tok + r) : __ldcg(a.tokens + (int64_t)r * t_max + p);
                        const float* pe = a.pos_emb + (int64_t)p * d;
#pragma unroll
                        for (int i = 0; i < PT; ++i) {
                            const int c = min(tid + i * NT, nv - 1);   // clamped: all loads are issued unconditionally, masked at use
                            g4[i] = __ldg(reinterpret_cast<const float4*>(D.g) + c);
                            b4[i] = __ldg(reinterpret_cast<const float4*>(D.b) + c);
                            if (D.stage == ST_LN_EMB) {
                                const float4 e4 = __ldg(reinterpret_cast<const float4*>(a.tok_emb + (int64_t)tok * d) + c);
                                const float4 p4 = __ldg(reinterpret_cast<const float4*>(pe) + c);
                                v[i] = make_float4(__fadd_rn(e4.x, p4.x), __fadd_rn(e4.y, p4.y), __fadd_rn(e4.z, p4.z), __fadd_rn(e4.w, p4.w));
                            } else {
                                v[i] = __ldcg(reinterpret_cast<const float4*>(x + (int64_t)r * d) + c);
                                if (D.stage != ST_LN_X) {
                                    const float4 p0 = __ldcg(reinterpret_cast<const float4*>(yp + (int64_t)r * d) + c);
                                    const float4 p1 = __ldcg(reinterpret_cast<const float4*>(yp + yps + (int64_t)r * d) + c);
                                    const float4 p2 = n_part > 2 ? __ldcg(reinterpret_cast<const float4*>(yp + 2 * yps + (int64_t)r * d) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
                                    const float4 p3 = n_part > 3 ? __ldcg(reinterpret_cast<const float4*>(yp + 3 * yps + (int64_t)r * d) + c) : make_float4(0.f, 0.f, 0.f, 0.f);
                                    v[i].x = __fadd_rn(v[i].x, __fadd_rn(__fadd_rn(p0.x, p1.x), __fadd_rn(p2.x, p3.x)));
                                    v[i].y = __fadd_rn(v[i].y, __fadd_rn(__fadd_rn(p0.y, p1.y), __fadd_rn(p2.y, p3.y)));
                                    v[i].z = __fadd_rn(v[i].z, __fadd_rn(__fadd_rn(p0.z, p1.z), __fadd_rn(p2.z, p3.z)));
                                    v[i].w = __fadd_rn(v[i].w, __fadd_rn(__fadd_rn(p0.w, p1.w), __fadd_rn(p2.w, p3.w)));
                                }
                            }
                        }
                        float sum = 0.0f;
#pragma unroll
                        for (int i = 0; i < PT; ++i) {
                            const int c = tid + i * NT;
                            if (c < nv) {
                                if (D.stage == ST_LN_EMB || D.stage == ST_LN_FOLD) reinterpret_cast<float4*>(x + (int64_t)r * d)[c] = v[i];   // only this CTA touches row r here
                                sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
                            }
                        }
                        sum = warp_sum(sum);
                        if (lane == 0) red[warp] = sum;
                        __syncthreads();
                        sum = 0.0f;
#pragma unroll
                        for (int w = 0; w < NW; ++w) sum += red[w];
                        const float mean = __fdiv_rn(sum, (float)d);
                        float q = 0.0f;
#pragma unroll
                        for (int i = 0; i < PT; ++i) {
                            if (tid + i * NT < nv) {
                                v[i].x = __fsub_rn(v[i].x, mean); v[i].y = __fsub_rn(v[i].y, mean);
                                v[i].z = __fsub_rn(v[i].z, mean); v[i].w = __fsub_rn(v[i].w, mean);
                                q = ln_sq_add4(q, v[i]);
                            }
                        }
                        q = warp_sum(q);
                        if (lane == 0) red[NW + warp] = q;
                        __syncthreads();
                        q = 0.0f;
#pragma unroll
                        for (int w = 0; w < NW; ++w) q += red[NW + w];
                        const float var = __fdiv_rn(q, (float)d);
                        const float den = LN_DEN(var, D.eps, a.eps_outside);
#pragma unroll
                        for (int i = 0; i < PT; ++i) {
                            const int c = tid + i * NT;
                            if (c < nv) {
                                const float4 o = ln_norm4(v[i], den, g4[i], b4[i]);
                                const int oks = D.ks, osl = (c * 4) / oks;   // slab-major output planes when the consuming linear stage splits K (oks == d: one slab)
                                store_frag(xn_hi + osl * (PL_ROWS * oks / 8), xn_lo + osl * (PL_ROWS * oks / 8), oks >> 5, r, c * 4 - osl * oks, o);
                            }
                        }
                    }
                } else if (D.kind == D5_KIND_ATTN) {
                    // ================= attention: self (causal over the row's ancestry) / cross (split over keys).
                    // Two (row, head[, split]) units per CTA at a time, 4 warps each (named barriers).
                    const bool is_cross = slot == SL_CROSS;
                    if (is_cross) fence_proxy_async();   // the ring aliases the planes written through the generic proxy
                    const int U = is_cross ? R * H * S : R * H;
                    const int grp = warp >> 2, wg = warp & 3, gt = tid & 127;
                    const KVT* ckvl = reinterpret_cast<const KVT*>(a.ckv) + (size_t)l * a.Mcap * 2 * d;
                    for (int u = blockIdx.x * 2 + grp; u < U; u += 2 * gridDim.x) {
                        int r, h, sp = 0;
                        if (is_cross) { sp = u % S; h = (u / S) % H; r = u / (S * H); }
                        else { r = u / H; h = u % H; }
                        if (gt < 16) {
                            float4 q4;
                            if (is_cross && cq_parts > 0) {   // (p0 + p1) + (p2 + p3), bias inside p0, then the (d/H)^-0.25 scale (EM_CQ)
                                const float4* pq = reinterpret_cast<const float4*>(yp + (int64_t)r * d + h * 64) + gt;
                                const float4 p0 = __ldcg(pq), p1 = __ldcg(pq + yps / 4);
                                const float4 p2 = cq_parts > 2 ? __ldcg(pq + 2 * (yps / 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
                                const float4 p3 = cq_parts > 3 ? __ldcg(pq + 3 * (yps / 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
                                q4.x = __fmul_rn(__fadd_rn(__fadd_rn(p0.x, p1.x), __fadd_rn(p2.x, p3.x)), scale);
                                q4.y = __fmul_rn(__fadd_rn(__fadd_rn(p0.y, p1.y), __fadd_rn(p2.y, p3.y)), scale);
                                q4.z = __fmul_rn(__fadd_rn(__fadd_rn(p0.z, p1.z), __fadd_rn(p2.z, p3.z)), scale);
                                q4.w = __fmul_rn(__fadd_rn(__fadd_rn(p0.w, p1.w), __fadd_rn(p2.w, p3.w)), scale);
                            } else {
                                q4 = __ldcg(reinterpret_cast<const float4*>(a.q + (int64_t)r * d + h * 64) + gt);
                            }
                            *reinterpret_cast<float4*>(qs + grp * 64 + gt * 4) = q4;
                        }
                        bar_named(1 + grp, 128);
                        int nk = p + 1;
                        AttnAcc A;
                        if (is_cross) {   // contiguous head-major block: 8-key batches by bulk copy into this warp's ring (aliases the planes, dead here)
                            const int w = __ldcg(a.row_window + r);
                            const int T = a.win_T[w];
                            const int per = (T + S - 1) / S;
                            const int kb0 = sp * per;
                            nk = max(0, min(T, kb0 + per) - kb0);
                            const KVT* kbase = ckvl + a.win_row_off[w] * (int64_t)(2 * d) + ((int64_t)h * T + kb0) * 128;
                            attn_warp_bulk<KV_STG, KVT>(qs + grp * 64, kbase, nk, wg, 4, kb0, reinterpret_cast<unsigned char*>(sm) + warp * RING_W,
                                                        kv_bar + warp * KV_STG, kv_count, A);
                        } else {
                            const int* anc = a.anc ? a.anc + (int64_t)r * t_max : nullptr;
                            auto kp = [&](int j) -> const KVT* {
                                const int rr = (anc && j < p) ? __ldcg(anc + j) : r + a.kv_row0;
                                return kcl + ((int64_t)rr * t_max + j) * d + h * 64;
                            };
                            auto vp = [&](int j) -> const KVT* {
                                const int rr = (anc && j < p) ? __ldcg(anc + j) : r + a.kv_row0;
                                return vcl + ((int64_t)rr * t_max + j) * d + h * 64;
                            };
                            if constexpr (sizeof(KVT) == 4) attn_warp(qs + grp * 64, nk, wg, 4, kp, vp, A);
                            else attn_warp_ring<RING_W / 2048>(qs + grp * 64, nk, wg, 4, kp, vp, reinterpret_cast<uint4*>(sm) + warp * (RING_W / 16), A);
                        }
                        if (lane < 4) {
#pragma unroll
                            for (int c = 0; c < 16; ++c) wo[warp * 64 + (is_cross ? attn_bulk_dim<KVT>(lane, c) : lane * 16 + c)] = A.o[c];
                        }
                        if (lane == 0) { wm[warp] = A.m; wl[warp] = A.l; }
                        bar_named(1 + grp, 128);
                        if (gt < 64) {
                            float M = -INFINITY;
#pragma unroll
                            for (int w2 = 0; w2 < 4; ++w2) M = fmaxf(M, wm[grp * 4 + w2]);
                            float Ls = 0.0f, o = 0.0f;
#pragma unroll
                            for (int w2 = 0; w2 < 4; ++w2) {
                                const float m = wm[grp * 4 + w2];
                                const float sc = m > -INFINITY ? expf(m - M) : 0.0f;
                                Ls += sc * wl[grp * 4 + w2];
                                o += sc * wo[(grp * 4 + w2) * 64 + gt];
                            }
                            if (!is_cross || S == 1) {
                                const int col = h * 64 + gt, asl = col / aks;   // slab-major planes: slab asl holds columns [asl * aks, +aks)
                                store_plane_elem(att_hi + asl * (PL_ROWS * aks / 8), att_lo + asl * (PL_ROWS * aks / 8), aks >> 5, r, col - asl * aks, __fdiv_rn(o, Ls));
                            } else {
                                const int64_t oi = ((int64_t)r * H + h) * S + sp;
                                a.part_o[oi * 64 + gt] = o;
                                if (gt == 0) { a.part_m[oi] = nk > 0 ? M : -INFINITY; a.part_l[oi] = Ls; }
                            }
                        }
                        bar_named(1 + grp, 128);
                    }
                } else {
                    // ================= one linear layer for all rows: out[r][n] = sum_k in[r][k] W[n][k] (+ bias)
                    const bool merge = D.stage == ST_CROSS && S > 1;
                    const bool lg = D.emit == EM_LOGITS;
                    const int ks = D.ks, nch_s = ks >> 8, nchunks_s = ks >> 5;   // this stage's K slab: chunks per warp / per row
                    const int n_tiles = D.N >> 4;
                    const int n_items = lg ? (int)gridDim.x : n_tiles * D.n_slabs;
                    int staged = -1;
                    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                        const int tile = lg ? 0 : item % n_tiles, slab = lg ? 0 : item / n_tiles;
                        if (!lg && !pf_valid) load_afrag(D, d, item, pf);
                        float prev[NE];
#pragma unroll
                        for (int e = 0; e < NE; ++e) {
                            const int idx = tid + e * NT;
                            prev[e] = (D.emit == EM_RESID && idx < 16 * RP && (idx >> 4) < R) ? __ldcg(x + (int64_t)(idx >> 4) * d + tile * 16 + (idx & 15)) : 0.0f;
                        }
                        if (slab != staged) {
                            staged = slab;
                            __syncthreads();
                            if (!merge) {
                                // ---- the producer wrote the planes in fragment order: plain asynchronous copy (rows < RP are a prefix)
                                const uint4* sh = (D.src == 2 ? hid_hi : D.src == 3 ? xn_hi : att_hi) + (int64_t)slab * (PL_ROWS * ks / 8);
                                const uint4* sl = sh + (D.src == 2 ? 4 * pl_plane : pl_plane);
                                const int n16 = NT8 * nchunks_s * 32;
                                // (bulk copies by one thread were measured here: 0.6 us faster in isolation -- scripts/ubench -- but 4 % slower in
                                // the kernel, profiles/r02_dec5_ab.txt; the per-thread cp.async stays)
                                for (int i = tid; i < n16; i += NT) {
                                    cp_async16(xhi + i, sh + i);
                                    cp_async16(xlo + i, sl + i);
                                }
                                cp_async_wait_all();
                            } else {
                                // ---- merge the cross-attention split partials (S > 1) while staging
                                float* wn = red;   // [RP][H][S] normalised split weights
                                for (int i = tid; i < RP * H; i += NT) {
                                    const int r = i / H, h = i % H;
                                    if (r < R) {
                                        const int64_t o = ((int64_t)r * H + h) * S;
                                        float pm[16], pl[16];
#pragma unroll
                                        for (int s = 0; s < 16; ++s) {
                                            pm[s] = s < S ? __ldcg(a.part_m + o + s) : -INFINITY;
                                            pl[s] = s < S ? __ldcg(a.part_l + o + s) : 0.0f;
                                        }
                                        float M = -INFINITY;
#pragma unroll
                                        for (int s = 0; s < 16; ++s) M = fmaxf(M, pm[s]);
                                        float den = 0.0f;
#pragma unroll
                                        for (int s = 0; s < 16; ++s) {
                                            pm[s] = pm[s] > -INFINITY ? expf(pm[s] - M) : 0.0f;
                                            den += pm[s] * pl[s];
                                        }
#pragma unroll
                                        for (int s = 0; s < 16; ++s)
                                            if (s < S) wn[i * S + s] = __fdiv_rn(pm[s], den);
                                    } else {
                                        for (int s = 0; s < S; ++s) wn[i * S + s] = 0.0f;
                                    }
                                }
                                __syncthreads();
                                for (int i = tid; i < RP * ks / 4; i += NT) {   // 4 consecutive dims of one (row, head), columns of this K slab
                                    const int r = (i * 4) / ks, cl = (i * 4) % ks, c = slab * ks + cl, rc = min(r, R - 1);
                                    const int h = c / 64;
                                    const float4* po = reinterpret_cast<const float4*>(a.part_o + (((int64_t)rc * H + h) * S) * 64 + (c & 63));
                                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
                                    for (int s = 0; s < S; ++s) {
                                        const float4 v = __ldcg(po + s * 16);
                                        const float wgt = wn[(r * H + h) * S + s];
                                        acc.x = fmaf(wgt, v.x, acc.x); acc.y = fmaf(wgt, v.y, acc.y);
                                        acc.z = fmaf(wgt, v.z, acc.z); acc.w = fmaf(wgt, v.w, acc.w);
                                    }
                                    store_frag(xhi, xlo, nchunks_s, r, cl, acc);
                                }
                            }
                        }
                        __syncthreads();
                        if (!lg) {
                            const AFrag cur = pf;
                            pf_valid = false;
                            if (item + (int)gridDim.x < n_items) { load_afrag(D, d, item + gridDim.x, pf); pf_valid = true; }   // next item of this CTA
                            float ah[NT8][4], al[NT8][4];
#pragma unroll
                            for (int j = 0; j < NT8; ++j)
#pragma unroll
                                for (int c = 0; c < 4; ++c) { ah[j][c] = 0.0f; al[j][c] = 0.0f; }
#pragma unroll
                            for (int c = 0; c < MAXCH; ++c) {
                                if (c < nch_s) {
                                    const int chunk = warp * nch_s + c;
#pragma unroll
                                    for (int j = 0; j < NT8; ++j) {
                                        const uint4 bh = xhi[(j * nchunks_s + chunk) * 32 + lane];
                                        const uint4 bl = xlo[(j * nchunks_s + chunk) * 32 + lane];
                                        mma16816(ah[j], cur.r0[c].x, cur.r8[c].x, cur.r0[c].y, cur.r8[c].y, bh.x, bh.y);
                                        mma16816(ah[j], cur.r0[c].z, cur.r8[c].z, cur.r0[c].w, cur.r8[c].w, bh.z, bh.w);
                                        mma16816(al[j], cur.r0[c].x, cur.r8[c].x, cur.r0[c].y, cur.r8[c].y, bl.x, bl.y);
                                        mma16816(al[j], cur.r0[c].z, cur.r8[c].z, cur.r0[c].w, cur.r8[c].w, bl.z, bl.w);
                                    }
                                }
                            }
                            // C fragment: c0,c1 -> (feature g, rows 2t, 2t+1), c2,c3 -> (feature g+8, rows 2t, 2t+1)
                            {
                                const int g = lane >> 2, t = lane & 3;
                                float* my = red + warp * (RP * RED_LD);
#pragma unroll
                                for (int j = 0; j < NT8; ++j) {
                                    const int r0 = j * 8 + 2 * t;
                                    my[r0 * RED_LD + g] = hl_join(ah[j][0], al[j][0]);
                                    my[(r0 + 1) * RED_LD + g] = hl_join(ah[j][1], al[j][1]);
                                    my[r0 * RED_LD + g + 8] = hl_join(ah[j][2], al[j][2]);
                                    my[(r0 + 1) * RED_LD + g + 8] = hl_join(ah[j][3], al[j][3]);
                                }
                            }
                            __syncthreads();
#pragma unroll
                            for (int e = 0; e < NE; ++e) {
                                const int idx = tid + e * NT;
                                if (idx < 16 * RP) {
                                    const int f = idx & 15, r = idx >> 4, n = tile * 16 + f;
                                    float v = cur.bias;
#pragma unroll
                                    for (int w = 0; w < NW; ++w) v += red[w * (RP * RED_LD) + r * RED_LD + f];
                                    if (r < R) {
                                        switch (D.emit) {
                                            case EM_QKV:      // mod.rs:429-431; q and k carry the (d/H)^-0.25 scale (:500-503)
                                                if (n < 2 * d) v = __fmul_rn(v, scale);
                                                if (n < d) a.q[(int64_t)r * d + n] = v;
                                                else if (n < 2 * d) kcl[((int64_t)(r + a.kv_row0) * t_max + p) * d + (n - d)] = (KVT)v;   // fp16 cache: round-to-nearest
                                                else vcl[((int64_t)(r + a.kv_row0) * t_max + p) * d + (n - 2 * d)] = (KVT)v;
                                                break;
                                            case EM_RESID:    // x += out-projection (mod.rs:346-347)
                                                x[(int64_t)r * d + n] = __fadd_rn(prev[e], v);
                                                break;
                                            case EM_CQ:       // cross query (mod.rs:483)
                                                a.q[(int64_t)r * d + n] = __fmul_rn(v, scale);
                                                break;
                                            case EM_HID:      // gelu(LN(x) W1 + b1) (mod.rs:377-378), written as fragment-order planes
                                                store_plane_elem(hid_hi + (n / hks) * (PL_ROWS * hks / 8), hid_lo + (n / hks) * (PL_ROWS * hks / 8), hks >> 5, r, n % hks, gelu_erf(v));
                                                break;
                                            default:          // EM_PART: MLP2 partial sum of this K slab
                                                a.ypart[slab * yps + (int64_t)r * d + n] = v;
                                                break;
                                        }
                                    }
                                }
                            }
                        } else {
                            // ================= logits = LN(x) tok_emb^T (mod.rs:155-156) -> lgbuf[R][V]; a warp streams 16-row tiles of E
                            const __half* E = reinterpret_cast<const __half*>(D.W);
                            const int g = lane >> 2, t = lane & 3;
                            const int v_tiles = (V + 15) / 16, ngrp = d / (32 * GC);
                            // tile t: CTA t % grid, warp (t / grid) % NW -- every CTA streams the same number of tiles (+-1)
                            const int t0w = (int)blockIdx.x + (int)gridDim.x * warp, tstep = (int)gridDim.x * NW;
                            const int my_tiles = t0w < v_tiles ? (v_tiles - t0w + tstep - 1) / tstep : 0;
                            const int total = my_tiles * ngrp;
                            uint4 A0[GC][2], A1[GC][2];
                            auto load_grp = [&](int it, uint4 (&A)[GC][2]) {
                                const int vt = t0w + (it / ngrp) * tstep, grp = it % ngrp;
                                const int ra = min(vt * 16 + g, V - 1), rb = min(vt * 16 + g + 8, V - 1);
                                const uint4* pa = reinterpret_cast<const uint4*>(E + (int64_t)ra * d + grp * (32 * GC) + t * 8);
                                const uint4* pb = reinterpret_cast<const uint4*>(E + (int64_t)rb * d + grp * (32 * GC) + t * 8);
#pragma unroll
                                for (int c = 0; c < GC; ++c) { A[c][0] = __ldg(pa + c * 4); A[c][1] = __ldg(pb + c * 4); }
                            };
                            if (total > 0) load_grp(0, A0);
                            float ah[NT8][4], al[NT8][4];
#pragma unroll 1
                            for (int it = 0; it < total; ++it) {
                                const int grp = it % ngrp;
                                if (grp == 0) {
#pragma unroll
                                    for (int j = 0; j < NT8; ++j)
#pragma unroll
                                        for (int c = 0; c < 4; ++c) { ah[j][c] = 0.0f; al[j][c] = 0.0f; }
                                }
                                if (it + 1 < total) load_grp(it + 1, A1);
#pragma unroll
                                for (int c = 0; c < GC; ++c) {
                                    const int chunk = grp * GC + c;
#pragma unroll
                                    for (int j = 0; j < NT8; ++j) {
                                        const uint4 bh = xhi[(j * nchunks + chunk) * 32 + lane];
                                        const uint4 bl = xlo[(j * nchunks + chunk) * 32 + lane];
                                        mma16816(ah[j], A0[c][0].x, A0[c][1].x, A0[c][0].y, A0[c][1].y, bh.x, bh.y);
                                        mma16816(ah[j], A0[c][0].z, A0[c][1].z, A0[c][0].w, A0[c][1].w, bh.z, bh.w);
                                        mma16816(al[j], A0[c][0].x, A0[c][1].x, A0[c][0].y, A0[c][1].y, bl.x, bl.y);
                                        mma16816(al[j], A0[c][0].z, A0[c][1].z, A0[c][0].w, A0[c][1].w, bl.z, bl.w);
                                    }
                                }
                                if (grp == ngrp - 1) {
                                    const int n0 = (t0w + (it / ngrp) * tstep) * 16;
#pragma unroll
                                    for (int j = 0; j < NT8; ++j) {
                                        const int r0 = j * 8 + 2 * t;
#pragma unroll
                                        for (int c = 0; c < 4; ++c) {
                                            const int n = n0 + g + (c >> 1) * 8, r = r0 + (c & 1);
                                            if (n < V && r < R) a.lgbuf[(int64_t)r * V + n] = hl_join(ah[j][c], al[j][c]);
                                        }
                                    }
                                }
#pragma unroll
                                for (int c = 0; c < GC; ++c) { A0[c][0] = A1[c][0]; A0[c][1] = A1[c][1]; }
                            }
                        }
                    }
                    __syncthreads();
                }
                // prefetch the first A fragments of the NEXT linear stage: weights do not depend on activations
                if (!pf_valid) {
                    int l2 = l, s2 = -1;
                    if (slot < SL_QKV) s2 = SL_QKV;
                    else if (slot < SL_OUT) s2 = SL_OUT;
                    else if (slot < SL_CQ) s2 = SL_CQ;
                    else if (slot < SL_COUT) s2 = SL_COUT;
                    else if (slot < SL_MLP1) s2 = SL_MLP1;
                    else if (slot < SL_MLP2) s2 = SL_MLP2;
                    else if (slot == SL_MLP2) {
                        if (l + 1 < L) { l2 = l + 1; s2 = SL_QKV; }
                        else if (!want_logits && step + 1 < a.n_steps) { l2 = 0; s2 = SL_QKV; }
                    }
                    if (s2 >= 0) {
                        const GemmDesc& Dn = ds[l2 * 16 + s2];
                        if ((int)blockIdx.x < (Dn.N >> 4) * Dn.n_slabs) { load_afrag(Dn, d, blockIdx.x, pf); pf_valid = true; }
                    }
                }
                WB_TRACE();
                grid_sync(a.bar, gen);
                WB_TRACE();
            }
        }
        if (want_logits) {
            // ================= per (row, slice): special-token mask (transcribe.rs:271-275), max, sum-exp, top candidates
            const int NSL = a.lg_slices;
            {
                const bool use_mask = SPECIAL_MASKED(a, p);
                const int per = (V + NSL - 1) / NSL;
                // k == 1 (greedy): a compact scan -- running (max, sum-exp) and the best (value, lowest index); this code runs
                // once per step, i.e. from a cold instruction cache, so its size is its cost
                if (a.k == 1) {
                    for (int u = blockIdx.x; u < R * NSL; u += gridDim.x) {
                        const int r = u / NSL, sl = u % NSL;
                        const int n_begin = sl * per, n_end = min(V, n_begin + per);
                        const float* row = a.lgbuf + (int64_t)r * V;
                        float m_run = -INFINITY, s_run = 0.0f, bv = -INFINITY;
                        int bi = INT_MAX;
                        // the id whose logit the greedy loop's EOT test reads, when this slice holds it
                        const int eot_cap = a.loop_rules && a.eot >= n_begin && a.eot < n_end ? a.eot : -1;
#pragma unroll 1
                        for (int n0 = n_begin + tid; n0 < n_end; n0 += NT * 8) {
                            float val[8];
                            unsigned char spf[8];
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const int n = min(n0 + i * NT, n_end - 1);
                                val[i] = __ldcg(row + n);
                                spf[i] = use_mask ? a.is_special[n] : (unsigned char)0;
                            }
                            float bm = -INFINITY;
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                if (spf[i]) val[i] = __fadd_rn(val[i], -INFINITY);
                                if (n0 + i * NT >= n_end) val[i] = -INFINITY;
                                bm = fmaxf(bm, val[i]);
                                if (val[i] > bv) { bv = val[i]; bi = n0 + i * NT; }   // indices grow: ties keep the lower id
                                if (n0 + i * NT == eot_cap) a.eot_logit[r] = val[i];
                            }
                            if (bm > -INFINITY) {
                                const float mn = fmaxf(m_run, bm);
                                float acc = s_run * expf(m_run - mn);
#pragma unroll
                                for (int i = 0; i < 8; ++i) acc += val[i] > -INFINITY ? expf(val[i] - mn) : 0.0f;
                                s_run = acc;
                                m_run = mn;
                            }
                        }
                        float* rec = red + warp * 4;
#pragma unroll 1
                        for (int pass = 0; pass < 2; ++pass) {   // pass 0: lanes of a warp, pass 1: the 8 warp records (one code path)
                            if (pass == 1) {
                                __syncthreads();
                                if (warp != 0) break;
                                m_run = lane < NW ? red[lane * 4] : -INFINITY;
                                s_run = lane < NW ? red[lane * 4 + 1] : 0.0f;
                                bv = lane < NW ? red[lane * 4 + 2] : -INFINITY;
                                bi = lane < NW ? __float_as_int(red[lane * 4 + 3]) : INT_MAX;
                            }
#pragma unroll 1
                            for (int off = 1; off < 32; off <<= 1) {
                                softmax_merge(m_run, s_run, __shfl_xor_sync(0xffffffffu, m_run, off), __shfl_xor_sync(0xffffffffu, s_run, off));
                                cand_xor(bv, bi, off);
                            }
                            if (pass == 0 && lane == 0) { rec[0] = m_run; rec[1] = s_run; rec[2] = bv; rec[3] = __int_as_float(bi); }
                        }
                        if (tid == 0) {   // the top-1 record
                            const int64_t o = (int64_t)sl * R + r;
                            a.lg_m[o] = m_run;
                            a.lg_s[o] = s_run;
                            a.lg_v[o] = bv;
                            a.lg_i[o] = bi;
                        }
                        __syncthreads();
                    }
                } else
                for (int u = blockIdx.x; u < R * NSL; u += gridDim.x) {
                    const int r = u / NSL, sl = u % NSL;
                    const int n_begin = sl * per, n_end = min(V, n_begin + per);
                    const float* row = a.lgbuf + (int64_t)r * V;
                    float m_run = -INFINITY, s_run = 0.0f;
                    Cand<KC> cand;
                    cand.init();
#pragma unroll 1
                    for (int n0 = n_begin + tid; n0 < n_end; n0 += NT * 8) {
                        float val[8];
                        unsigned char spf[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) {   // all loads of the batch first (clamped addresses, no control flow in between)
                            const int n = min(n0 + i * NT, n_end - 1);
                            val[i] = __ldcg(row + n);
                            spf[i] = use_mask ? a.is_special[n] : (unsigned char)0;
                        }
                        float bm = -INFINITY;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            if (spf[i]) val[i] = __fadd_rn(val[i], -INFINITY);
                            if (n0 + i * NT >= n_end) val[i] = -INFINITY;
                            bm = fmaxf(bm, val[i]);
                        }
                        if (bm > -INFINITY) {   // one rescale per batch, then 8 independent exponentials
                            const float mn = fmaxf(m_run, bm);
                            float acc = s_run * expf(m_run - mn);
#pragma unroll
                            for (int i = 0; i < 8; ++i) acc += val[i] > -INFINITY ? expf(val[i] - mn) : 0.0f;
                            s_run = acc;
                            m_run = mn;
                        }
                        if (bm > cand.v[KC - 1]) {   // rarely taken once the candidates have warmed up (ties never replace: indices only grow)
#pragma unroll 1
                            for (int i = 0; i < 8; ++i) {
                                float rv = val[0];
#pragma unroll
                                for (int k = 1; k < 8; ++k) rv = (i == k) ? val[k] : rv;
                                if (n0 + i * NT < n_end) cand.push(rv, n0 + i * NT);
                            }
                        }
                    }
#pragma unroll 1
                    for (int off = 1; off < 32; off <<= 1) {
                        const float m2 = __shfl_xor_sync(0xffffffffu, m_run, off);
                        const float s2 = __shfl_xor_sync(0xffffffffu, s_run, off);
                        float cv[KC];
                        int ci[KC];
#pragma unroll
                        for (int k = 0; k < KC; ++k) { cv[k] = __shfl_xor_sync(0xffffffffu, cand.v[k], off); ci[k] = __shfl_xor_sync(0xffffffffu, cand.i[k], off); }
                        const float mn = fmaxf(m_run, m2);
                        const float e1 = m_run > -INFINITY ? expf(m_run - mn) : 0.0f;
                        const float e2 = m2 > -INFINITY ? expf(m2 - mn) : 0.0f;
                        s_run = s_run * e1 + s2 * e2;
                        m_run = mn;
#pragma unroll 1
                        for (int k = 0; k < a.k; ++k) {   // only the k best are ever needed (candidate lists are sorted)
                            float pv = cv[0];
                            int pi = ci[0];
#pragma unroll
                            for (int kk = 1; kk < KC; ++kk) { pv = (k == kk) ? cv[kk] : pv; pi = (k == kk) ? ci[kk] : pi; }
                            cand.push(pv, pi);
                        }
                    }
                    float* rec = red + warp * (2 + 2 * KC);
                    if (lane == 0) {
                        rec[0] = m_run;
                        rec[1] = s_run;
#pragma unroll
                        for (int k = 0; k < KC; ++k) { rec[2 + k] = cand.v[k]; rec[2 + KC + k] = __int_as_float(cand.i[k]); }
                    }
                    __syncthreads();
                    if (tid == 0) fold_records<KC>(a, red, NW, 2 + 2 * KC, a.k, (int64_t)sl * R + r);
                    __syncthreads();
                }
            }
            WB_TRACE();
            grid_sync(a.bar, gen);
            WB_TRACE();
            // ================= finish: log_softmax of the candidates, k best, greedy bookkeeping
            if (a.k == 1) {   // greedy: one warp per row over the NSL <= 16 slice records
                for (int r = blockIdx.x; r < R; r += gridDim.x)
                    if (warp == 0) finish_row_top1<1>(a, r, p, NSL);
            } else
            for (int r = blockIdx.x; r < R; r += gridDim.x) finish_row_topk<KC>(a, r, p, NSL, wm, reinterpret_cast<int*>(wl));
            WB_TRACE();
            grid_sync(a.bar, gen);
            WB_TRACE();
            // stop as soon as every search has produced EOT (beam.rs:22-27)
            if (a.greedy && rows_open(a) == 0) {
                if (blockIdx.x == 0 && tid == 0) decode_done(a, p + 1, 0, step + 1);
                return;
            }
        }
    }
    if (blockIdx.x == 0 && tid == 0) decode_done(a, a.pos0 + a.n_steps, rows_open(a), a.n_steps);
}

size_t dec5_smem_bytes(int d, int NT8, int L) {
    return std::max((size_t)2 * NT8 * (PLANE_COLS_MAX(d) / 32) * 32 * 16, (size_t)NW * RING_W) + sizeof(float) * ((size_t)NW * NT8 * 8 * RED_LD + 128 + 2 * NW + NW * 64) + (size_t)(L * 16 + 16) * sizeof(Dec5Desc) + NW * 8 * 8 + 64;
}

template <int NT8, typename KVT>
bool launch5_t(const DecArgs& a, int n_ctas, cudaStream_t st) {
    const size_t smem = dec5_smem_bytes(a.d, NT8, a.L);
    auto k = dec5_kernel<NT8, KVT>;
    static PerDeviceConfig cfg;   // per instantiation
    const bool fits = cfg.ensure(smem, [&] {
        if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        int per_sm = 0;
        WB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, NT, smem));
        return per_sm >= 1;
    });
    if (!fits) return false;
    void* args[] = {(void*)&a};
    WB_CUDA(cudaLaunchCooperativeKernel((void*)k, dim3(n_ctas), dim3(NT), args, smem, st));
    WB_LAUNCH_CHECK();
    return true;
}

// one launch of <= 32 rows; false when the configuration is not covered.  The split stage table serves launches whose cross
// attention is NOT split over keys (n_splits == 1: at least one (row, head) unit per SM, the batched shapes the split is for);
// small batches keep the unsplit stages, whose cross-out staging merges the key-split partials over all d columns.
bool launch5(DecArgs a, const Dec5Tables& t, int n_ctas, bool w_half, cudaStream_t st) {
    a.d5 = (a.n_splits == 1 && t.split.p != nullptr) ? t.split.p : t.unsplit.p;
    if (!w_half || a.R < 1 || a.R > 32 || a.d % 256 != 0 || a.d > 1280 || a.H * 64 != a.d || n_ctas < 32) return false;
    if (a.lgbuf == nullptr || a.ypart == nullptr || a.att_pl == nullptr || a.hid_pl == nullptr || a.d5 == nullptr || a.lg_slices < 1 || a.k > DEC5_KC) return false;
    if (a.n_splits > 16 || (size_t)a.R * a.H * a.n_splits > (size_t)NW * ((a.R + 7) / 8) * 8 * RED_LD) return false;   // cross-merge weights live in the reduction buffer
    const int nt8 = (a.R + 7) / 8;
#define WB_D5(NT8_) (a.kv_half ? launch5_t<NT8_, __half>(a, n_ctas, st) : launch5_t<NT8_, float>(a, n_ctas, st))
    if (nt8 == 1) return WB_D5(1);
    if (nt8 == 2) return WB_D5(2);
    if (nt8 == 3) return WB_D5(3);
    return WB_D5(4);
#undef WB_D5
}

}  // namespace

size_t dec5_plane_uint4(int d) { return (size_t)PL_ROWS * d / 8; }   // uint4 per global plane (one K slab of d columns)

void dec5_build_tables(const Model& m, int n_sm, Dec5Tables& t) {
    if (!m.fp16_exact) return;
    const int d = m.dims.n_text_state, L = m.dims.n_text_layer, V = m.dims.n_vocab;
    auto gemm = [&](Dec5Desc& q, const void* Wp, const float* bias, int N, int n_slabs, int stage, int emit, int src) {
        q.kind = D5_KIND_GEMM; q.W = Wp; q.bias = bias; q.N = N; q.n_slabs = n_slabs; q.stage = stage; q.emit = emit; q.src = src; q.ks = d;
    };
    auto ln = [&](Dec5Desc& q, const LayerNormW& w, int stage) {
        q.kind = D5_KIND_LN; q.g = w.g; q.b = w.b; q.eps = w.eps; q.stage = stage; q.ks = d;
    };
    // The d x d projections (out, cross query, cross out) have only d/16 feature tiles -- 48 of 132 CTAs busy for small.en, each
    // staging all K columns of every row.  When d/256 slabs x d/16 tiles still fit ONE round of the grid, they run as K slabs of
    // 256 columns (one 32-column chunk per warp): three times the CTAs, a third of the staging each; the partial sums go to
    // ypart and are folded, in a fixed order, by the consumer (the next LayerNorm stage / the cross-attention query load).
    const int psl = d / 256;
    const bool can_split = d % 256 == 0 && psl >= 2 && psl <= 4 && (d / 16) * psl <= n_sm;
    auto build = [&](bool split_dd, DevBuf<Dec5Desc>& dst) {
        std::vector<Dec5Desc> ds((size_t)L * 16 + 16);
        for (int l = 0; l < L; ++l) {
            const DecBlockW& B = m.dec[(size_t)l];
            Dec5Desc* q = ds.data() + (size_t)l * 16;
            ln(q[0], B.attn_ln, l == 0 ? D5_ST_LN_EMB : D5_ST_LN_FOLD);
            gemm(q[1], B.qkv.w16, B.qkv.b, 3 * d, 1, D5_ST_PLANES, D5_EM_QKV, 3);
            q[2].kind = D5_KIND_ATTN;
            gemm(q[3], B.out.w16, B.out.b, d, 1, D5_ST_PLANES, D5_EM_RESID, 1);
            ln(q[4], B.cross_ln, D5_ST_LN_X);
            gemm(q[5], B.cq.w16, B.cq.b, d, 1, D5_ST_PLANES, D5_EM_CQ, 3);
            q[6].kind = D5_KIND_ATTN;
            gemm(q[7], B.cout.w16, B.cout.b, d, 1, D5_ST_CROSS, D5_EM_RESID, 1);
            ln(q[8], B.mlp_ln, D5_ST_LN_X);
            gemm(q[9], B.mlp1.w16, B.mlp1.b, 4 * d, 1, D5_ST_PLANES, D5_EM_HID, 3);
            gemm(q[10], B.mlp2.w16, B.mlp2.b, d, 4, D5_ST_PLANES, D5_EM_PART, 2);
            // MLP2 K = 4d: 3 slabs of 4d/3 when that keeps the 8-warp K split (multiple of 256, <= 1280): d/16 tiles x 3 slabs
            // = 144 items for small.en -> fewer rounds than 192 items
            if ((4 * d) % 3 == 0 && (4 * d / 3) % 256 == 0 && 4 * d / 3 <= 1280) { q[10].n_slabs = 3; q[10].ks = 4 * d / 3; }
            if (split_dd) {
                for (int sl : {3, 5, 7}) { q[sl].n_slabs = psl; q[sl].ks = 256; q[sl].emit = D5_EM_PART; }
                q[4].stage = D5_ST_LN_FOLD; q[4].n_fold = psl; q[4].ks = 256;   // folds the out projection, feeds the split cross query
                q[8].stage = D5_ST_LN_FOLD; q[8].n_fold = psl;                  // folds the cross out projection
            }
            if (l > 0) q[0].n_fold = q[10].n_slabs;                             // folds MLP2 of the previous layer
        }
        ln(ds[(size_t)L * 16 + 11], m.dec_ln, D5_ST_LN_FOLD_NOPUB);
        ds[(size_t)L * 16 + 11].n_fold = ds[(size_t)(L - 1) * 16 + 10].n_slabs;
        gemm(ds[(size_t)L * 16 + 12], m.tok_emb16, nullptr, V, 1, D5_ST_PLANES, D5_EM_LOGITS, 3);
        dst.alloc(ds.size());
        WB_CUDA(cudaMemcpy(dst.p, ds.data(), ds.size() * sizeof(Dec5Desc), cudaMemcpyHostToDevice));
    };
    build(false, t.unsplit);
    if (can_split) build(true, t.split);
}

int launch_dec5(const DecArgs& a, const Dec5Tables& t, int n_ctas, bool w_half, cudaStream_t st) {
    if (a.R <= 32) return launch5(a, t, n_ctas, w_half, st) ? 1 : 0;
    // more rows than one launch takes (beams of many windows, BASELINE configs[4]: 48 windows x 5 beams per GPU): row groups
    // of 32, one launch each on the stream; rows are independent, ancestry entries stay absolute cache rows (kv_row0 = first
    // cache row of the group)
    if (!w_half || a.d % 256 != 0 || a.d > 1280 || a.k > DEC_KC) return 0;
    int gi = 0;
    for (int r0 = 0; r0 < a.R; r0 += 32, ++gi) {
        const int Rg = std::min(32, a.R - r0), d = a.d;
        DecArgs g = a;
        g.R = Rg; g.kv_row0 = r0;
        g.x += (int64_t)r0 * d; g.q += (int64_t)r0 * d; g.att += (int64_t)r0 * d; g.hid += (int64_t)r0 * 4 * d;
        g.row_window += r0;
        if (g.anc) g.anc += (int64_t)r0 * a.t_max;
        g.tokens += (int64_t)r0 * a.t_max; g.token_lp += (int64_t)r0 * a.t_max; g.cur_tok += r0; g.lengths += r0; g.finished += r0;
        if (g.eot_logit) g.eot_logit += r0;
        g.topk_id += (int64_t)r0 * a.k; g.topk_lp += (int64_t)r0 * a.k;
        if (g.logits_out) { g.logits_out += (int64_t)r0 * a.V; g.lgbuf = g.logits_out; }
        g.lg_slices = std::max(1, std::min(16, n_ctas / std::max(1, Rg)));
        g.n_splits = std::max(1, std::min(16, n_ctas / std::max(1, Rg * a.H)));
        g.steps_done += std::min(gi, 127); g.n_unfinished += std::min(gi, 127);
        WB_CUDA(cudaMemsetAsync(a.bar, 0, 4 * sizeof(unsigned int), st));
        if (!launch5(g, t, n_ctas, true, st)) fail(WB_ERR_UNSUPPORTED, "decoder5 rejected a row group");
    }
    return gi;
}

}  // namespace wb
