// Cluster / DSMEM persistent decoder for small batches (R <= 8 rows, d <= 512: tiny / base) on sm_90a.
//
// Same math and same single-launch structure as decoder3.cu (prefill + every greedy step in one kernel), but
// the per-layer stage chain no longer crosses the chip: ONE 16-CTA thread-block cluster owns one batch row.
//   * activations (q|k|v, attention output, out-projection deltas, MLP hidden) are exchanged by DSMEM
//     broadcast -- the producing warp stores each value into the same shared-memory slot of all 16 CTAs --
//     so every stage reads its input from LOCAL shared memory;
//   * stages are separated by the hardware cluster barrier (barrier.cluster arrive.release / wait.acquire,
//     ~0.2 us) instead of the 1.3 us grid barrier through L2 (decoder3.cu: 34 per step);
//   * weights do not depend on activations: the CTA's rows of the large matrices (Wqkv, W1, W2) are bulk-copied into
//     shared memory stages ahead, the small ones' rows loaded into registers BEFORE the barrier, so after the barrier
//     a stage is LayerNorm + FMAs on on-chip data;
//   * every CTA keeps its own copy of the row's residual stream x and applies the broadcast deltas itself.
// Only the vocabulary projection is chip-wide: x rows are published, a grid barrier, all 128 CTAs stream the
// tied-embedding matrix (fused mask / online softmax / top candidates), a grid barrier, one CTA per row
// finishes (log-softmax of the candidates, token, EOT), a grid barrier.  3 grid + 32 cluster barriers / step.
// Reference math: see decoder3.cu.  Greedy path only (beam steps use decoder3.cu).
#include <cooperative_groups.h>

#include "dec_common.cuh"

namespace cg = cooperative_groups;

namespace wb {

namespace {

// End of a stage: every CTA sends its slice of the stage output to all 16 CTAs of the cluster, then needs everybody's slice.
// D4_ASYNC 1: the slices travel as st.async stores that complete transaction bytes on an mbarrier of the RECEIVING CTA; a CTA
//   waits on its own mbarrier for the expected byte count -- no cluster barrier, no release fence on the sending side (the
//   fence + barrier.cluster.arrive was ~0.5 us per stage).  The all-to-all data dependence orders everything else: a CTA can
//   only send stage k+1 after it has received stage k from everyone, i.e. after everyone finished reading what stage k-1 sent.
// D4_ASYNC 0: plain remote stores + barrier.cluster arrive (release) / wait (acquire), the prefetch between the two.
#ifndef D4_ASYNC
#define D4_ASYNC 1
#endif
// IDX: stage (mbarrier) index, RXBYTES: bytes this CTA receives in the stage, SEND: lambda issuing this CTA's sends (staged
// values are complete: a __syncthreads precedes it), PF: lambda prefetching the next stage's static operands
#define D4_EXCHANGE(IDX, RXBYTES, SEND, PF)                  \
    do {                                                     \
        WB_FINE();                                           \
        __syncthreads();                                     \
        WB_FINE();                                           \
        SEND();                                              \
        WB_FINE();                                           \
        if (D4_ASYNC) {                                      \
            PF();                                            \
            WB_FINE();                                       \
            xwait(xbar + (IDX), (RXBYTES), lc & 1u);         \
        } else {                                             \
            cluster_arrive();                                \
            PF();                                            \
            WB_FINE();                                       \
            cluster_wait();                                  \
        }                                                    \
    } while (0)
// sub-stage time stamps (profiling builds only: -DD4_FINE=1)
#ifndef D4_FINE
#define D4_FINE 0
#endif
#if D4_FINE
#define WB_FINE() WB_TRACE()
#else
#define WB_FINE() do { } while (0)
#endif

constexpr int CS = 16;   // CTAs per cluster
constexpr int LG_NBUF = 3;                 // logits stage: ring slots per warp
constexpr int LG_RB = 8;                   // vocabulary rows per slot
constexpr int KV_STG = 4;                  // cross attention: stages (8 keys each) of the per-warp K/V ring
// cross K/V in L2: 1 kept with the weights (evict_last), 0 streamed (evict_first, the faster one on the H100 for fp32 and
// fp16 K/V: the kept set then outgrows what the L2 holds for reads from all SMs; DESIGN.md section 5)
#ifndef D4_L2_CKV_KEEP
#define D4_L2_CKV_KEEP 0
#endif
__device__ __forceinline__ uint64_t ckv_policy() { return D4_L2_CKV_KEEP ? l2_policy_evict_last() : l2_policy_evict_first(); }

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

template <int NR>
struct RowBias {
    float bias[NR];   // fetched before the barrier
    float bias_own;   // bias of row (lane >> 1): the row whose sum warp_reduce_owner leaves in this lane
};
template <int NR, int VPL>
struct RowRegs : RowBias<NR> {
    uint4 v[NR][VPL];
};

// biases of rows row0, row0 + step, ... -> registers
template <int NR>
__device__ __forceinline__ void load_bias(const float* __restrict__ bias, int row0, int step, RowBias<NR>& r) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < NR; ++i) r.bias[i] = __ldg(bias + row0 + i * step);
    r.bias_own = __ldg(bias + row0 + min(lane >> 1, NR - 1) * step);
}
// rows row0, row0 + step, ... of W[.][K] (fp16) -> registers; lane-strided 16-byte vectors
template <int NR, int VPL>
__device__ __forceinline__ void load_rows(const __half* __restrict__ W, const float* __restrict__ bias, int K, int row0, int step,
                                          RowRegs<NR, VPL>& r, uint64_t pol) {
    const int lane = threadIdx.x & 31, nv = K / 8;
    load_bias<NR>(bias, row0, step, r);
#pragma unroll
    for (int i = 0; i < NR; ++i) {
        const uint4* p = reinterpret_cast<const uint4*>(W + (int64_t)(row0 + i * step) * K);
#pragma unroll
        for (int j = 0; j < VPL; ++j) {
            const int v = j * 32 + lane;
            r.v[i][j] = v < nv ? ldg_l2(p + v, pol) : make_uint4(0, 0, 0, 0);
        }
    }
}
// acc[i] = <row i, xs> (all lanes)
// Sums of NR values over the warp with 16 + ... shuffles instead of 5 * NR: recursive halving on the value index -- after the
// rounds with lane offsets 16, 8, 4, 2 every lane holds ONE value (index lane >> 1), a last exchange completes it.  Returns
// the total of value (lane >> 1) (NR <= 16; values >= NR are zero padding).
template <int NR>
__device__ __forceinline__ float warp_reduce_owner(const float (&acc)[NR]) {
    const int lane = threadIdx.x & 31;
    float v8[8], v4[4], v2[2];
    {
        const bool up = lane & 16;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float lo = i < NR ? acc[i] : 0.0f, hi = i + 8 < NR ? acc[i + 8] : 0.0f;
            const float recv = __shfl_xor_sync(0xffffffffu, up ? lo : hi, 16);
            v8[i] = (up ? hi : lo) + recv;
        }
    }
    {
        const bool up = lane & 8;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float recv = __shfl_xor_sync(0xffffffffu, up ? v8[i] : v8[i + 4], 8);
            v4[i] = (up ? v8[i + 4] : v8[i]) + recv;
        }
    }
    {
        const bool up = lane & 4;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float recv = __shfl_xor_sync(0xffffffffu, up ? v4[i] : v4[i + 2], 4);
            v2[i] = (up ? v4[i + 2] : v4[i]) + recv;
        }
    }
    const bool up = lane & 2;
    float v = (up ? v2[1] : v2[0]) + __shfl_xor_sync(0xffffffffu, up ? v2[0] : v2[1], 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// wv(i, j): 16-byte vector j * 32 + lane of the warp's row i
template <int NR, int VPL, bool REDUCE, typename WV>
__device__ __forceinline__ void dot_rows(WV&& wv, const float* xs, int K, float (&acc)[NR]) {
    const int lane = threadIdx.x & 31, nv = K / 8;
#pragma unroll
    for (int i = 0; i < NR; ++i) acc[i] = 0.0f;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
        const int v = j * 32 + lane;
        if (v < nv) {
            const float4 x0 = *reinterpret_cast<const float4*>(xs + v * 8);
            const float4 x1 = *reinterpret_cast<const float4*>(xs + v * 8 + 4);
#pragma unroll
            for (int i = 0; i < NR; ++i) {
                float w[8];
                cvt8(wv(i, j), w);
                float a = acc[i];
                a = fmaf(w[0], x0.x, a); a = fmaf(w[1], x0.y, a); a = fmaf(w[2], x0.z, a); a = fmaf(w[3], x0.w, a);
                a = fmaf(w[4], x1.x, a); a = fmaf(w[5], x1.y, a); a = fmaf(w[6], x1.z, a); a = fmaf(w[7], x1.w, a);
                acc[i] = a;
            }
        }
    }
    if constexpr (REDUCE) {
#pragma unroll
        for (int i = 0; i < NR; ++i) acc[i] = warp_sum(acc[i]);
    }
}
// the warp's rows from registers (load_rows)
template <int NR, int VPL, bool REDUCE = true>
__device__ __forceinline__ void dot_rows1(const RowRegs<NR, VPL>& r, const float* xs, int K, float (&acc)[NR]) {
    dot_rows<NR, VPL, REDUCE>([&](int i, int j) { return r.v[i][j]; }, xs, K, acc);
}
// the same rows from shared memory: ws is the CTA's slice [NR * NW][K] (bulk_rows), row i of warp w is row w + i * NW
template <int NR, int VPL, bool REDUCE = true>
__device__ __forceinline__ void dot_rows1s(const uint8_t* ws, const float* xs, int K, float (&acc)[NR]) {
    const int lane = threadIdx.x & 31, nv = K / 8;
    const uint4* w = reinterpret_cast<const uint4*>(ws) + (threadIdx.x >> 5) * nv;
    dot_rows<NR, VPL, REDUCE>([&](int i, int j) { return w[i * NW * nv + j * 32 + lane]; }, xs, K, acc);
}
// rows [row0, row0 + n) of W[.][K] (fp16, one contiguous block) -> shared memory at dst: one bulk copy, completing on bar.
// Called by one thread; fence_proxy_async() orders the CTA's generic reads of dst (before a barrier) ahead of the copy.
__device__ __forceinline__ void bulk_rows(uint8_t* dst, const __half* W, int K, int row0, int n, uint64_t* bar) {
    const uint32_t bytes = (uint32_t)n * K * 2;
    fence_proxy_async();
    mbar_expect_tx(bar, bytes);
    bulk_g2s_l2(dst, W + (int64_t)row0 * K, bytes, bar, l2_policy_evict_last());
}

// 16 bytes -> shared memory of another CTA of the cluster, completing 16 transaction bytes on that CTA's mbarrier
__device__ __forceinline__ void st_async_v4(uint32_t raddr, const float4& v, uint32_t rbar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(raddr), "f"(v.x),
                 "f"(v.y), "f"(v.z), "f"(v.w), "r"(rbar)
                 : "memory");
}
// 16 bytes to CTA `dest`: dst / bar are LOCAL addresses of the destination array element and of the stage's mbarrier
__device__ __forceinline__ void put16(cg::cluster_group& cl, float* dst, uint64_t* bar, int dest, const float4& v) {
#if D4_ASYNC
    st_async_v4(mapa_u32(smem_u32(dst), (uint32_t)dest), v, mapa_u32(smem_u32(bar), (uint32_t)dest));
#else
    *reinterpret_cast<float4*>(cl.map_shared_rank(dst, dest)) = v;
#endif
}
// A CTA's contiguous slice of a stage output (CNT floats staged in local shared memory) -> the same slice of the destination
// array in every CTA of the cluster.  16-byte stores, consecutive lanes -> consecutive addresses of one destination.
template <int CNT>
__device__ __forceinline__ void put_slice(cg::cluster_group& cl, const float* stage_s, float* dst_local, uint64_t* bar) {
    static_assert(CNT % 4 == 0, "slice must be a whole number of 16-byte vectors");
    constexpr int Q = CNT / 4;
    for (int i = threadIdx.x; i < CS * Q; i += NT) {
        const int dest = i / Q, q = i - dest * Q;
        put16(cl, dst_local + 4 * q, bar, dest, reinterpret_cast<const float4*>(stage_s)[q]);
    }
}
// wait until `bytes` have arrived on this CTA's stage mbarrier (D4_ASYNC): thread 0 posts the expectation, everybody polls
__device__ __forceinline__ void xwait(uint64_t* bar, uint32_t bytes, uint32_t parity) {
    if (threadIdx.x == 0) mbar_expect_tx(bar, bytes);
    const uint32_t mb = smem_u32(bar);
    uint32_t done = 0;
    int spins = 0;
    while (!done) {
        done = mbar_try_wait(mb, parity);
        if (!done && ++spins > (1 << 24)) __trap();   // a lost message must not hang the GPU
    }
}

// The residual row x is double-buffered in shared memory (read one copy, write the other); every warp of the CTA loads it
// into registers (lane owns the float4s lane, lane+32, ...), applies the broadcast delta and runs LayerNorm ITSELF (two
// shuffle reductions, no block barrier); the 8 warps compute identical values, warp 0 writes the updated row back.
template <int PF>
struct XRegs {
    float4 v[PF];
};
__device__ __forceinline__ float4 add4(const float4& a, const float4& b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}
template <int PF>
__device__ __forceinline__ void x_update(XRegs<PF>& x, const float* src_s, const float* d_s, float* dst_s) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < PF; ++k)
        x.v[k] = add4(reinterpret_cast<const float4*>(src_s)[lane + 32 * k], reinterpret_cast<const float4*>(d_s)[lane + 32 * k]);
    if (dst_s != nullptr && threadIdx.x < 32) {
#pragma unroll
        for (int k = 0; k < PF; ++k) reinterpret_cast<float4*>(dst_s)[lane + 32 * k] = x.v[k];
    }
}
// gamma | beta of a LayerNorm a few stages ahead -> this WARP's private copy (2D floats), lane-private 16-byte cp.async
// (each lane copies exactly the vectors it reads in ln_warp): no register stall, no barrier; cp_async_wait_all() before use.
template <int D, int PF>
__device__ __forceinline__ void ln_fetch(float* lnp, const float* __restrict__ g, const float* __restrict__ b, uint64_t pol) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < PF; ++k) {
        cp_async16_l2(lnp + 4 * (lane + 32 * k), g + 4 * (lane + 32 * k), pol);
        cp_async16_l2(lnp + D + 4 * (lane + 32 * k), b + 4 * (lane + 32 * k), pol);
    }
}
// LayerNorm (burn 0.9 eps placement; fmaf square sum and reciprocal normalisation, prims.cuh ln_sq_fma4 / ln_norm4_rcp) of the
// warp's register copy of x -> out_s (shared memory).  Every warp stores the same values (identical arithmetic) and reads them
// back after its own stores.
template <int D, int PF>
__device__ __forceinline__ void ln_warp(XRegs<PF>& x, const float* gb_s, float eps, int eps_outside, float* out_s) {
    const int lane = threadIdx.x & 31;
    cp_async_wait_all();   // this lane's gamma / beta vectors (ln_fetch)
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < PF; ++k) s += (x.v[k].x + x.v[k].y) + (x.v[k].z + x.v[k].w);
    s = warp_sum(s);
    const float mean = __fdiv_rn(s, (float)D);
    float q = 0.0f;
#pragma unroll
    for (int k = 0; k < PF; ++k) {
        x.v[k].x = __fsub_rn(x.v[k].x, mean); x.v[k].y = __fsub_rn(x.v[k].y, mean);
        x.v[k].z = __fsub_rn(x.v[k].z, mean); x.v[k].w = __fsub_rn(x.v[k].w, mean);
        q = ln_sq_fma4(q, x.v[k]);
    }
    q = warp_sum(q);
    const float var = __fdiv_rn(q, (float)D);
    const float rinv = __fdiv_rn(1.0f, LN_DEN(var, eps, eps_outside));
#pragma unroll
    for (int k = 0; k < PF; ++k) {
        const float4 g = reinterpret_cast<const float4*>(gb_s)[lane + 32 * k];
        const float4 b = reinterpret_cast<const float4*>(gb_s + D)[lane + 32 * k];
        reinterpret_cast<float4*>(out_s)[lane + 32 * k] = ln_norm4_rcp(x.v[k], rinv, g, b);
    }
    __syncwarp();
}

template <int D, int RC, typename KVT>
__global__ void __launch_bounds__(NT, 1)
dec4_kernel(const DecArgs a) {
    extern __shared__ __align__(16) float sm[];
    cg::cluster_group cl = cg::this_cluster();
    constexpr int H = D / 64;
    constexpr int VPL = (D / 8 + 31) / 32;        // vectors per lane for K = D
    constexpr int VPL4 = (4 * D / 8 + 31) / 32;   // K = 4D
    constexpr int NR_QKV = 3 * D / (CS * NW), NR_D = D / (CS * NW), NR_H = 4 * D / (CS * NW);
    const int L = a.L, V = a.V, R = a.R, t_max = a.t_max;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = (int)cl.block_rank();
    const int row = blockIdx.x / CS;              // batch row of this cluster
    const bool active = row < R;

    float* lnp = sm + warp * 2 * D;   // [NW][2D] LayerNorm gamma | beta of the next LayerNorm, one private copy per warp
    float* qkv_s = sm + NW * 2 * D;   // [3D]  q | k | v of the current position
    float* att_s = qkv_s + 3 * D;     // [D]   attention output (self, then merged cross)
    float* dl_s = att_s + D;          // [D]   out-projection / MLP2 output incl. bias ("delta" for x)
    float* q2_s = dl_s + D;           // [D]   cross query
    float* hid_s = q2_s + D;          // [4D]
    float* part_s = hid_s + 4 * D;    // [CS][68] cross partials: M, L, -, -, o[64]
    float* wm = part_s + CS * 68;     // [NW]
    float* wl = wm + NW;              // [NW]
    float* wo = wl + NW;              // [NW][64]
    float* ao = wo + NW * 64;         // [64]
    float* ML = ao + 64;              // [2]
    constexpr int STG_N = 4 * D / CS > 68 ? 4 * D / CS : 68;
    float* stg_s = ML + 4;            // [STG_N] this CTA's slice of a stage output, staged for the 16-byte sends
    float* xb = stg_s + STG_N;        // [2][D] residual row x, two copies used alternately (read one, write the other)
    float* xn_s = xb + 2 * D;         // [D]   LayerNorm output (written identically by every warp)
    float* red = xn_s + D;            // [NW][8 rows][m, s, best value, best id] logits merge scratch (sized [NW*4][RC][6])
    constexpr int RINGW = (LG_NBUF * LG_RB * D * 2 > KV_STG * 8 * 128 * 4) ? LG_NBUF * LG_RB * D * 2 : KV_STG * 8 * 128 * 4;   // bytes of a warp's ring (logits rows / cross K/V batches)
    constexpr int LG_PITCH = D * 2;                                        // bytes per staged vocabulary row (rows contiguous: one bulk copy per block)
    uint8_t* ring = reinterpret_cast<uint8_t*>(red + NW * 4 * RC * 6);      // [NW][LG_NBUF][LG_RB][LG_PITCH]
    uint64_t* lg_bar = reinterpret_cast<uint64_t*>(ring + (size_t)NW * RINGW);   // [NW][LG_NBUF]
    uint64_t* kv_bar = lg_bar + NW * LG_NBUF;   // [NW][KV_STG] cross-attention K/V ring (aliases the logits ring: different stages)
    uint64_t* xbar = kv_bar + NW * KV_STG;      // [8] stage exchange barriers (D4_ASYNC): transaction bytes sent by the 16 CTAs of the cluster
    uint64_t* wt_bar = xbar + 8;                // [3] this CTA's Wqkv / W1 / W2 rows in the ring (each copy completes once per layer)
    uint4* pl_hi = reinterpret_cast<uint4*>(wt_bar + 4);   // logits stage: fragment-order fp16 hi plane of the 8 (padded) LayerNorm rows [D/32][32]
    uint4* pl_lo = pl_hi + (D / 32) * 32;                           // same, residual * 2^11
    // The large layer matrices come from shared memory (DESIGN.md section 5): this CTA's rows of Wqkv, W1 and W2 are one
    // contiguous block each, bulk-copied into the ring while it is otherwise idle.  Timeline of the ring within a layer:
    //   S1      Wqkv [QKV_OFF, +QKV_B)                  (issued during S7 of the previous layer, or after the vocabulary loop)
    //   S1-S2   self K/V staging, first 8 KB of each warp's RINGW
    //   S3-S5   cross K/V ring, first 16 KB of each warp's RINGW
    //   S5-S7   W1 [W1_OFF, +W1_B)                      (issued when S5's cross attention has released the ring)
    //   S5-S8   W2 [W2_OFF, +W2_B)                      (same)
    //   S7-S1   next layer's Wqkv                       (issued when S7 has read W1; W2 is still being read)
    //   last layer, logits positions: the vocabulary half-tiles take the whole ring once S8 has read W2
    constexpr int QKV_B = 3 * D / CS * D * 2, W1_B = 4 * D / CS * D * 2, W2_B = D / CS * 4 * D * 2;
    constexpr int QKV_OFF = 0, W1_OFF = 0, W2_OFF = W1_OFF + W1_B;
    static_assert(W2_OFF + W2_B <= NW * RINGW, "W1 and W2 must fit the ring");
    static_assert(QKV_OFF + QKV_B <= W2_OFF, "the next layer's Wqkv arrives while W2 is read: no overlap");
    static_assert(QKV_B % 16 == 0 && W1_B % 16 == 0 && W2_B % 16 == 0 && W2_OFF % 16 == 0, "bulk copies move 16-byte units");
    if (lane == 0) {
        for (int j = 0; j < KV_STG; ++j) mbar_init(kv_bar + warp * KV_STG + j, 1);
        for (int j = 0; j < LG_NBUF; ++j) mbar_init(lg_bar + warp * LG_NBUF + j, 1);
        if (warp == 0) {
            for (int j = 0; j < 8; ++j) mbar_init(xbar + j, 1);
            for (int j = 0; j < 3; ++j) mbar_init(wt_bar + j, 1);
        }
        mbar_fence_init();
    }
    cl.sync();                   // every CTA's stage barriers exist before the first remote store can target them
    unsigned int lc = 0;         // layers this CTA has run: phase parity of the stage barriers (each is used once per layer)
    unsigned int kv_count = 0;   // batches this warp has pushed through its K/V ring
    unsigned int lg_count = 0;   // blocks this warp has pushed through its ring since kernel start (slot / parity bookkeeping)
    unsigned int gen = 0;
    unsigned int lstep = 0;      // vocabulary steps this launch has finished (ticket / flag bookkeeping)
    int tr_n = 0;
    const float scale = a.qk_scale;
    // this CTA's rows of layer l's Wqkv -> the ring (thread 0: every reader of the region is behind a barrier)
    auto issue_qkv = [&](int l) {
        if (tid == 0) bulk_rows(ring + QKV_OFF, reinterpret_cast<const __half*>(a.layers[l].Wqkv), D, rank * (3 * D / CS), 3 * D / CS, wt_bar + 0);
    };
    // L2 plan (DESIGN.md section 5): the layer weights, LayerNorm parameters and self K/V are re-read at every position and
    // kept (evict_last); the vocabulary half-tiles and is_special are read once per position and go first (evict_first);
    // cross K/V follows D4_L2_CKV_KEEP; biases keep normal priority.
    // Every line marked evict_last goes back to normal priority before the kernel exits (all CTAs, the ranges split over the grid).
    auto demote = [&]() {
        const size_t gt = (size_t)blockIdx.x * NT + tid, gn = (size_t)gridDim.x * NT;
        for (int l = 0; l < L; ++l) {
            const DecLayer& W = a.layers[l];
            l2_demote(W.Wqkv, (size_t)3 * D * D * 2, gt, gn);
            l2_demote(W.Wo, (size_t)D * D * 2, gt, gn);
            l2_demote(W.Wcq, (size_t)D * D * 2, gt, gn);
            l2_demote(W.Wco, (size_t)D * D * 2, gt, gn);
            l2_demote(W.W1, (size_t)4 * D * D * 2, gt, gn);
            l2_demote(W.W2, (size_t)4 * D * D * 2, gt, gn);
            l2_demote(W.ln1_g, D * 4, gt, gn); l2_demote(W.ln1_b, D * 4, gt, gn); l2_demote(W.ln2_g, D * 4, gt, gn);
            l2_demote(W.ln2_b, D * 4, gt, gn); l2_demote(W.ln3_g, D * 4, gt, gn); l2_demote(W.ln3_b, D * 4, gt, gn);
        }
        l2_demote(a.lnf_g, D * 4, gt, gn);
        l2_demote(a.lnf_b, D * 4, gt, gn);
        const size_t kv_bytes = (size_t)L * a.Rmax * t_max * D * sizeof(KVT);
        l2_demote(a.kc, kv_bytes, gt, gn);
        l2_demote(a.vc, kv_bytes, gt, gn);
        if (D4_L2_CKV_KEEP) l2_demote(a.ckv, (size_t)L * a.Mcap * 2 * D * sizeof(KVT), gt, gn);
    };
    WB_TRACE();

    const __half* nullw = nullptr;
    (void)nullw;
    for (int step = 0; step < a.n_steps; ++step) {
        const int p = a.pos0 + step;
        const bool want_logits = p >= a.logits_from;
        // ---- vocabulary tiles of this warp (round robin over all warps of the grid).  The tied-embedding matrix does not depend
        // on the activations: every warp takes its first LG_NBUF half-tiles into its ring BEFORE the grid barrier -- warps of
        // clusters without a row right away, the others as soon as the last layer's cross attention has released the ring.
        constexpr int KH = D / 2, NCH = KH / 32;               // columns / 32-column chunks per half-tile
        constexpr uint32_t BLKB = 16 * KH * 2;                 // bytes per half-tile
        static_assert(LG_NBUF * LG_RB * D * 2 >= LG_NBUF * (int)BLKB, "ring slot too small");
        const __half* Et = reinterpret_cast<const __half*>(a.E_tiled);
        const int v_tiles = (V + 15) / 16;
        // tile t belongs to CTA t % grid and, inside it, to warp (t / grid) % NW: every CTA streams the same number of tiles (+-1) --
        // with tiles dealt to the warps of the whole grid in order, the first CTAs got 32 tiles and the last 24 (3242 tiles, 896 warps)
        const int t0w = (int)blockIdx.x + (int)gridDim.x * warp, tstep = (int)gridDim.x * NW;
        const int my_tiles = t0w < v_tiles ? (v_tiles - t0w + tstep - 1) / tstep : 0;
        const int total = my_tiles * 2;                        // half-tiles of this warp
        auto tile_of = [&](int i) { return t0w + i * tstep; };
        uint8_t* wring = ring + (size_t)warp * RINGW;
        uint64_t* wbar = lg_bar + warp * LG_NBUF;
        auto issue = [&](int it) {
            if (it < total && lane == 0) {
                const int vt = tile_of(it >> 1);
                const int slot = (int)((lg_count + (unsigned int)it) % LG_NBUF);
                mbar_expect_tx(wbar + slot, BLKB);
                bulk_g2s_l2(wring + (size_t)slot * BLKB, Et + ((int64_t)vt * 2 + (it & 1)) * 16 * KH, BLKB, wbar + slot, l2_policy_evict_first());
            }
        };
        uint4* gpl_hi = reinterpret_cast<uint4*>(a.att_pl);   // published final-LayerNorm rows: fragment-order fp16 hi / lo planes [D/32][32]
        uint4* gpl_lo = gpl_hi + (D / 32) * 32;
        if (want_logits && !active) {
#pragma unroll
            for (int j = 0; j < LG_NBUF; ++j) issue(j);
        }
        if (active) {
            // ---- embed (mod.rs:141-146): every CTA of the cluster builds its own copy of x
            const int tok = __ldcg(a.tokens + (int64_t)row * t_max + p);
            // cross attention geometry of this CTA: head = rank % H, the CTAs of a head split the keys
            const int xh = rank % H, xci = rank / H;
            const int xnch = (CS - xh + H - 1) / H;              // CTAs working on head xh
            const int xw = __ldcg(a.row_window + row);
            const int xT = a.win_T[xw];
            const int64_t xoff = a.win_row_off[xw] * (int64_t)(2 * D) + (int64_t)xh * xT * 128;   // head-major K | V block
            const int sub = lane >> 2, l4 = lane & 3;
            const bool self_fast = p + 1 <= NW * 16;             // self attention: every cached position fits one register batch
            constexpr int PF = D / 128;   // float4s of the row per lane
            static_assert(D % 128 == 0, "row must be a whole number of float4s per lane");
            int xsel = 0;                 // which copy of x is current
            XRegs<PF> x;
#pragma unroll
            for (int k = 0; k < PF; ++k)
                x.v[k] = add4(__ldg(reinterpret_cast<const float4*>(a.tok_emb + (int64_t)tok * D) + lane + 32 * k),
                              __ldg(reinterpret_cast<const float4*>(a.pos_emb + (int64_t)p * D) + lane + 32 * k));
            if (warp == 0) {
#pragma unroll
                for (int k = 0; k < PF; ++k) reinterpret_cast<float4*>(xb)[lane + 32 * k] = x.v[k];
            }
            RowBias<NR_QKV> b_qkv;
            load_bias<NR_QKV>(a.layers[0].bqkv, rank * (3 * D / CS) + warp, NW, b_qkv);
            if (step == 0) issue_qkv(0);   // later steps: issued by the previous step (last layer, or after its vocabulary loop)
            if (step == 0) ln_fetch<D, PF>(lnp, a.layers[0].ln1_g, a.layers[0].ln1_b, l2_policy_evict_last());   // later steps: fetched by the previous step's last layer
            __syncthreads();
            for (int l = 0; l < L; ++l) {
                const DecLayer& W = a.layers[l];
                KVT* kcl = reinterpret_cast<KVT*>(a.kc) + (size_t)l * a.Rmax * t_max * D;
                KVT* vcl = reinterpret_cast<KVT*>(a.vc) + (size_t)l * a.Rmax * t_max * D;
                // ================= S1: q | k | v = LN1(x) Wqkv + b
                if (l > 0) {   // += MLP2 of the previous layer
                    x_update<PF>(x, xb + xsel * D, dl_s, xb + (xsel ^ 1) * D);
                    xsel ^= 1;
                }
                ln_warp<D, PF>(x, lnp, W.ln1_eps, a.eps_outside, xn_s);
                ln_fetch<D, PF>(lnp, W.ln2_g, W.ln2_b, l2_policy_evict_last());
                {
                    float acc[NR_QKV];
                    mbar_wait(wt_bar + 0, lc & 1u);
                    dot_rows1s<NR_QKV, VPL, false>(ring + QKV_OFF, xn_s, D, acc);
                    float mine = warp_reduce_owner<NR_QKV>(acc);   // lanes 2i, 2i+1: sum of row i
                    mine = __fadd_rn(mine, b_qkv.bias_own);
                    const int j = warp + (lane >> 1) * NW;          // index inside this CTA's slice
                    if (rank * (3 * D / CS) + j < 2 * D) mine = __fmul_rn(mine, scale);
                    if (!(lane & 1) && (lane >> 1) < NR_QKV) stg_s[j] = mine;
                }
                RowRegs<NR_D, VPL> w_o;
                // self attention (next stage): the cached positions j < p of this head are copied (asynchronously, lane-private
                // slots of this warp's ring, free from S1's read of Wqkv until the cross K/V prefill of S3) ahead of their use -- they are from earlier
                // steps; position p itself is taken from the broadcast q|k|v row afterwards.  Key j = warp + NW*(u*8+sub).
                constexpr int SNV = sizeof(KVT) == 4 ? 4 : 2;   // 16-byte vectors per lane and tensor (16 dims)
                uint8_t* sring = ring + (size_t)warp * RINGW;
                auto pre_s2 = [&]() {
                    load_rows<NR_D, VPL>(reinterpret_cast<const __half*>(W.Wo), W.bo, D, rank * (D / CS) + warp, NW, w_o, l2_policy_evict_last());
                    if (rank < H && self_fast) {
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            const int j = warp + NW * (u * 8 + sub);
                            if (j < p) {
                                const int64_t o = ((int64_t)row * t_max + j) * D + rank * 64 + l4 * 16;
#pragma unroll
                                for (int c = 0; c < SNV; ++c) {
                                    cp_async16_l2(sring + ((u * 2 + 0) * 4 + c) * 512 + lane * 16, reinterpret_cast<const uint4*>(kcl + o) + c, l2_policy_evict_last());
                                    cp_async16_l2(sring + ((u * 2 + 1) * 4 + c) * 512 + lane * 16, reinterpret_cast<const uint4*>(vcl + o) + c, l2_policy_evict_last());
                                }
                            }
                        }
                    }
                };
                auto send_s1 = [&]() {
                    put_slice<3 * D / CS>(cl, stg_s, qkv_s + rank * (3 * D / CS), xbar + 0);
                    if (tid < 3 * D / CS) {   // k | v of this position -> cache (one coalesced run per CTA)
                        const int n = rank * (3 * D / CS) + tid;
                        const float v = stg_s[tid];
                        if (n >= 2 * D) vcl[((int64_t)row * t_max + p) * D + (n - 2 * D)] = (KVT)v;
                        else if (n >= D) kcl[((int64_t)row * t_max + p) * D + (n - D)] = (KVT)v;
                    }
                };
                D4_EXCHANGE(0, 3 * D * 4, send_s1, pre_s2);
                if (D4_ASYNC && !self_fast) cl.sync();   // the long-context path reads position p's k | v back from the cache: order the stores
                WB_TRACE();
                // ================= S2: self attention, head = rank (ranks >= H idle)
                if (rank < H) {
                    const int h = rank;
                    if (self_fast) {
                        cp_async_wait_all();
                        float q[16];
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const float4 t4 = *reinterpret_cast<const float4*>(qkv_s + h * 64 + l4 * 16 + c * 4);
                            q[c * 4] = t4.x; q[c * 4 + 1] = t4.y; q[c * 4 + 2] = t4.z; q[c * 4 + 3] = t4.w;
                        }
                        AttnAcc A;
                        A.m = -INFINITY;
                        A.l = 0.0f;
#pragma unroll
                        for (int c = 0; c < 16; ++c) A.o[c] = 0.0f;
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            const int j = warp + NW * (u * 8 + sub);
                            float4 skk[4], svv[4];
                            if (j < p) {
                                if constexpr (sizeof(KVT) == 4) {
#pragma unroll
                                    for (int c = 0; c < 4; ++c) {
                                        skk[c] = *reinterpret_cast<const float4*>(sring + ((u * 2 + 0) * 4 + c) * 512 + lane * 16);
                                        svv[c] = *reinterpret_cast<const float4*>(sring + ((u * 2 + 1) * 4 + c) * 512 + lane * 16);
                                    }
                                } else {
#pragma unroll
                                    for (int c = 0; c < 2; ++c) {
                                        float w8[8];
                                        cvt8(*reinterpret_cast<const uint4*>(sring + ((u * 2 + 0) * 4 + c) * 512 + lane * 16), w8);
                                        skk[2 * c] = make_float4(w8[0], w8[1], w8[2], w8[3]); skk[2 * c + 1] = make_float4(w8[4], w8[5], w8[6], w8[7]);
                                        cvt8(*reinterpret_cast<const uint4*>(sring + ((u * 2 + 1) * 4 + c) * 512 + lane * 16), w8);
                                        svv[2 * c] = make_float4(w8[0], w8[1], w8[2], w8[3]); svv[2 * c + 1] = make_float4(w8[4], w8[5], w8[6], w8[7]);
                                    }
                                }
                            } else {
#pragma unroll
                                for (int c = 0; c < 4; ++c) { skk[c] = make_float4(0.f, 0.f, 0.f, 0.f); svv[c] = skk[c]; }
                            }
                            if (j == p) {   // the current position: from the broadcast row, rounded like the cache entry
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    float4 k4 = *reinterpret_cast<const float4*>(qkv_s + D + h * 64 + l4 * 16 + c * 4);
                                    float4 v4 = *reinterpret_cast<const float4*>(qkv_s + 2 * D + h * 64 + l4 * 16 + c * 4);
                                    if constexpr (sizeof(KVT) == 2) {
                                        k4 = make_float4((float)(KVT)k4.x, (float)(KVT)k4.y, (float)(KVT)k4.z, (float)(KVT)k4.w);
                                        v4 = make_float4((float)(KVT)v4.x, (float)(KVT)v4.y, (float)(KVT)v4.z, (float)(KVT)v4.w);
                                    }
                                    skk[c] = k4;
                                    svv[c] = v4;
                                }
                            }
                            attn_regs_step(q, skk, svv, j <= p, A);
                        }
                        attn_merge_subs(A);
                        attn_cta_tail(A, wm, wl, wo, ao, ML);
                    } else {
                        const KVT* kb = kcl + h * 64;
                        const KVT* vb = vcl + h * 64;
                        auto kp = [&](int j) { return kb + ((int64_t)row * t_max + j) * D; };
                        auto vp = [&](int j) { return vb + ((int64_t)row * t_max + j) * D; };
                        attn_cta(qkv_s + h * 64, p + 1, kp, vp, wm, wl, wo, ao, ML);
                    }
                }
                auto send_s2 = [&]() {   // the 6 head CTAs: 64 normalised values -> every CTA (thread = destination x float4)
                    if (rank < H) {
                        const int dest = tid >> 4, q = tid & 15;
                        const float4 o4 = reinterpret_cast<const float4*>(ao)[q];
                        const float den = ML[1];
                        put16(cl, att_s + rank * 64 + 4 * q, xbar + 1, dest,
                              make_float4(__fdiv_rn(o4.x, den), __fdiv_rn(o4.y, den), __fdiv_rn(o4.z, den), __fdiv_rn(o4.w, den)));
                    }
                };
                auto pf_none = [&]() {};
                D4_EXCHANGE(1, D * 4, send_s2, pf_none);
                WB_TRACE();
                // ================= S3: delta = att Wo + bo
                {
                    float acc[NR_D];
                    dot_rows1<NR_D, VPL>(w_o, att_s, D, acc);
                    WB_FINE();
                    if (lane == 0) {
#pragma unroll
                        for (int i = 0; i < NR_D; ++i) stg_s[warp + i * NW] = __fadd_rn(acc[i], w_o.bias[i]);
                    }
                }
                RowRegs<NR_D, VPL> w_cq;
                auto pre_s4 = [&]() {
                    load_rows<NR_D, VPL>(reinterpret_cast<const __half*>(W.Wcq), W.bcq, D, rank * (D / CS) + warp, NW, w_cq, l2_policy_evict_last());
                    // first batches of this layer's cross K/V: static data, two barriers ahead of its use; the ring held Wqkv and
                    // the self K/V (generic reads before the barrier)
                    fence_proxy_async();
                    attn_bulk_prefill<KV_STG, KVT, true>(reinterpret_cast<const KVT*>(a.ckv) + (size_t)l * a.Mcap * 2 * D + xoff, xT, xci * NW + warp,
                                                         xnch * NW, ring + (size_t)warp * RINGW, kv_bar + warp * KV_STG, kv_count, ckv_policy());
                };
                auto send_s3 = [&]() { put_slice<D / CS>(cl, stg_s, dl_s + rank * (D / CS), xbar + 2); };
                D4_EXCHANGE(2, D * 4, send_s3, pre_s4);
                WB_TRACE();
                // ================= S4: x += delta; cross query = LN2(x) Wcq + b
                x_update<PF>(x, xb + xsel * D, dl_s, xb + (xsel ^ 1) * D);
                xsel ^= 1;
                ln_warp<D, PF>(x, lnp, W.ln2_eps, a.eps_outside, xn_s);
                ln_fetch<D, PF>(lnp, W.ln3_g, W.ln3_b, l2_policy_evict_last());
                WB_FINE();
                {
                    float acc[NR_D];
                    dot_rows1<NR_D, VPL>(w_cq, xn_s, D, acc);
                    WB_FINE();
                    if (lane == 0) {
#pragma unroll
                        for (int i = 0; i < NR_D; ++i) stg_s[warp + i * NW] = __fmul_rn(__fadd_rn(acc[i], w_cq.bias[i]), scale);
                    }
                }
                RowRegs<NR_D, VPL> w_co;
                auto pre_s6 = [&]() { load_rows<NR_D, VPL>(reinterpret_cast<const __half*>(W.Wco), W.bco, D, rank * (D / CS) + warp, NW, w_co, l2_policy_evict_last()); };
                auto send_s4 = [&]() { put_slice<D / CS>(cl, stg_s, q2_s + rank * (D / CS), xbar + 3); };
                D4_EXCHANGE(3, D * 4, send_s4, pre_s6);
                WB_TRACE();
                // ================= S5: cross attention; head = rank % H, the CTAs of a head split the keys
                {
                    const int h = xh, ci = xci, nch = xnch, T = xT;
                    const KVT* kbase = reinterpret_cast<const KVT*>(a.ckv) + (size_t)l * a.Mcap * 2 * D + xoff;
                    // keys j == ci*NW + warp (mod nch*NW); the contiguous head-major block arrives in 8-key batches by bulk copy into
                    // this warp's ring (shared with the logits stage)
                    AttnAcc A;
                    attn_warp_bulk<KV_STG, KVT, true>(q2_s + h * 64, kbase, T, ci * NW + warp, nch * NW, 0, ring + (size_t)warp * RINGW,
                                                      kv_bar + warp * KV_STG, kv_count, A, true, ckv_policy());
                    if (lane < 4) {
#pragma unroll
                        for (int c = 0; c < 16; ++c) wo[warp * 64 + attn_bulk_dim<KVT>(lane, c)] = A.o[c];
                    }
                    if (lane == 0) { wm[warp] = A.m; wl[warp] = A.l; }
                    __syncthreads();
                    if (tid < 64) {
                        float M = -INFINITY;
#pragma unroll
                        for (int w2 = 0; w2 < NW; ++w2) M = fmaxf(M, wm[w2]);
                        float Ls = 0.0f, o = 0.0f;
#pragma unroll
                        for (int w2 = 0; w2 < NW; ++w2) {
                            const float m = wm[w2];
                            const float sc = m > -INFINITY ? expf(m - M) : 0.0f;
                            Ls += sc * wl[w2];
                            o += sc * wo[w2 * 64 + tid];
                        }
                        stg_s[4 + tid] = o;                      // this CTA's partial: M, L, -, -, o[64]
                        if (tid < 4) stg_s[tid] = tid == 0 ? M : tid == 1 ? Ls : 0.0f;
                    }
                }
                auto send_s5 = [&]() { put_slice<68>(cl, stg_s, part_s + rank * 68, xbar + 4); };
                auto pre_mlp = [&]() {   // the cross K/V ring is drained: this CTA's W1 and W2 rows, two and three stages ahead
                    if (tid == 0) {
                        bulk_rows(ring + W1_OFF, reinterpret_cast<const __half*>(W.W1), D, rank * (4 * D / CS), 4 * D / CS, wt_bar + 1);
                        bulk_rows(ring + W2_OFF, reinterpret_cast<const __half*>(W.W2), 4 * D, rank * (D / CS), D / CS, wt_bar + 2);
                    }
                };
                D4_EXCHANGE(4, CS * 68 * 4, send_s5, pre_mlp);
                WB_TRACE();
                // ================= S6: merge the head partials, delta = cross Wco + bco
                for (int c = tid; c < D; c += NT) {
                    const int h = c / 64;
                    float M = -INFINITY;
                    for (int k = h; k < CS; k += H) M = fmaxf(M, part_s[k * 68]);
                    float den = 0.0f, num = 0.0f;
                    for (int k = h; k < CS; k += H) {
                        const float m = part_s[k * 68];
                        const float wgt = m > -INFINITY ? expf(m - M) : 0.0f;
                        den += wgt * part_s[k * 68 + 1];
                        num += wgt * part_s[k * 68 + 4 + (c & 63)];
                    }
                    att_s[c] = __fdiv_rn(num, den);
                }
                __syncthreads();
                {
                    float acc[NR_D];
                    dot_rows1<NR_D, VPL>(w_co, att_s, D, acc);
                    if (lane == 0) {
#pragma unroll
                        for (int i = 0; i < NR_D; ++i) stg_s[warp + i * NW] = __fadd_rn(acc[i], w_co.bias[i]);
                    }
                }
                RowBias<NR_H> b_1;
                auto pre_s7 = [&]() { load_bias<NR_H>(W.b1, rank * (4 * D / CS) + warp, NW, b_1); };
                auto send_s6 = [&]() { put_slice<D / CS>(cl, stg_s, dl_s + rank * (D / CS), xbar + 5); };
                D4_EXCHANGE(5, D * 4, send_s6, pre_s7);
                WB_TRACE();
                // ================= S7: x += delta; hid = gelu(LN3(x) W1 + b1)
                x_update<PF>(x, xb + xsel * D, dl_s, xb + (xsel ^ 1) * D);
                xsel ^= 1;
                ln_warp<D, PF>(x, lnp, W.ln3_eps, a.eps_outside, xn_s);
                if (l == L - 1 && want_logits && rank == 0 && warp == 0) {   // this warp publishes the row: final LayerNorm next
                    ln_fetch<D, PF>(lnp, a.lnf_g, a.lnf_b, l2_policy_evict_last());
                } else {   // LN1 of the next layer, or of layer 0 for the next position
                    const DecLayer& Wn = a.layers[l + 1 < L ? l + 1 : 0];
                    ln_fetch<D, PF>(lnp, Wn.ln1_g, Wn.ln1_b, l2_policy_evict_last());
                }
                WB_FINE();
                {
                    float acc[NR_H];
                    mbar_wait(wt_bar + 1, lc & 1u);
                    dot_rows1s<NR_H, VPL, false>(ring + W1_OFF, xn_s, D, acc);
                    // lanes 2i, 2i+1 end up with the sum of row i: ONE erf-GELU per row instead of one per lane and row
                    float mine = warp_reduce_owner<NR_H>(acc);
                    mine = gelu_erf(__fadd_rn(mine, b_1.bias_own));
                    WB_FINE();
                    if (!(lane & 1) && (lane >> 1) < NR_H) stg_s[warp + (lane >> 1) * NW] = mine;
                }
                RowBias<NR_D> b_2;
                auto pre_s8 = [&]() {
                    load_bias<NR_D>(W.b2, rank * (D / CS) + warp, NW, b_2);
                    // W1 is read: the next layer's Wqkv (or layer 0's for the next position when this one has no vocabulary stage)
                    if (l + 1 < L) issue_qkv(l + 1);
                    else if (!want_logits && step + 1 < a.n_steps) issue_qkv(0);
                };
                auto send_s7 = [&]() { put_slice<4 * D / CS>(cl, stg_s, hid_s + rank * (4 * D / CS), xbar + 6); };
                D4_EXCHANGE(6, 4 * D * 4, send_s7, pre_s8);
                WB_TRACE();
                // ================= S8: delta = hid W2 + b2
                {
                    float acc[NR_D];
                    mbar_wait(wt_bar + 2, lc & 1u);
                    dot_rows1s<NR_D, VPL4>(ring + W2_OFF, hid_s, 4 * D, acc);
                    if (lane == 0) {
#pragma unroll
                        for (int i = 0; i < NR_D; ++i) stg_s[warp + i * NW] = __fadd_rn(acc[i], b_2.bias[i]);
                    }
                }
                auto pre_s1 = [&]() {
                    if (l + 1 < L) {
                        load_bias<NR_QKV>(a.layers[l + 1].bqkv, rank * (3 * D / CS) + warp, NW, b_qkv);
                    } else if (want_logits) {   // W2 is read, the ring is free until the next position: first vocabulary half-tiles of this warp
                        fence_proxy_async();    // generic reads of the ring before the bulk copies
#pragma unroll
                        for (int j = 0; j < LG_NBUF; ++j) issue(j);
                    }
                };
                auto send_s8 = [&]() { put_slice<D / CS>(cl, stg_s, dl_s + rank * (D / CS), xbar + 7); };
                D4_EXCHANGE(7, D * 4, send_s8, pre_s1);
                ++lc;
                WB_TRACE();
            }
            // final residual add + final LayerNorm (mod.rs:153-155); rank 0 publishes the row for the vocabulary projection, already
            // split into the fp16 hi / lo fragment planes every CTA needs (rows of other clusters land in the same planes)
            if (want_logits && rank == 0 && warp == 0) {
                x_update<PF>(x, xb + xsel * D, dl_s, nullptr);
                ln_warp<D, PF>(x, lnp, a.lnf_eps, a.eps_outside, xn_s);
                // RC == 4 (<= 4 rows): the residual plane of row r travels as batch column r + 4 of the SAME plane, so one MMA yields
                // the hi product in columns 0..3 and the lo product in columns 4..7 (half the tensor-core instructions of the stage)
#pragma unroll
                for (int k = 0; k < PF; ++k)
                    store_frag(gpl_hi, RC == 4 ? gpl_hi + 16 : gpl_lo, D / 32, row, 4 * (lane + 32 * k), reinterpret_cast<const float4*>(xn_s)[lane + 32 * k]);
                ln_fetch<D, PF>(lnp, a.layers[0].ln1_g, a.layers[0].ln1_b, l2_policy_evict_last());   // LN1 of layer 0 for the next position
            }
        }
        if (!want_logits) {   // prefill positions: clusters stay independent, no chip-wide step
            if (D4_ASYNC && active) cl.sync();   // this position's k | v stores (global) are ordered before the next position reads them
            continue;
        }
        WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
        // ================= logits (all CTAs): LN(x) tok_emb^T + mask + online softmax + candidates
        {
            const bool use_mask = SPECIAL_MASKED(a, p);
            const int eot_cap = a.loop_rules ? a.eot : -1;   // the id whose logit the greedy loop's EOT test reads
            // the published rows: fp16 hi / lo planes in MMA fragment order (decoder5.cu); rows >= R are never used
            for (int i = tid; i < 2 * (D / 32) * 32; i += NT) cp_async16(pl_hi + i, gpl_hi + i);   // pl_lo follows pl_hi in both spaces
            cp_async_wait_all();
            __syncthreads();
            WB_TRACE();
            // Swap-AB tensor-core product: a warp owns tiles of 16 vocabulary rows (M), the 8 padded batch rows are N, K = D.
            // The matrix is streamed as contiguous half-tiles [16][D/2] (one bulk copy each, TMA engine) through this warp's
            // ring -- LG_NBUF-1 copies in flight while the MMAs of the current half-tile run from shared memory.
            const int g = lane >> 2, t = lane & 3;
            float m_run[2] = {-INFINITY, -INFINITY}, s_run[2] = {0.0f, 0.0f}, bv[2] = {-INFINITY, -INFINITY};
            int bi[2] = {INT_MAX, INT_MAX};
            float ah[4], al[4];
            unsigned int sp01 = 0;   // is_special of vocabulary rows g / g+8 of the current tile: fetched a half-tile ahead of its use
#pragma unroll 1
            for (int it = 0; it < total; ++it) {
                const unsigned int cnt = lg_count + (unsigned int)it;
                const int slot = (int)(cnt % LG_NBUF);
                mbar_wait(wbar + slot, (cnt / LG_NBUF) & 1);
                const uint8_t* blk = wring + (size_t)slot * BLKB;
                const int half = it & 1;
                if (half == 0) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) { ah[c] = 0.0f; al[c] = 0.0f; }
                    if (use_mask) {
                        const int n = tile_of(it >> 1) * 16 + g;
                        sp01 = (n < V ? ldg_l2(a.is_special + n, l2_policy_evict_first()) : 0u) | (n + 8 < V ? ldg_l2(a.is_special + n + 8, l2_policy_evict_first()) << 8 : 0u);
                    }
                }
#pragma unroll
                for (int c = 0; c < NCH; ++c) {
                    // A fragment: 8 consecutive halves of rows g and g+8 (K permutation inside the 32-column chunk, decoder5.cu)
                    const uint4 a0 = *reinterpret_cast<const uint4*>(blk + (size_t)g * (KH * 2) + c * 64 + t * 16);
                    const uint4 a8 = *reinterpret_cast<const uint4*>(blk + (size_t)(g + 8) * (KH * 2) + c * 64 + t * 16);
                    const int chunk = half * NCH + c;
                    const uint4 bh = pl_hi[chunk * 32 + lane];
                    mma16816(ah, a0.x, a8.x, a0.y, a8.y, bh.x, bh.y);
                    mma16816(ah, a0.z, a8.z, a0.w, a8.w, bh.z, bh.w);
                    if constexpr (RC != 4) {
                        const uint4 bl = pl_lo[chunk * 32 + lane];
                        mma16816(al, a0.x, a8.x, a0.y, a8.y, bl.x, bl.y);
                        mma16816(al, a0.z, a8.z, a0.w, a8.w, bl.z, bl.w);
                    }
                }
                if (half == 1) {
                    // C fragment: c0,c1 -> (vocabulary row g, batch rows 2t, 2t+1), c2,c3 -> (row g+8, same batch rows)
                    const int n0 = tile_of(it >> 1) * 16;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const int n = n0 + g + (c >> 1) * 8, e = c & 1;
                        if constexpr (RC == 4) al[c] = __shfl_xor_sync(0xffffffffu, ah[c], 2);   // lo product of rows 2t, 2t+1: columns 2t+4, 2t+5 = lane t + 2
                        if (n < V && 2 * t + e < R) {   // RC == 4: R <= 4, i.e. lanes t < 2
                            const float raw = hl_join(ah[c], al[c]);
                            const float v = (use_mask && ((sp01 >> ((c >> 1) * 8)) & 0xffu)) ? __fadd_rn(raw, -INFINITY) : raw;
                            if (v > -INFINITY) softmax_add(m_run[e], s_run[e], v);
                            if (cand_better(v, n, bv[e], bi[e])) { bv[e] = v; bi[e] = n; }
                            if (n == eot_cap) a.eot_logit[2 * t + e] = v;
                        }
                    }
                }
                __syncwarp();   // every lane is done with the slot
                issue(it + LG_NBUF);
            }
            lg_count += (unsigned int)total;
            WB_TRACE();
            // merge the 8 lanes that share t (batch rows 2t, 2t+1), then the 8 warps through shared memory
#pragma unroll
            for (int e = 0; e < 2; ++e) {
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
                    softmax_merge(m_run[e], s_run[e], __shfl_xor_sync(0xffffffffu, m_run[e], off), __shfl_xor_sync(0xffffffffu, s_run[e], off));
                    cand_xor(bv[e], bi[e], off);
                }
                if (g == 0) {
                    float* rec = red + (warp * 8 + 2 * t + e) * 4;
                    rec[0] = m_run[e]; rec[1] = s_run[e]; rec[2] = bv[e]; rec[3] = __int_as_float(bi[e]);
                }
            }
            __syncthreads();
            if (active && step + 1 < a.n_steps) issue_qkv(0);   // every warp has drained its ring: layer 0's Wqkv for the next position
            if (tid < R) fold_records_top1(a, red + tid * 4, NW, 8 * 4, (int64_t)blockIdx.x * R + tid);
        }
        WB_TRACE();
        // ================= finish (greedy: beam.rs:9-37 with beam_size 1) by the LAST CTA to deliver its records, one warp
        // per row -- one flag wait instead of two grid barriers around the finish.
        ++lstep;
        __syncthreads();
        if (tid == 0) reinterpret_cast<int*>(ML)[2] = last_ticket(a.bar, lstep);
        __syncthreads();
        WB_TRACE();
        if (reinterpret_cast<int*>(ML)[2]) {
            __threadfence();
            // <= 128 co-resident CTAs: at most 4 records per lane
            for (int r = warp; r < R; r += NW) finish_row_top1<4>(a, r, p, gridDim.x);
            __syncthreads();
            if (tid == 0) release_flag(a.bar, lstep);
        }
        WB_TRACE();
        if (tid == 0) wait_flag(a.bar, lstep, 40000000000LL);   // ~20 s of SM clocks
        __syncthreads();
        WB_TRACE();
        if (rows_open(a) == 0) {
            if (active && tid == 0 && step + 1 < a.n_steps) mbar_wait(wt_bar + 0, lc & 1u);   // no bulk copy outlives the CTA
            if (blockIdx.x == 0 && tid == 0) decode_done(a, p + 1, 0, step + 1);
            demote();   // every CTA is past the flag: no evict_last load is left
            return;
        }
    }
    // after a prefill position clusters run independently: all of them finish their loads before any line is demoted
    if (a.n_steps > 0 && a.pos0 + a.n_steps - 1 < a.logits_from) grid_sync(a.bar, gen);
    demote();
    if (blockIdx.x == 0 && tid == 0) decode_done(a, a.pos0 + a.n_steps, rows_open(a), a.n_steps);
}

template <int D, int RC>
constexpr size_t dec4_smem() {
    return sizeof(float) * ((size_t)(2 * NW + 13) * D + (4 * D / CS > 68 ? 4 * D / CS : 68) + CS * 68 + 2 * NW + NW * 64 + 64 + 4 + (size_t)NW * 4 * RC * 6 + 16) +
           (size_t)NW * std::max(LG_NBUF * LG_RB * D * 2, KV_STG * 8 * 128 * 4) + NW * LG_NBUF * 8 + NW * KV_STG * 8 + 8 * 8 + 4 * 8 + (size_t)2 * (D / 32) * 32 * 16 + 16;
}
static_assert(dec4_smem<384, 8>() <= 227 * 1024 && dec4_smem<384, 4>() <= 227 * 1024, "dec4_kernel exceeds the shared memory of an sm_90 CTA");

template <int D, int RC, typename KVT>
bool launch4_t(const DecArgs& a, cudaStream_t st) {
    const void* k = (const void*)dec4_kernel<D, RC, KVT>;
    const size_t smem = dec4_smem<D, RC>();
    static ClusterLaunch cl;   // per instantiation
    const int n_cl = std::min(cl.capacity(k, CS, NT, smem, "dec4"), 8);   // one cluster per row, at most 8
    if (n_cl < 1 || a.R > n_cl) return false;
    void* args[] = {(void*)&a};
    cl.launch(k, CS, n_cl, NT, smem, args, st, "dec4");
    return true;
}

}  // namespace

// Returns false when this configuration is not covered.
bool launch_dec4(const DecArgs& a, bool w_half, cudaStream_t st) {
    if (!w_half || a.R > 8 || a.R < 1 || a.k != 1 || !a.greedy || a.use_cur_tok || a.anc != nullptr || a.logits_out != nullptr) return false;
    if (a.H * 64 != a.d || a.H > CS || a.E_tiled == nullptr) return false;
#define WB_D4(DD)                                                                                         \
    do {                                                                                                  \
        if (a.kv_half) return a.R <= 4 ? launch4_t<DD, 4, __half>(a, st) : launch4_t<DD, 8, __half>(a, st); \
        return a.R <= 4 ? launch4_t<DD, 4, float>(a, st) : launch4_t<DD, 8, float>(a, st);                 \
    } while (0)
    if (a.d == 384) WB_D4(384);
    if (a.d == 128) WB_D4(128);
#undef WB_D4
    return false;
}

}  // namespace wb
