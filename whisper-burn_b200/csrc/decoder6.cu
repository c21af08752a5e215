// Head-fused cluster decoder for L2-resident models (d = 128 / 384: tiny.en and the test models), greedy path and beam search.
//
// Same math and single-launch structure as decoder3.cu (TextDecoder::forward src/model/mod.rs:131-157, blocks :345-350,
// attention :428-533, MLP :376-382, search closure src/transcribe.rs:253-307; prefill + every greedy step in one kernel), but
// the per-layer chain is cut from 8 cluster-wide stages (decoder4.cu) to THREE exchanges, and every linear layer runs on the
// tensor cores (Hopper warpgroup MMA):
//
//   one thread-block cluster of CS = H CTAs owns one batch row; CTA h owns attention head h.
//   phase 1  x -> LN1 -> q_h | k_h | v_h (192 weight rows) -> causal self attention of head h -> the head's K-slice of the
//            out projection: y = Wo[:, 64h..64h+64) . o_h   (a partial d-vector)
//   phase 2  x -> LN2 -> cross query of head h -> cross attention of head h over the window's keys
//            (head-major K/V block streamed by bulk copies) -> y = Wco[:, 64h..) . o_h (un-normalised, with its (max, sum))
//   phase 3  x -> LN3 -> a 4d/CS slice of the MLP hidden layer (GELU) -> y = W2[:, slice] . hid_slice
//   after each phase every CTA sends its partial record (y, max, sum) to ALL CTAs of the cluster with ONE bulk shared-memory ->
//   distributed-shared-memory copy per destination (cp.async.bulk.shared::cluster.shared::cta) that signals the destination's
//   mbarrier with complete_tx; the receiver adds bias + the weighted partials (an attention record weighted by 1 / its
//   softmax sum; in a fixed order, identically in every CTA) and owns a full copy of the residual stream again.  No hardware
//   cluster barrier inside the step, no cross-thread release/acquire chains: data and its "ready" signal travel together.
//
//   Linear layers = swap-AB wgmma.mma_async (m64n8k16, fp16 operands, fp32 accumulate; M = weight rows): the weight slices of
//   this CTA are pre-packed per (layer, CTA) as 128-row x 64-column slabs in the canonical K-major 128B-swizzled shared-memory
//   image (dec6_pack_kernel), so a slab is ONE 16 KB bulk copy (TMA engine) into a ring slot and IS the A operand of two
//   m64 MMAs; the activation is the B operand: 8 rows of which row 0 = fp16(x) and row 1 = fp16((x - hi) * 2048) (the
//   hi/lo split of prims.cuh: exact products, fp32 accumulation), the rest zero.  The two consumer warpgroups take the 128-row output
//   tiles in turn (ping-pong: one group's epilogue overlaps the other's MMAs); the accumulator lives in the registers of the
//   group, columns 0 and 1 of a row in one thread, which combines hi + lo / 2048 after a shuffle that gives every lane one row
//   and applies bias / scale / GELU.  Weights do not depend on activations, so they never wait for the chain: a PRODUCER warp
//   streams weight slabs and the cross K/V block through the ring (full / empty mbarriers); the 8 consumer warps run the
//   dependent chain: LayerNorm, the MMAs (releasing a slot when the MMAs that read it have completed), attention (8 lanes per
//   key), epilogues, the exchange.
//
//   Only the vocabulary projection is chip-wide (as in decoder4.cu: bulk-copy ring of contiguous half-tiles of the tied
//   embedding, mma.sync swap-AB with fp16 hi/lo activation planes, fused mask / online softmax / arg-max), behind ONE grid
//   barrier; the per-row finish is done by the LAST CTA to deliver its records (ticket), which then releases a flag.
//
// Beam mode (dec6_kernel<..., BEAM = true>, a.beam = B in 2..7): the same kernel runs the prefill and the whole width-B search of
// R / B windows: row w * B + i is slot i of window w, self attention goes through the ancestry table, the vocabulary records
// keep DEC_KC candidates, and the finisher selects the next beams on the device (finish_beam, host/beam.hpp).
//
// Requirements: fp16-exact weights, d in {128, 384}, R <= 24 rows, t_max <= 128; greedy (k = 1) with identity ancestry, or
// the beam mode.  Everything else is handled by decoder5.cu / decoder3.cu.
#include <cooperative_groups.h>

#include <cstdlib>

#include "dec_common.cuh"
#include "wgmma.cuh"

namespace cg = cooperative_groups;

namespace wb {

namespace {

constexpr int NCW = 8;                    // consumer warps (threads 0..255)
constexpr int NPROD = 1;                  // producer warps (each walks the whole schedule and issues every NPROD-th chunk)
constexpr int W_PROD = NCW;
constexpr int NTH6 = (NCW + NPROD) * 32;          // + producer warps
constexpr int SLOT = 16384;               // bytes per ring slot = one 128-row x 64-column fp16 slab
constexpr int NSLOT = 8;
constexpr int LG_NBUF = 2;                // logits stage: ring slots per warp (aliases the weight ring)
constexpr int BX_SLAB = 1024;             // B operand: 8 rows x 128 bytes (one swizzle atom) per 64-column slab

template <int D>
struct Geo {
    static constexpr int H = D / 64, CS = H, NS = 4 * D / CS, SEND = D + 4;
    static constexpr int pad128(int n) { return (n + 127) / 128 * 128; }
    // packed weight segments of one (layer, rank), bytes: [tiles of 128 rows (the last one 64 rows when N % 128 == 64)][K / 64 slabs][rows x 128 B]
    static constexpr int OFF_QKV = 0, OFF_O = OFF_QKV + 192 * D * 2, OFF_CQ = OFF_O + D * 64 * 2, OFF_CO = OFF_CQ + 64 * D * 2,
                         OFF_W1 = OFF_CO + D * 64 * 2, OFF_W2 = OFF_W1 + NS * D * 2, PACK = OFF_W2 + D * NS * 2;
    static_assert(D % 128 == 0 && NS % 128 == 0, "only the 192- and 64-row segments end in a 64-row tile");
    // parameter block of one (layer, rank), floats
    static constexpr int P_LN1G = 0, P_LN1B = D, P_LN2G = 2 * D, P_LN2B = 3 * D, P_LN3G = 4 * D, P_LN3B = 5 * D, P_BO = 6 * D,
                         P_BCO = 7 * D, P_B2 = 8 * D, P_BQKV = 9 * D, P_BCQ = 9 * D + 192, P_B1 = 9 * D + 256, P_EPS = 9 * D + 256 + NS, PARAMS = 9 * D + 256 + NS + 4;
    static constexpr int KMAX = D > NS ? D : NS;   // widest B operand
    static_assert(PARAMS % 4 == 0 && SEND % 4 == 0 && NS % 64 == 0 && D % 64 == 0, "layout");
};

// ---- small PTX helpers -------------------------------------------------------------------------------------
__device__ long long g_watchdog = 20000000000LL;   // SM clocks a wait may last before the kernel traps (fail loudly instead of hanging the GPU); host-settable
// local shared memory -> the same offset in CTA `rank` of the cluster, completion on that CTA's mbarrier
__device__ __forceinline__ void bulk_s2peer(void* dst_local, const void* src, uint32_t bytes, uint64_t* bar_local, uint32_t rank) {
    const uint32_t rd = mapa_u32(smem_u32(dst_local), rank);
    const uint32_t rb = mapa_u32(smem_u32(bar_local), rank);
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(rd), "r"(smem_u32(src)), "r"(bytes), "r"(rb) : "memory");
}
__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void bar_all() { asm volatile("bar.sync 2, %0;" ::"n"(NTH6) : "memory"); }
__device__ __forceinline__ float group8_sum(float v) {   // sum over the 8 lanes that share lane >> 3 (all lanes converged)
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    return v;
}
// byte offset of element (row, k) inside a K-major 128B-swizzled operand whose 64-column slabs are `slab_bytes` apart
__device__ __host__ __forceinline__ uint32_t sw128_off(int row, int k, int slab_bytes) {
    return (uint32_t)((k >> 6) * slab_bytes + row * 128 + ((((k & 63) >> 3) ^ (row & 7)) << 4) + (k & 7) * 2);
}

// which of the 64 head dims is element i (0..7) of lane l8: two 16-byte chunks (fp32: l8 and l8 + 8) / one (fp16: l8)
template <typename KVT>
__device__ __forceinline__ int hdim(int l8, int i) {
    if constexpr (sizeof(KVT) == 4) return (i < 4 ? 4 * l8 : 32 + 4 * l8) + (i & 3);
    else return 8 * l8 + i;
}
// the lane's 8 elements of a 64-dim K or V row; par = 1 on odd positions of the head-major cross layout (XOR-4 chunk swizzle)
template <typename KVT>
__device__ __forceinline__ void load_row8(const KVT* row, int l8, int par, float (&f)[8], bool smem) {
    if constexpr (sizeof(KVT) == 4) {
        const float4* p = reinterpret_cast<const float4*>(row);
        const float4 a = smem ? p[l8 ^ (4 * par)] : __ldcg(p + (l8 ^ (4 * par)));
        const float4 b = smem ? p[(l8 + 8) ^ (4 * par)] : __ldcg(p + ((l8 + 8) ^ (4 * par)));
        f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    } else {
        const uint4* p = reinterpret_cast<const uint4*>(row);
        const uint4 u = smem ? p[l8 ^ (4 * par)] : __ldcg(p + (l8 ^ (4 * par)));
        cvt8(u, f);
    }
}

struct Softmax8 {   // online softmax state of one (warp, rg) key slot; o = the lane's 8 dims
    float m, l, o[8];
    __device__ __forceinline__ void init() {
        m = -INFINITY; l = 0.0f;
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = 0.0f;
    }
    __device__ __forceinline__ void add(float s, const float (&v)[8]) {
        const float mn = fmaxf(m, s);
        const float corr = expf(m - mn), e = expf(s - mn);
        l = l * corr + e;
        m = mn;
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = fmaf(e, v[i], o[i] * corr);
    }
    __device__ __forceinline__ void merge_xor(int off) {   // all lanes converged
        const float m2 = __shfl_xor_sync(0xffffffffu, m, off), l2 = __shfl_xor_sync(0xffffffffu, l, off);
        const float mn = fmaxf(m, m2);
        const float c1 = m > -INFINITY ? expf(m - mn) : 0.0f, c2 = m2 > -INFINITY ? expf(m2 - mn) : 0.0f;
        l = l * c1 + l2 * c2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float o2 = __shfl_xor_sync(0xffffffffu, o[i], off);
            o[i] = o[i] * c1 + o2 * c2;
        }
        m = mn;
    }
};

// ---- weight / parameter packing (once per session) ---------------------------------------------------------------------
// Segment [N][K] (fp16, source rows n0 + (r / piece) * piece_stride + r % piece, columns k0 .. k0 + K of a [.][ldk] matrix) as
// tiles of 128 rows (a last tile of 64 rows when N % 128 == 64), each tile as K / 64 slabs of rows x 128 B in the K-major
// 128B-swizzled shared-memory image: 16-byte unit (row r, chunk c) of a slab at r * 128 + ((c ^ (r & 7)) << 4).  A slab is what
// one bulk copy moves and what one group of four K steps of wgmma (two m64 row halves, or one for a 64-row tile) reads.
struct PackSeg {
    const __half* src;
    int ldk, n0, k0, N, K;
    int piece, piece_stride;
    int64_t dst_off;   // bytes
};
__global__ void dec6_pack_kernel(const PackSeg* segs, int n_segs, uint8_t* dst) {
    for (int s = blockIdx.y; s < n_segs; s += gridDim.y) {
        const PackSeg g = segs[s];
        const int nslab = g.K / 64;
        const int64_t n16 = (int64_t)g.N * g.K / 8;   // 16-byte units; N is a multiple of 64
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (int64_t)gridDim.x * blockDim.x) {
            // source order: unit i = (row, column chunk)
            const int row = (int)(i / (g.K / 8)), cc = (int)(i % (g.K / 8));
            const int t = row >> 7, r = row & 127, sl = cc >> 3, c = cc & 7;
            const int trows = min(128, g.N - t * 128);                       // rows of this tile: 128 or 64
            const int64_t tile_base = (int64_t)t * 128 * g.K * 2;            // full tiles precede
            const int srow = g.n0 + (row / g.piece) * g.piece_stride + row % g.piece;
            const uint4 v = *reinterpret_cast<const uint4*>(g.src + (int64_t)srow * g.ldk + g.k0 + cc * 8);
            *reinterpret_cast<uint4*>(dst + g.dst_off + tile_base + (int64_t)sl * trows * 128 + r * 128 + ((c ^ (r & 7)) << 4)) = v;
        }
        (void)nslab;
    }
}
struct ParamSeg {
    const float* src;
    int n;
    int64_t dst_off;   // floats
};
__global__ void dec6_param_kernel(const ParamSeg* segs, int n_segs, float* dst) {
    for (int s = blockIdx.x; s < n_segs; s += gridDim.x) {
        const ParamSeg g = segs[s];
        for (int i = threadIdx.x; i < g.n; i += blockDim.x) dst[g.dst_off + i] = g.src[i];
    }
}

// ---- building blocks of a phase.  Code size is latency here (decoder5.cu, lesson 2): the layer body runs once per layer and
// position, i.e. mostly from a cold instruction cache, so every block exists ONCE (noinline, runtime shapes) and the phases are
// short call sequences.

// the B operand of the next linear layer: value v of column k -> fp16 hi in row 0, fp16 (residual * 2048) in row 1
__device__ __forceinline__ void bx_store(uint8_t* bx, int k, float v) {
    __half h, l;
    hl_split(v, h, l);
    *reinterpret_cast<__half*>(bx + sw128_off(0, k, BX_SLAB)) = h;
    *reinterpret_cast<__half*>(bx + sw128_off(1, k, BX_SLAB)) = l;
}

struct Pipe {        // shared-memory handles of the ring / tensor-core pipeline
    uint8_t* ring;   // [NSLOT][SLOT]
    uint64_t *full, *empty;      // per slot
    uint8_t* bx;     // [KMAX / 64][BX_SLAB] B operand
};
struct Counters {    // progress counters every role keeps in registers (identical sequences by construction)
    uint32_t n;      // ring chunks consumed / issued
    uint32_t tile;   // output tiles
};

enum { EM_PLAIN = 0, EM_QKV = 1, EM_CQ = 2, EM_HID = 3 };
template <typename KVT>
struct GemvOut {
    int mode;
    const float* bias;
    float scale;
    float* out;        // EM_PLAIN: y[n]; EM_QKV: qkv_s[n]; EM_CQ: q2_s[n]; EM_HID: hid_s[n]
    KVT *kdst, *vdst;  // EM_QKV: this position's 64-element head slice of the self K / V cache
};

// One linear layer y[n] = sum_k W[n][k] x[k] (n < N, N padded to tiles of 128 rows) by the consumer warps, the B operand
// written: warpgroup (tile & 1) takes the tile -- its K slabs from the ring, one or two m64n8k16 MMAs per K step, the slot
// released once the MMAs that read it have completed -- and applies the epilogue.  Ends with a barrier of the consumer warps.
template <typename KVT>
__device__ __noinline__ Counters gemv_epi6(const Pipe P, Counters c, int N, int n_slabs, const GemvOut<KVT> o) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    fence_proxy_async();   // generic writes of the B operand -> tensor-core (async proxy) reads
    bar_consumers();
    const int n_tiles = (N + 127) >> 7;
    const uint32_t ring0 = smem_u32(P.ring), bx0 = smem_u32(P.bx);
#pragma unroll 1
    for (int t = 0; t < n_tiles; ++t) {
        const uint32_t T = c.tile + (uint32_t)t, g = T & 1;
        if ((uint32_t)(warp >> 2) != g) continue;
        const bool half_tile = N - t * 128 < 128;   // the last tile of a 192- / 64-row segment has 64 rows
        float acc0[4] = {0.0f, 0.0f, 0.0f, 0.0f}, acc1[4] = {0.0f, 0.0f, 0.0f, 0.0f};   // rows 0..63 / 64..127 of the tile
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        uint32_t n = c.n + (uint32_t)(t * n_slabs);
#pragma unroll 1
        for (int s = 0; s < n_slabs; ++s, ++n) {
            const uint32_t slot = n % NSLOT;
            mbar_wait_bounded(P.full + slot, (n / NSLOT) & 1, g_watchdog);
            // rows 64..127 of a slab start 8 swizzle atoms (8192 bytes) in; K step = 32 bytes -> +2 in the (>> 4) address field.
            // A 64-row slab leaves the second half of its slot stale: that MMA runs anyway (no branch between the MMAs, which
            // would serialise them) and its rows are discarded.
            const uint64_t da = wgmma_desc(ring0 + slot * SLOT), db = wgmma_desc(bx0 + s * BX_SLAB);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                wgmma_m64n8k16(acc0, da + 2 * k, db + 2 * k);
                wgmma_m64n8k16(acc1, da + (8192 >> 4) + 2 * k, db + 2 * k);
            }
            wgmma_commit();
            wgmma_wait<1>();   // the previous slab's MMAs have completed: its slot may be overwritten
            if (s > 0 && (tid & 127) == 0) mbar_arrive(P.empty + (n - 1) % NSLOT);
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        if ((tid & 127) == 0) mbar_arrive(P.empty + (n - 1) % NSLOT);
        // m64n8 fragment: lane 4i of warp w holds columns 0 (hi), 1 (lo) of rows 16 w + i (registers 0, 1) and 16 w + i + 8
        // (registers 2, 3).  Lane L takes row 64 (L >> 4) + 16 w + 8 ((L >> 3) & 1) + (L & 7) of the tile from lane 4 (L & 7).
        const int src = (lane & 7) * 4, sel = lane >> 3;
        float hv[4], lv[4];
        hv[0] = __shfl_sync(0xffffffffu, acc0[0], src); lv[0] = __shfl_sync(0xffffffffu, acc0[1], src);
        hv[1] = __shfl_sync(0xffffffffu, acc0[2], src); lv[1] = __shfl_sync(0xffffffffu, acc0[3], src);
        hv[2] = __shfl_sync(0xffffffffu, acc1[0], src); lv[2] = __shfl_sync(0xffffffffu, acc1[1], src);
        hv[3] = __shfl_sync(0xffffffffu, acc1[2], src); lv[3] = __shfl_sync(0xffffffffu, acc1[3], src);
        const float hi = sel == 0 ? hv[0] : sel == 1 ? hv[1] : sel == 2 ? hv[2] : hv[3];
        const float lo = sel == 0 ? lv[0] : sel == 1 ? lv[1] : sel == 2 ? lv[2] : lv[3];
        const int row = t * 128 + 64 * (lane >> 4) + 16 * (warp & 3) + 8 * ((lane >> 3) & 1) + (lane & 7);
        if (row < N && (!half_tile || lane < 16)) {
            const float s = hl_join(hi, lo);
            if (o.mode == EM_PLAIN) {
                o.out[row] = s;
            } else if (o.mode == EM_QKV) {       // mod.rs:429-431; q and k carry (d/H)^-0.25 each (:500-503)
                float v = __fadd_rn(s, o.bias[row]);
                if (row < 128) v = __fmul_rn(v, o.scale);
                if (row >= 64) {
                    const KVT r = (KVT)v;          // fp16 cache: round-to-nearest where the value enters the cache
                    (row < 128 ? o.kdst : o.vdst)[row & 63] = r;
                    v = (float)r;
                }
                o.out[row] = v;
            } else if (o.mode == EM_CQ) {        // cross query (mod.rs:483)
                o.out[row] = __fmul_rn(__fadd_rn(s, o.bias[row]), o.scale);
            } else {                             // gelu(LN(x) W1 + b1) (mod.rs:377-378)
                o.out[row] = gelu_erf(__fadd_rn(s, o.bias[row]));
            }
        }
    }
    c.tile += (uint32_t)n_tiles;
    c.n += (uint32_t)(n_tiles * n_slabs);
    bar_consumers();
    return c;
}

// LayerNorm (burn 0.9 form, prims.cuh) of the row x_s[D] by the 8 consumer warps: every warp computes the
// statistics for itself (no block reduction), thread t normalises elements t, t + 256 and writes them as the B operand.
template <int D>
__device__ __noinline__ void ln6(const float* x_s, const float* g, const float* b, float eps, int eps_outside, uint8_t* bx) {
    const int tid = threadIdx.x, lane = tid & 31;
    float v[D / 32];
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i < D / 32; ++i) { v[i] = x_s[lane + 32 * i]; sum += v[i]; }
    sum = warp_sum(sum);
    const float mean = __fdiv_rn(sum, (float)D);
    float q = 0.0f;
#pragma unroll
    for (int i = 0; i < D / 32; ++i) q = ln_sq_add(q, __fsub_rn(v[i], mean));
    q = warp_sum(q);
    const float var = __fdiv_rn(q, (float)D);
    const float den = LN_DEN(var, eps, eps_outside);
#pragma unroll 1
    for (int c = tid; c < D; c += 256) bx_store(bx, c, ln_norm(__fsub_rn(x_s[c], mean), den, g, b, c));
}

// merges the 8 per-warp attention records (wm, wl, wo) into the head's un-normalised output, written as the B operand of the
// out projection, and its (max, sum) record
__device__ __noinline__ void attn_merge6(const float* wm, const float* wl, const float* wo, uint8_t* bx, float* rec) {
    const int tid = threadIdx.x;
    bar_consumers();
    if (tid < 64) {
        float M = -INFINITY;
#pragma unroll
        for (int w2 = 0; w2 < NCW; ++w2) M = fmaxf(M, wm[w2]);
        float Ls = 0.0f, o = 0.0f;
#pragma unroll
        for (int w2 = 0; w2 < NCW; ++w2) {
            const float sc = wm[w2] > -INFINITY ? expf(wm[w2] - M) : 0.0f;
            Ls += sc * wl[w2];
            o += sc * wo[w2 * 64 + tid];
        }
        bx_store(bx, tid, o);
        if (tid == 0) { rec[0] = M; rec[1] = Ls; }
    }
}

enum { MODE_SUM = 0, MODE_ATTN = 1 };

// x += bias + sum over sources of weight * partial (fixed order, identical in every CTA of the cluster).  pr = the phase's
// records [CS][D + 4] (y, max, sum, unused); MODE_ATTN: y is head h's un-normalised attention output projected by its slice
// of the out projection, weight 1 / sum (mod.rs:516-527); MODE_SUM: plain sum.  Ends with a barrier.
template <int D>
__device__ __noinline__ void combine6(const float* pr, uint64_t* bar, uint32_t parity, int mode, const float* bias, float* x_s, float* wsrc_s) {
    constexpr int CS = Geo<D>::CS, SEND = Geo<D>::SEND;
    const int tid = threadIdx.x;
    if (tid == 0) mbar_expect_tx(bar, CS * SEND * 4);
    mbar_wait_bounded(bar, parity, g_watchdog);
    if (tid < CS) {
        const float* me = pr + tid * SEND + D;
        wsrc_s[tid] = mode == MODE_SUM ? 1.0f : me[0] > -INFINITY ? __fdiv_rn(1.0f, me[1]) : 0.0f;
    }
    bar_consumers();
#pragma unroll 1
    for (int c = tid; c < D; c += 256) {
        float acc = bias[c];
#pragma unroll 4
        for (int s = 0; s < CS; ++s) acc = fmaf(wsrc_s[s], pr[s * SEND + c], acc);
        x_s[c] = __fadd_rn(x_s[c], acc);
    }
    bar_consumers();
}

// causal self attention of one head over positions 0..p (mod.rs:428-436 with the mask of :535-544 = "keys <= p"): 32 (warp, rg)
// key slots, 8 lanes per key; keys < p come from the cache (L2), key p from shared memory.  Leaves per-warp records in wm/wl/wo.
// ANC (beam search): key j < p lives in cache row anc[j], i.e. at kbase + anc[j] * row_ld + j * ld (decoder3.cu addressing).
template <typename KVT, bool ANC>
__device__ __forceinline__ void self_attn6_body(const float* qkv_s, const KVT* kbase, const KVT* vbase, int ld, int p, const int* anc,
                                                int64_t row_ld, float* wm, float* wl, float* wo) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, rg = lane >> 3, l8 = lane & 7;
    float q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] = qkv_s[hdim<KVT>(l8, i)];
    Softmax8 A;
    A.init();
    float kf[4][8], vf[4][8];
    const int j0 = warp * 4 + rg;
#pragma unroll
    for (int u = 0; u < 4; ++u) {                          // all loads first (t_max <= 128 -> at most 4 keys per slot)
        const int j = j0 + 32 * u;
        if (j < p) {
            const int64_t off = ANC ? (int64_t)__ldcg(anc + j) * row_ld + (int64_t)j * ld : (int64_t)j * ld;
            load_row8<KVT>(kbase + off, l8, 0, kf[u], false);
            load_row8<KVT>(vbase + off, l8, 0, vf[u], false);
        } else if (j == p) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { kf[u][i] = qkv_s[64 + hdim<KVT>(l8, i)]; vf[u][i] = qkv_s[128 + hdim<KVT>(l8, i)]; }
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) { kf[u][i] = 0.0f; vf[u][i] = 0.0f; }
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < 8; ++i) s = fmaf(q[i], kf[u][i], s);
        s = group8_sum(s);
        if (j0 + 32 * u <= p) A.add(s, vf[u]);
    }
    A.merge_xor(8);
    A.merge_xor(16);
    if (rg == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) wo[warp * 64 + hdim<KVT>(l8, i)] = A.o[i];
        if (l8 == 0) { wm[warp] = A.m; wl[warp] = A.l; }
    }
}
template <typename KVT>
__device__ __noinline__ void self_attn6(const float* qkv_s, const KVT* kbase, const KVT* vbase, int ld, int p, float* wm, float* wl, float* wo) {
    self_attn6_body<KVT, false>(qkv_s, kbase, vbase, ld, p, nullptr, 0, wm, wl, wo);
}
template <typename KVT>
__device__ __noinline__ void self_attn6_anc(const float* qkv_s, const KVT* kbase, const KVT* vbase, int ld, int p, const int* anc, int64_t row_ld,
                                            float* wm, float* wl, float* wo) {
    self_attn6_body<KVT, true>(qkv_s, kbase, vbase, ld, p, anc, row_ld, wm, wl, wo);
}

// cross attention of one head over the T keys of the window (mod.rs:482-490), the head-major K/V block arriving through
// the ring in chunks of KPC keys; 8 lanes per key.  A slot is released by the LAST of the 8 warps to finish with it (the slots'
// empty barriers take one arrival, as the MMA warpgroup gives them for weight slabs).  (Waiting for several chunks at once to batch
// the per-key latency chains was measured SLOWER, 6 -> 12 us per layer: the chunks arrive one per ~0.3 us and the batch waits for
// the last one.)  Returns the ring counter.
template <typename KVT>
__device__ __noinline__ uint32_t cross_attn6(const Pipe P, uint32_t n, int* slot_cnt, const float* q2_s, int T, float* wm, float* wl, float* wo) {
    constexpr int ROWB = 128 * (int)sizeof(KVT), KPC = SLOT / ROWB;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, rg = lane >> 3, l8 = lane & 7;
    float q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] = q2_s[hdim<KVT>(l8, i)];
    Softmax8 A;
    A.init();
#pragma unroll 1
    for (int k0 = 0; k0 < T; k0 += KPC) {
        const int nk = min(KPC, T - k0);
        const uint32_t slot = n % NSLOT;
        mbar_wait_bounded(P.full + slot, (n / NSLOT) & 1, g_watchdog);
        const uint8_t* blk = P.ring + slot * SLOT;
#pragma unroll 2
        for (int kk = warp * 4 + rg; kk < nk; kk += 32) {
            const int par = (k0 + kk) & 1;
            const KVT* rowp = reinterpret_cast<const KVT*>(blk + (size_t)kk * ROWB);
            float kf[8], vf[8];
            load_row8<KVT>(rowp, l8, par, kf, true);
            load_row8<KVT>(rowp + 64, l8, par, vf, true);
            float s = 0.0f;
#pragma unroll
            for (int i = 0; i < 8; ++i) s = fmaf(q[i], kf[i], s);
            const unsigned int gm = 0xffu << (lane & 24);
            s += __shfl_xor_sync(gm, s, 1);
            s += __shfl_xor_sync(gm, s, 2);
            s += __shfl_xor_sync(gm, s, 4);
            A.add(s, vf);
        }
        __syncwarp();
        if (lane == 0 && atomicAdd(slot_cnt + slot, 1) == NCW - 1) {
            slot_cnt[slot] = 0;
            mbar_arrive(P.empty + slot);
        }
        ++n;
    }
    __syncwarp();
    A.merge_xor(8);
    A.merge_xor(16);
    if (rg == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) wo[warp * 64 + hdim<KVT>(l8, i)] = A.o[i];
        if (l8 == 0) { wm[warp] = A.m; wl[warp] = A.l; }
    }
    return n;
}

// ---- beam mode: the finisher's work at a search position p (depth = p - logits_from), by the last CTA to deliver its records.
constexpr int BM_LIVE = 24;                                          // rows of a beam launch
constexpr int BM_NX = 3 * BM_LIVE + 3 * NCW * beamfx::MAX_NODES;     // finish_beam's shared scratch (ints)
//   (a) each live slot's B best candidates by the rounded log-prob (v - max) - lse, ranked by cand_better, from the CTAs'
//       records -> topk_id / topk_lp [row][B];
//   (b) one warp per unfinished window: beamfx::beam_step on the carried nodes (lane 0), the new nodes' sequences and the
//       log-probs their tokens were scored with (bm_seq / bm_seq_lp, the warp); the next position's live slots w * B + i in
//       carried order, each with its parent's cache row and its token.  A window whose search has not started (p + 1 is
//       inside its prompt: dec_common.cuh id_limit) keeps slot 0 live in its own row with its next prompt token;
//   (c) a window is done when its best carried node is finished or at max_depth steps after its own prompt; the search
//       ends when every window is done: then the best
//       sequence of every window goes to bm_out / bm_out_lp and bar[3] is set; otherwise the next position's slots, tokens and ancestry
//       table (anc_new[r][j] = anc_old[parent[r]][j] for j <= p, anc_new[r][p + 1] = r) are written.
// Called by the 256 consumer threads; ends with a barrier of the consumers.
__device__ __noinline__ void finish_beam(const DecArgs& a, int p, int depth, const int* anc_cur, uint8_t* scratch, const int* live, int* nx,
                                         int* ctl) {
    namespace fx = beamfx;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int R = a.R, B = a.beam, t_max = a.t_max, NW = a.n_win;
    int* nx_par = nx;
    int* nx_tok = nx_par + BM_LIVE;
    int* nx_live = nx_tok + BM_LIVE;
    int* pk_src = nx_live + BM_LIVE + warp * 3 * fx::MAX_NODES;   // this warp's picks: source, token, length
    int* pk_tok = pk_src + fx::MAX_NODES;
    int* pk_len = pk_tok + fx::MAX_NODES;
    // ---- (a)
    constexpr int RINGW = NSLOT * SLOT / NCW;
    static_assert(160 * DEC_KC * 8 <= RINGW, "finisher candidate scratch");
    for (int r = warp; r < R; r += NCW) {
        if (!live[r]) continue;
        const int NP = gridDim.x;   // <= 160 co-resident CTAs
        float rm[5], rs[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const int c = min(lane + 32 * k, NP - 1);
            rm[k] = __ldcg(a.lg_m + (int64_t)c * R + r);
            rs[k] = __ldcg(a.lg_s + (int64_t)c * R + r);
        }
        float mx;
        const float lse = row_lse<5>(rm, rs, NP, mx);
        // the row's NP * DEC_KC candidates as (log-prob, id) in this warp's share of the (idle) ring
        float* cv = reinterpret_cast<float*>(scratch + (size_t)warp * RINGW);
        int* ci = reinterpret_cast<int*>(cv + 160 * DEC_KC);
        const int NC = NP * DEC_KC;
        for (int q = lane; q < NC; q += 32) {
            const int64_t o = ((int64_t)(q / DEC_KC) * R + r) * DEC_KC + q % DEC_KC;
            ci[q] = __ldcg(a.lg_i + o);
            cv[q] = __fsub_rn(__fsub_rn(__ldcg(a.lg_v + o), mx), lse);
        }
        __syncwarp();
        float prev_v = INFINITY;
        int prev_i = -1;
        for (int kk = 0; kk < B; ++kk) {   // the best candidate ranked after the previous one
            float bv = -INFINITY;
            int bi = INT_MAX;
            for (int q = lane; q < NC; q += 32) {
                const int idx = ci[q];
                if (idx == INT_MAX) continue;
                const float v = cv[q];
                if (cand_better(prev_v, prev_i, v, idx) && cand_better(v, idx, bv, bi)) { bv = v; bi = idx; }
            }
            warp_best(bv, bi);
            if (lane == 0) {
                a.topk_id[(int64_t)r * B + kk] = bi == INT_MAX ? -1 : bi;
                a.topk_lp[(int64_t)r * B + kk] = bv;
            }
            prev_v = bv;
            prev_i = bi;
        }
        __syncwarp();
    }
    bar_consumers();
    // ---- (b)
    for (int w = warp; w < NW; w += NCW) {
        const int buf = __ldcg(a.bm_win + 2 * w);
        if (__ldcg(a.bm_win + 2 * w + 1)) {   // done: its slots stay idle
            if (lane < B) nx_live[w * B + lane] = 0;
            continue;
        }
        if (p + 2 + a.max_depth <= id_limit(a, w * B)) {   // the window's search starts at its last prompt position
            if (lane < B) nx_live[w * B + lane] = lane == 0 ? 1 : 0;
            if (lane == 0) {
                nx_par[w * B] = w * B;
                nx_tok[w * B] = __ldcg(a.tokens + (int64_t)w * B * t_max + p + 1);
            }
            continue;
        }
        const int nb = buf ^ 1;
        int n_out = 0;
        if (lane == 0) {
            fx::Head in[fx::MAX_NODES];
            int step_row[fx::MAX_NODES], cid[fx::MAX_NODES * fx::MAX_BEAM];
            double clp[fx::MAX_NODES * fx::MAX_BEAM];
            const int n_in = __ldcg(a.bm_cnt + buf * NW + w);
            const fx::Head* hs = a.bm_head + ((size_t)buf * NW + w) * fx::MAX_NODES;
            int li = 0;
            for (int b = 0; b < n_in; ++b) {
                in[b].log_prob = __ldcg(&hs[b].log_prob);
                in[b].finished = __ldcg(&hs[b].finished);
                in[b].row = __ldcg(&hs[b].row);
                in[b].len = __ldcg(&hs[b].len);
                in[b].pad = 0;
                if (in[b].finished) continue;
                const int r = w * B + li++;   // the li-th live node sat in slot r at this position
                step_row[b] = r;
                for (int i = 0; i < B; ++i) {
                    cid[b * B + i] = __ldcg(a.topk_id + (int64_t)r * B + i);
                    clp[b * B + i] = (double)__ldcg(a.topk_lp + (int64_t)r * B + i);
                }
            }
            fx::Pick out[fx::MAX_NODES];
            n_out = fx::beam_step(in, n_in, step_row, cid, clp, B, a.eot, out);
            fx::Head* ho = a.bm_head + ((size_t)nb * NW + w) * fx::MAX_NODES;
            float* lp_dst = a.bm_seq_lp + ((size_t)nb * NW + w) * fx::MAX_NODES * t_max;
            int nl = 0;
            for (int i = 0; i < n_out; ++i) {
                ho[i] = out[i].head;
                in[i] = out[i].head;   // (for the stop test below)
                pk_src[i] = out[i].src;
                pk_tok[i] = out[i].token;
                pk_len[i] = out[i].head.len;
                if (out[i].token >= 0) lp_dst[i * t_max + out[i].head.len - 1] = (float)out[i].lp;   // exact: a widened f32
                if (!out[i].head.finished) {
                    const int s = w * B + nl++;
                    nx_par[s] = out[i].head.row;
                    nx_tok[s] = out[i].token;
                    nx_live[s] = 1;
                }
            }
            for (; nl < B; ++nl) nx_live[w * B + nl] = 0;
            a.bm_cnt[nb * NW + w] = n_out;
            a.bm_win[2 * w] = nb;
            a.bm_win[2 * w + 1] = (fx::search_done(in, n_out) || p + 2 >= id_limit(a, w * B)) ? 1 : 0;
        }
        n_out = __shfl_sync(0xffffffffu, n_out, 0);
        __syncwarp();
        const int* src = a.bm_seq + ((size_t)buf * NW + w) * fx::MAX_NODES * t_max;
        int* dst = a.bm_seq + ((size_t)nb * NW + w) * fx::MAX_NODES * t_max;
        const float* src_lp = a.bm_seq_lp + ((size_t)buf * NW + w) * fx::MAX_NODES * t_max;
        float* dst_lp = a.bm_seq_lp + ((size_t)nb * NW + w) * fx::MAX_NODES * t_max;
        for (int i = 0; i < n_out; ++i) {   // node i = its source's sequence (+ the token it appends, its log-prob written above)
            const int s = pk_src[i], tk = pk_tok[i], ln = pk_len[i] - (tk >= 0 ? 1 : 0);
            for (int j = lane; j < ln; j += 32) {   // both loads before either store: one L2 round trip per position
                const int t = __ldcg(src + s * t_max + j);
                const float l = __ldcg(src_lp + s * t_max + j);
                dst[i * t_max + j] = t;
                dst_lp[i * t_max + j] = l;
            }
            if (lane == 0 && tk >= 0) dst[i * t_max + ln] = tk;
        }
        __syncwarp();
    }
    bar_consumers();
    // ---- (c)
    if (tid == 0) {
        int open = 0;
        for (int w = 0; w < NW; ++w) open += __ldcg(a.bm_win + 2 * w + 1) ? 0 : 1;
        ctl[2] = open == 0 ? 1 : 0;
        ctl[3] = open;
    }
    bar_consumers();
    if (ctl[2] == 0) {
        int* an = (depth & 1) ? const_cast<int*>(a.anc) : a.anc_alt;   // beam mode owns both tables (session anc0 / anc1)
        if (tid < R) {
            a.slot_live[tid] = nx_live[tid];
            if (nx_live[tid]) a.tokens[(int64_t)tid * t_max + p + 1] = nx_tok[tid];
        }
        const int P = p + 2;
        for (int q = tid; q < R * P; q += 256) {
            const int r = q / P, j = q % P;
            if (nx_live[r]) an[(int64_t)r * t_max + j] = j <= p ? __ldcg(anc_cur + (int64_t)nx_par[r] * t_max + j) : r;
        }
    } else {
        for (int w = warp; w < NW; w += NCW) {
            const int buf = __ldcg(a.bm_win + 2 * w);
            const fx::Head* hs = a.bm_head + ((size_t)buf * NW + w) * fx::MAX_NODES;
            int best = 0, len = 0;
            if (lane == 0) {
                const int n = __ldcg(a.bm_cnt + buf * NW + w);
                fx::Head hn[fx::MAX_NODES];
                for (int b = 0; b < n; ++b) { hn[b].log_prob = __ldcg(&hs[b].log_prob); hn[b].finished = __ldcg(&hs[b].finished); }
                best = max(fx::max_by_last(hn, n), 0);
                len = n > 0 ? __ldcg(&hs[best].len) : 0;
                a.bm_out_len[w] = len;
            }
            best = __shfl_sync(0xffffffffu, best, 0);
            len = __shfl_sync(0xffffffffu, len, 0);
            const size_t o = (((size_t)buf * NW + w) * fx::MAX_NODES + best) * t_max;
            for (int j = lane; j < len; j += 32) {
                const int t = __ldcg(a.bm_seq + o + j);
                const float l = __ldcg(a.bm_seq_lp + o + j);
                a.bm_out[(int64_t)w * t_max + j] = t;
                a.bm_out_lp[(int64_t)w * t_max + j] = l;
            }
        }
        if (tid == 0) {
            decode_done(a, p + 1, ctl[3], depth + 1);
            a.bar[3] = 1;
        }
    }
    bar_consumers();
}

// =====================================================================================================================
// BEAM: the beam search (a.beam = B > 1).  A slot without a live beam idles at a position (no layer work, empty records);
// the finisher (last CTA to deliver its records) ranks each live slot's candidates, runs one beamfx::beam_step per
// unfinished window, places the new live beams in slots w * B + i, and builds the next position's ancestry table.
template <int D, int NT8, typename KVT, bool BEAM = false>
__global__ void __launch_bounds__(NTH6, 1)
dec6_kernel(const DecArgs a) {
    using G = Geo<D>;
    constexpr int CS = G::CS, NS = G::NS, SEND = G::SEND, PARAMS = G::PARAMS;
    constexpr int KPC = SLOT / (128 * (int)sizeof(KVT));   // cross keys per ring chunk
    constexpr int ROWB = 128 * (int)sizeof(KVT);
    extern __shared__ __align__(1024) unsigned char smraw_[];
    uint8_t* smraw = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smraw_) + 1023) & ~(uintptr_t)1023);
    cg::cluster_group cl = cg::this_cluster();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = (int)cl.block_rank(), h = rank;
    const int cluster_id = blockIdx.x / CS, n_clusters = gridDim.x / CS;
    const int L = a.L, V = a.V, R = a.R, t_max = a.t_max;

    // ---- shared memory carve-up (ring and B operand 1024-byte aligned: swizzle atoms)
    uint8_t* ring_mem = smraw;                                              // [NSLOT][SLOT]
    uint8_t* bx = ring_mem + NSLOT * SLOT;                                  // [KMAX / 64][8 rows][128 B]  B operand (rows 0, 1 live)
    float* params = reinterpret_cast<float*>(bx + (G::KMAX / 64) * BX_SLAB);   // [2][PARAMS]
    float* part = params + 2 * PARAMS;                                      // [2][CS][SEND] partial records of the cluster
    float* y_s = part + 2 * CS * SEND;                                      // [2][SEND]     this CTA's outgoing record
    float* x_s = y_s + 2 * SEND;                                            // [D]           residual stream (own copy)
    float* qkv_s = x_s + D;                                                 // [192]         q_h | k_h | v_h of the current position
    float* q2_s = qkv_s + 192;                                              // [64]
    float* hid_s = q2_s + 64;                                               // [NS]          MLP hidden slice
    float* wsrc_s = hid_s + NS;                                             // [16]          merge weights of the sources
    float* wm = wsrc_s + 16;                                                // [8]
    float* wl = wm + 8;                                                     // [8]
    float* wo = wl + 8;                                                     // [8][64]
    int* ctl = reinterpret_cast<int*>(wo + 512);                            // [4] stop flag, is_last
    int* slot_cnt = ctl + 4;                                                // [NSLOT] warps done with a K/V chunk
    uint64_t* bars = reinterpret_cast<uint64_t*>(slot_cnt + NSLOT);
    uint64_t* full = bars;                    // [NSLOT]
    uint64_t* empty = full + NSLOT;           // [NSLOT]
    uint64_t* pfull = empty + NSLOT;          // [2] parameter block landed
    uint64_t* pfree = pfull + 2;              // [2] consumers are done with the parameter block
    uint64_t* pbar = pfree + 2;               // [2] partial records of a phase landed
    uint64_t* lg_bar = pbar + 2;              // [NCW][LG_NBUF] logits stage
    // beam mode: live slots of a step, double-buffered by step parity (the producer may still read one step's set while the
    // consumers publish the next): [2][BM_LIVE] flags, [2][BM_LIVE] compact list of live rows, [2] their count; then the
    // finisher's scratch (finish_beam)
    int* live_s = reinterpret_cast<int*>(lg_bar + NCW * LG_NBUF);
    int* live_rows = live_s + 2 * BM_LIVE;
    int* n_live_s = live_rows + 2 * BM_LIVE;
    int* nx_s = n_live_s + 2;                 // [BM_NX]
    // logits-stage scratch aliases the (then dead) parameter / partial buffers
    uint4* pl_hi = reinterpret_cast<uint4*>(params);                        // [NT8][D/32][32] fp16 hi plane of the LayerNorm rows, fragment order
    uint4* pl_lo = pl_hi + NT8 * (D / 32) * 32;
    float* red = reinterpret_cast<float*>(pl_lo + NT8 * (D / 32) * 32);     // [NCW][8 * NT8][4]

    if (tid == 0) {
        for (int i = 0; i < NSLOT; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 1); slot_cnt[i] = 0; }
        for (int i = 0; i < 2; ++i) { mbar_init(pfull + i, 1); mbar_init(pfree + i, NCW); mbar_init(pbar + i, 1); }
        for (int i = 0; i < NCW * LG_NBUF; ++i) mbar_init(lg_bar + i, 1);
        ctl[0] = 0; ctl[1] = 0;
        mbar_fence_init();
    }
    for (int i = tid; i < (G::KMAX / 64) * BX_SLAB / 16; i += NTH6) reinterpret_cast<uint4*>(bx)[i] = make_uint4(0, 0, 0, 0);   // rows 2..7 stay zero
    // beam mode: step 0's live slots (set by the host: slot 0 of every window) into buffer 0
    auto snapshot_live = [&](int buf) {   // tid < R load, one barrier, tid 0 compacts; the caller's next barrier publishes
        if (tid < R) live_s[buf * BM_LIVE + tid] = __ldcg(a.slot_live + tid);
        bar_consumers();
        if (tid == 0) {
            int n = 0;
            for (int r = 0; r < R; ++r)
                if (live_s[buf * BM_LIVE + r]) live_rows[buf * BM_LIVE + n++] = r;
            n_live_s[buf] = n;
        }
    };
    if constexpr (BEAM) {
        if (tid < 256) snapshot_live(0);
    }
    cl.sync();   // every CTA's mbarriers exist before any peer signals them
    Pipe P;
    P.ring = ring_mem; P.full = full; P.empty = empty; P.bx = bx;

    const uint8_t* pack = reinterpret_cast<const uint8_t*>(a.d6_pack);
    const float* gparams = a.d6_params;
    constexpr int S_D = D / 64, S_NS = NS / 64;   // K slabs of a linear layer

    if (warp >= W_PROD) {
        // ===================================================== PRODUCERS: weight slabs, parameters and cross K/V, in consumer order;
        // producer warp pw issues chunks n with n % NPROD == pw (every producer walks the whole schedule)
        const uint32_t pw = (uint32_t)(warp - W_PROD);
        uint32_t n = 0, pl = 0;
        auto push = [&](const void* src, uint32_t bytes) {
            if (n % NPROD == pw) {
                const uint32_t slot = n % NSLOT;
                if (n >= NSLOT) mbar_wait_bounded(empty + slot, ((n / NSLOT) - 1) & 1, g_watchdog);
                mbar_expect_tx(full + slot, bytes);
                bulk_g2s(ring_mem + slot * SLOT, src, bytes, full + slot);
            }
            ++n;
        };
        for (int step = 0; step < a.n_steps; ++step) {
            if (lane == 0) {
                const int n_iter = BEAM ? n_live_s[step & 1] : R;
                for (int it = cluster_id; it < n_iter; it += n_clusters) {
                    const int row = BEAM ? live_rows[(step & 1) * BM_LIVE + it] : it;
                    const int w = __ldg(a.row_window + row);
                    const int T = __ldg(a.win_T + w);
                    for (int l = 0; l < L; ++l) {
                        if (pw == 0) {
                            const uint32_t b = pl & 1, u = pl >> 1;
                            if (u >= 1) mbar_wait_bounded(pfree + b, (u - 1) & 1, g_watchdog);
                            mbar_expect_tx(pfull + b, PARAMS * 4);
                            bulk_g2s(params + b * PARAMS, gparams + ((size_t)l * CS + rank) * PARAMS, PARAMS * 4, pfull + b);
                        }
                        ++pl;
                        const uint8_t* base = pack + ((size_t)l * CS + rank) * G::PACK;
                        auto seg = [&](int off, int N, int K) {   // tiles of 128 rows (last one 64), K / 64 slabs each, one bulk copy per slab
                            const uint8_t* src = base + off;
                            for (int r0 = 0; r0 < N; r0 += 128) {
                                const uint32_t bytes = (uint32_t)min(128, N - r0) * 128;
                                for (int sl = 0; sl < K / 64; ++sl, src += bytes) push(src, bytes);
                            }
                        };
                        seg(G::OFF_QKV, 192, D);
                        seg(G::OFF_O, D, 64);
                        seg(G::OFF_CQ, 64, D);
                        {
                            const KVT* kv = reinterpret_cast<const KVT*>(a.ckv) + (size_t)l * a.Mcap * 2 * D + __ldg(a.win_row_off + w) * (int64_t)(2 * D) +
                                            (int64_t)h * T * 128;
                            for (int k0 = 0; k0 < T; k0 += KPC) push(kv + (int64_t)k0 * 128, (uint32_t)(min(KPC, T - k0) * ROWB));
                        }
                        seg(G::OFF_CO, D, 64);
                        seg(G::OFF_W1, NS, D);
                        seg(G::OFF_W2, D, NS);
                    }
                }
            }
            __syncwarp();
            bar_all();   // the ring is lent to the logits stage until the consumers finish the step
            if (*reinterpret_cast<volatile int*>(ctl) != 0) break;
        }
    } else {
        // ===================================================== CONSUMERS
        Counters c{0, 0};
        uint32_t pl = 0;     // parameter blocks consumed
        uint32_t ph = 0;     // exchange phases completed (buffer = ph & 1)
        unsigned int gen = 0;
        unsigned int lg_count = 0;
        int tr_n = 0;
        const float scale = a.qk_scale;
        const int gw = blockIdx.x * NCW + warp, n_gw = gridDim.x * NCW;

        auto trace = [&]() {
            if (a.trace && blockIdx.x == 0 && tid == 0 && tr_n < a.trace_cap / 2) a.trace[tr_n++] = gtime();
        };
        // sends y_s[ph & 1] (D values + max, sum, active) to every CTA of the cluster
        auto send = [&]() {
            fence_proxy_async();
            bar_consumers();
            if (tid < CS) {   // one issuing thread per destination
                const uint32_t b = ph & 1;
                bulk_s2peer(part + (b * CS + rank) * SEND, y_s + b * SEND, SEND * 4, pbar + b, (uint32_t)tid);
            }
        };
        auto combine = [&](int mode, const float* bias) {
            combine6<D>(part + (ph & 1) * CS * SEND, pbar + (ph & 1), (ph >> 1) & 1, mode, bias, x_s, wsrc_s);
            ++ph;
        };

#pragma unroll 1
        for (int step = 0; step < a.n_steps; ++step) {
            const int p = a.pos0 + step;
            const bool want_logits = p >= a.logits_from;
            const int depth = p - a.logits_from;   // beam mode: search depth (< 0 in the prefill)
            const int n_iter = BEAM ? n_live_s[step & 1] : R;
            const int* anc_cur = depth > 0 && (depth & 1) ? a.anc_alt : a.anc;   // the prefill reads the identity table of depth 0
#pragma unroll 1
            for (int it = cluster_id; it < n_iter; it += n_clusters) {
                const int row = BEAM ? live_rows[(step & 1) * BM_LIVE + it] : it;
                // ---- embed (mod.rs:141-146): every CTA of the cluster builds its own copy of x
                {
                    const int tok = __ldcg(a.tokens + (int64_t)row * t_max + p);
                    for (int c2 = tid; c2 < D; c2 += 256) x_s[c2] = __fadd_rn(__ldg(a.tok_emb + (int64_t)tok * D + c2), __ldg(a.pos_emb + (int64_t)p * D + c2));
                }
                const int w = __ldg(a.row_window + row);
                const int T = __ldg(a.win_T + w);
                bar_consumers();
                trace();
#pragma unroll 1
                for (int l = 0; l < L; ++l) {
                    KVT* kcl = reinterpret_cast<KVT*>(a.kc) + (size_t)l * a.Rmax * t_max * D;
                    KVT* vcl = reinterpret_cast<KVT*>(a.vc) + (size_t)l * a.Rmax * t_max * D;
                    // ================= phase 1: x += MLP of the previous layer; self attention of head h (mod.rs:346)
                    if (l > 0) {
                        combine(MODE_SUM, params + ((pl + 1) & 1) * PARAMS + G::P_B2);   // previous layer's block: bias of its MLP2
                        __syncwarp();
                        if (lane == 0) mbar_arrive(pfree + ((pl + 1) & 1));               // previous layer's parameters are dead now
                    }
                    trace();   // [t1] records of the previous phase combined
                    mbar_wait_bounded(pfull + (pl & 1), (pl >> 1) & 1, g_watchdog);
                    const float* prm = params + (pl & 1) * PARAMS;
                    ++pl;
                    float* ys = y_s + (ph & 1) * SEND;
                    ln6<D>(x_s, prm + G::P_LN1G, prm + G::P_LN1B, prm[G::P_EPS + 0], a.eps_outside, bx);
                    KVT* kd = kcl + ((int64_t)row * t_max + p) * D + h * 64;
                    KVT* vd = vcl + ((int64_t)row * t_max + p) * D + h * 64;
                    c = gemv_epi6<KVT>(P, c, 192, S_D, GemvOut<KVT>{EM_QKV, prm + G::P_BQKV, scale, qkv_s, kd, vd});
                    trace();   // [t2] q | k | v done
                    if constexpr (BEAM)
                        self_attn6_anc<KVT>(qkv_s, kcl + h * 64, vcl + h * 64, D, p, anc_cur + (int64_t)row * t_max, (int64_t)t_max * D, wm, wl, wo);
                    else
                        self_attn6<KVT>(qkv_s, kcl + (int64_t)row * t_max * D + h * 64, vcl + (int64_t)row * t_max * D + h * 64, D, p, wm, wl, wo);
                    attn_merge6(wm, wl, wo, bx, ys + D);
                    trace();   // [t3] self attention done
                    c = gemv_epi6<KVT>(P, c, D, 1, GemvOut<KVT>{EM_PLAIN, nullptr, 1.0f, ys, nullptr, nullptr});
                    trace();   // [t4] out-projection slice done
                    send();
                    trace();   // [t5] sent
                    // ================= phase 2: x += self-attention output; cross attention of head h (mod.rs:347)
                    combine(MODE_ATTN, prm + G::P_BO);
                    trace();   // [t6] combined
                    ys = y_s + (ph & 1) * SEND;
                    ln6<D>(x_s, prm + G::P_LN2G, prm + G::P_LN2B, prm[G::P_EPS + 1], a.eps_outside, bx);
                    c = gemv_epi6<KVT>(P, c, 64, S_D, GemvOut<KVT>{EM_CQ, prm + G::P_BCQ, scale, q2_s, nullptr, nullptr});
                    trace();   // [t7] cross query done
                    c.n = cross_attn6<KVT>(P, c.n, slot_cnt, q2_s, T, wm, wl, wo);
                    attn_merge6(wm, wl, wo, bx, ys + D);
                    trace();   // [t8] cross attention done
                    c = gemv_epi6<KVT>(P, c, D, 1, GemvOut<KVT>{EM_PLAIN, nullptr, 1.0f, ys, nullptr, nullptr});
                    trace();   // [t9]
                    send();
                    trace();   // [t10]
                    // ================= phase 3: x += cross-attention output; MLP slice (mod.rs:348, :376-382)
                    combine(MODE_ATTN, prm + G::P_BCO);
                    trace();   // [t11]
                    ys = y_s + (ph & 1) * SEND;
                    ln6<D>(x_s, prm + G::P_LN3G, prm + G::P_LN3B, prm[G::P_EPS + 2], a.eps_outside, bx);
                    c = gemv_epi6<KVT>(P, c, NS, S_D, GemvOut<KVT>{EM_HID, prm + G::P_B1, 1.0f, hid_s, nullptr, nullptr});
                    for (int c2 = tid; c2 < NS; c2 += 256) bx_store(bx, c2, hid_s[c2]);   // every MMA of the W1 product has completed: the B operand may change
                    trace();   // [t12] hidden slice done
                    c = gemv_epi6<KVT>(P, c, D, S_NS, GemvOut<KVT>{EM_PLAIN, nullptr, 1.0f, ys, nullptr, nullptr});
                    trace();   // [t13]
                    send();
                    trace();   // [t14]
                }
                // ---- x += MLP of the last layer; rank 0 publishes the row for the vocabulary projection
                combine(MODE_SUM, params + ((pl + 1) & 1) * PARAMS + G::P_B2);
                __syncwarp();
                if (lane == 0) mbar_arrive(pfree + ((pl + 1) & 1));
                if (want_logits && rank == 0)
                    for (int c = tid; c < D; c += 256) a.x[(int64_t)row * D + c] = x_s[c];
                bar_consumers();
            }
            int stop = 0;
            if (want_logits) {
                // ---- vocabulary tiles of this warp.  CTAs of clusters without a row have nothing to do until the rows are published:
                // they take the first LG_NBUF half-tiles into their ring BEFORE the grid barrier (the embedding matrix does not depend on
                // the activations), and their warps get `na` extra tile each (stage A) so that the stream that remains after the
                // barrier is spread evenly (stage B: round robin over all warps).
                const int lg_g = lane >> 2, lg_t = lane & 3;
                constexpr int KH = D / 2, NCH = KH / 32;
                constexpr uint32_t BLKB = 16 * KH * 2;
                constexpr int RINGW = NSLOT * SLOT / NCW;
                static_assert(LG_NBUF * (int)BLKB <= RINGW, "logits ring");
                const __half* Et = reinterpret_cast<const __half*>(a.E_tiled);
                const int v_tiles = (V + 15) / 16;
                const int R_act = BEAM ? n_live_s[step & 1] : R;   // clusters >= R_act had no row this step
                const bool idle_cta = cluster_id >= R_act;
                const int n_idle_w = max(0, n_clusters - R_act) * CS * NCW;
                const int na = (n_idle_w > 0 && 2 * n_idle_w <= v_tiles) ? 1 : 0;   // = what an idle warp has in its ring when the barrier opens
                const int tiles_a = na * n_idle_w, tiles_b = v_tiles - tiles_a;
                const int iw = ((cluster_id - R_act) * CS + rank) * NCW + warp;             // index among the idle warps
                const int my_a = idle_cta ? na : 0;
                const int my_tiles = my_a + (gw < tiles_b ? (tiles_b - gw + n_gw - 1) / n_gw : 0);
                const int total = my_tiles * 2;
                auto tile_of = [&](int i) { return i < my_a ? iw + i * n_idle_w : tiles_a + gw + (i - my_a) * n_gw; };
                uint8_t* wring = ring_mem + (size_t)warp * RINGW;
                uint64_t* wbar = lg_bar + warp * LG_NBUF;
                auto issue = [&](int it) {
                    if (it < total && lane == 0) {
                        const int vt = tile_of(it >> 1);
                        const int slot = (int)((lg_count + (unsigned int)it) % LG_NBUF);
                        mbar_expect_tx(wbar + slot, BLKB);
                        bulk_g2s(wring + (size_t)slot * BLKB, Et + ((int64_t)vt * 2 + (it & 1)) * 16 * KH, BLKB, wbar + slot);
                    }
                };
                if (idle_cta) {
                    fence_proxy_async();
#pragma unroll
                    for (int j = 0; j < LG_NBUF; ++j) issue(j);
                }
                // ---- the one grid barrier of the step: every row's x is published
                trace();
                if (tid == 0) {
                    ++gen;
                    __threadfence();
                    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.bar) : "memory");
                    const unsigned int target = gen * gridDim.x;
                    const long long t0 = clock64(), wd = g_watchdog;
                    while (ld_acquire(a.bar) < target)
                        if (clock64() - t0 > wd) __trap();
                } else {
                    ++gen;
                }
                bar_consumers();
                trace();
                // ================= logits (all CTAs): LN(x) tok_emb^T + mask + online softmax + arg-max (mod.rs:155-156, transcribe.rs:271-276)
                const bool use_mask = SPECIAL_MASKED(a, p);
                const int eot_cap = !BEAM && a.loop_rules ? a.eot : -1;   // the id whose logit the greedy loop's EOT test reads
                // LayerNorm rows straight into fp16 hi / lo planes in MMA fragment order (decoder5.cu); rows >= R are zero
                for (int r = warp; r < 8 * NT8; r += NCW) {
                    constexpr int NV = D / 128;   // float4 per lane
                    float4 v[NV];
                    if (r < R && (!BEAM || live_s[(step & 1) * BM_LIVE + r])) {
#pragma unroll
                        for (int i = 0; i < NV; ++i) v[i] = __ldcg(reinterpret_cast<const float4*>(a.x + (int64_t)r * D) + lane + 32 * i);
                        float sum = 0.0f;
#pragma unroll
                        for (int i = 0; i < NV; ++i) sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
                        sum = warp_sum(sum);
                        const float mean = __fdiv_rn(sum, (float)D);
                        float q = 0.0f;
#pragma unroll
                        for (int i = 0; i < NV; ++i) {
                            v[i].x = __fsub_rn(v[i].x, mean); v[i].y = __fsub_rn(v[i].y, mean); v[i].z = __fsub_rn(v[i].z, mean); v[i].w = __fsub_rn(v[i].w, mean);
                            q = ln_sq_add4(q, v[i]);
                        }
                        q = warp_sum(q);
                        const float var = __fdiv_rn(q, (float)D);
                        const float den = LN_DEN(var, a.lnf_eps, a.eps_outside);
#pragma unroll
                        for (int i = 0; i < NV; ++i) {
                            const float4 g4 = __ldg(reinterpret_cast<const float4*>(a.lnf_g) + lane + 32 * i);
                            const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.lnf_b) + lane + 32 * i);
                            store_frag(pl_hi, pl_lo, D / 32, r, (lane + 32 * i) * 4, ln_norm4(v[i], den, g4, b4));
                        }
                    } else {
#pragma unroll
                        for (int i = 0; i < NV; ++i) store_frag(pl_hi, pl_lo, D / 32, r, (lane + 32 * i) * 4, make_float4(0.f, 0.f, 0.f, 0.f));
                    }
                }
                bar_consumers();
                trace();
                {
                    // Swap-AB tensor-core product (decoder4.cu): a warp owns tiles of 16 vocabulary rows (M), 8 batch rows per n-tile
                    // (N), K = D; the matrix is streamed as contiguous half-tiles [16][D/2] (one bulk copy each) through this warp's
                    // share of the ring, LG_NBUF - 1 copies in flight.
                    const int g = lg_g, t = lg_t;
                    float m_run[NT8][2], s_run[NT8][2], bv[NT8][2];
                    int bi[NT8][2];
#pragma unroll
                    for (int j = 0; j < NT8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) { m_run[j][e] = -INFINITY; s_run[j][e] = 0.0f; bv[j][e] = -INFINITY; bi[j][e] = INT_MAX; }
                    // beam mode: this warp's candidate list per batch row, behind its logits buffers in its share of the ring
                    constexpr int LST = 8 * NT8 * DEC_KC;
                    static_assert(!BEAM || LG_NBUF * (int)BLKB + LST * 8 <= RINGW, "beam candidate lists");
                    float* cl_v = reinterpret_cast<float*>(wring + LG_NBUF * BLKB);
                    int* cl_i = reinterpret_cast<int*>(cl_v + LST);
                    unsigned int live_m = 0;   // live batch rows
                    if constexpr (BEAM) {
                        for (int i = lane; i < LST; i += 32) { cl_v[i] = -INFINITY; cl_i[i] = INT_MAX; }
                        for (int r = 0; r < R; ++r) live_m |= live_s[(step & 1) * BM_LIVE + r] ? 1u << r : 0u;
                        __syncwarp();
                    }
                    if (!idle_cta) {
                        fence_proxy_async();   // the ring was last written by bulk copies and read through the generic proxy
#pragma unroll
                        for (int j = 0; j < LG_NBUF; ++j) issue(j);
                    }
                    float ah[NT8][4], al[NT8][4];
#pragma unroll 1
                    for (int it = 0; it < total; ++it) {
                        const unsigned int cnt = lg_count + (unsigned int)it;
                        const int slot = (int)(cnt % LG_NBUF);
                        mbar_wait_bounded(wbar + slot, (cnt / LG_NBUF) & 1, g_watchdog);
                        const uint8_t* blk = wring + (size_t)slot * BLKB;
                        const int half = it & 1;
                        if (half == 0) {
#pragma unroll
                            for (int j = 0; j < NT8; ++j)
#pragma unroll
                                for (int c = 0; c < 4; ++c) { ah[j][c] = 0.0f; al[j][c] = 0.0f; }
                        }
#pragma unroll
                        for (int c = 0; c < NCH; ++c) {
                            const uint4 a0 = *reinterpret_cast<const uint4*>(blk + (size_t)g * (KH * 2) + c * 64 + t * 16);
                            const uint4 a8 = *reinterpret_cast<const uint4*>(blk + (size_t)(g + 8) * (KH * 2) + c * 64 + t * 16);
                            const int chunk = half * NCH + c;
#pragma unroll
                            for (int j = 0; j < NT8; ++j) {
                                const uint4 bh = pl_hi[(j * (D / 32) + chunk) * 32 + lane];
                                const uint4 bl = pl_lo[(j * (D / 32) + chunk) * 32 + lane];
                                mma16816(ah[j], a0.x, a8.x, a0.y, a8.y, bh.x, bh.y);
                                mma16816(ah[j], a0.z, a8.z, a0.w, a8.w, bh.z, bh.w);
                                mma16816(al[j], a0.x, a8.x, a0.y, a8.y, bl.x, bl.y);
                                mma16816(al[j], a0.z, a8.z, a0.w, a8.w, bl.z, bl.w);
                            }
                        }
                        if (BEAM && half == 1) {
                            // as below, but every value is a candidate: the lanes of one g insert theirs into the warp's
                            // per-row lists, g by g (the four lanes of one g own distinct rows)
                            const int n0 = tile_of(it >> 1) * 16;
                            float cv[NT8][4];
#pragma unroll
                            for (int j = 0; j < NT8; ++j)
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    const int n = n0 + g + (c >> 1) * 8, e = c & 1, rr = j * 8 + 2 * t + e;
                                    cv[j][c] = __int_as_float(0x7fffffff);   // NaN: never inserted
                                    if (n < V && rr < R && ((live_m >> rr) & 1u)) {
                                        const float raw = hl_join(ah[j][c], al[j][c]);
                                        const float v = (use_mask && a.is_special[n]) ? __fadd_rn(raw, -INFINITY) : raw;
                                        if (v > -INFINITY) softmax_add(m_run[j][e], s_run[j][e], v);
                                        cv[j][c] = v;
                                    }
                                }
#pragma unroll 1
                            for (int gi = 0; gi < 8; ++gi) {
                                if (g == gi) {
#pragma unroll
                                    for (int j = 0; j < NT8; ++j)
#pragma unroll
                                        for (int c = 0; c < 4; ++c) {
                                            const int rr = j * 8 + 2 * t + (c & 1);
                                            cand_insert(cl_v + rr * DEC_KC, cl_i + rr * DEC_KC, cv[j][c], n0 + g + (c >> 1) * 8);
                                        }
                                }
                                __syncwarp();
                            }
                        } else if (half == 1) {
                            // C fragment: c0,c1 -> (vocabulary row g, batch rows 2t, 2t+1), c2,c3 -> (row g+8, same batch rows)
                            const int n0 = tile_of(it >> 1) * 16;
#pragma unroll
                            for (int j = 0; j < NT8; ++j)
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    const int n = n0 + g + (c >> 1) * 8, e = c & 1;
                                    if (n < V && j * 8 + 2 * t + e < R) {
                                        const float raw = hl_join(ah[j][c], al[j][c]);
                                        const float v = (use_mask && a.is_special[n]) ? __fadd_rn(raw, -INFINITY) : raw;
                                        if (v > -INFINITY) softmax_add(m_run[j][e], s_run[j][e], v);
                                        if (cand_better(v, n, bv[j][e], bi[j][e])) { bv[j][e] = v; bi[j][e] = n; }
                                        if (n == eot_cap) a.eot_logit[j * 8 + 2 * t + e] = v;
                                    }
                                }
                        }
                        __syncwarp();                 // every lane is done with the slot
                        issue(it + LG_NBUF);
                    }
                    lg_count += (unsigned int)total;
                    trace();
                    // merge the 8 lanes that share t (batch rows 2t, 2t+1 of every n-tile), then the 8 warps through shared memory
#pragma unroll
                    for (int j = 0; j < NT8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
#pragma unroll
                            for (int off = 4; off < 32; off <<= 1) {
                                softmax_merge(m_run[j][e], s_run[j][e], __shfl_xor_sync(0xffffffffu, m_run[j][e], off),
                                              __shfl_xor_sync(0xffffffffu, s_run[j][e], off));
                                if (!BEAM) cand_xor(bv[j][e], bi[j][e], off);
                            }
                            if (g == 0) {
                                float* rec = red + (warp * 8 * NT8 + j * 8 + 2 * t + e) * 4;
                                rec[0] = m_run[j][e]; rec[1] = s_run[j][e]; rec[2] = bv[j][e]; rec[3] = __int_as_float(bi[j][e]);
                            }
                        }
                    bar_consumers();
                    if (BEAM && tid < R && ((live_m >> tid) & 1u)) {
                        // the CTA's record of a live row: (max, sum-exp) of the 8 warps, and its DEC_KC best (value, id) from their
                        // lists, merged into warp 0's list (each list is sorted: the first entry that stays out ends a list)
                        const float2 ms = fold_softmax(red + tid * 4, NCW, 8 * NT8 * 4);
                        float* acc_v = reinterpret_cast<float*>(ring_mem + LG_NBUF * BLKB) + tid * DEC_KC;
                        int* acc_i = reinterpret_cast<int*>(reinterpret_cast<float*>(ring_mem + LG_NBUF * BLKB) + LST) + tid * DEC_KC;
                        for (int w2 = 1; w2 < NCW; ++w2) {
                            const float* sv = reinterpret_cast<const float*>(ring_mem + (size_t)w2 * RINGW + LG_NBUF * BLKB) + tid * DEC_KC;
                            const int* si = reinterpret_cast<const int*>(reinterpret_cast<const float*>(ring_mem + (size_t)w2 * RINGW + LG_NBUF * BLKB) + LST) + tid * DEC_KC;
                            for (int k = 0; k < DEC_KC; ++k)
                                if (!cand_insert(acc_v, acc_i, sv[k], si[k])) break;
                        }
                        const int64_t o = (int64_t)blockIdx.x * R + tid;
                        a.lg_m[o] = ms.x;
                        a.lg_s[o] = ms.y;
#pragma unroll
                        for (int k = 0; k < DEC_KC; ++k) { a.lg_v[o * DEC_KC + k] = acc_v[k]; a.lg_i[o * DEC_KC + k] = acc_i[k]; }
                    } else if (!BEAM && tid < R) {
                        fold_records_top1(a, red + tid * 4, NCW, 8 * NT8 * 4, (int64_t)blockIdx.x * R + tid);
                    }
                }
                trace();
                // ================= finish (greedy: beam.rs:9-37 with beam_size 1) by the LAST CTA to deliver its records
                bar_consumers();
                if (tid == 0) ctl[1] = last_ticket(a.bar, gen);
                bar_consumers();
                if (ctl[1]) {
                    __threadfence();
                    if constexpr (BEAM) {
                        finish_beam(a, p, depth, anc_cur, ring_mem, live_s + (step & 1) * BM_LIVE, nx_s, ctl);
                    } else {
                        // <= 160 co-resident CTAs: at most 5 records per lane
                        for (int r = warp; r < R; r += NCW) finish_row_top1<5>(a, r, p, gridDim.x);
                    }
                    bar_consumers();
                    if (tid == 0) release_flag(a.bar, gen);
                }
                if (tid == 0) wait_flag(a.bar, gen, g_watchdog);
                bar_consumers();
                trace();
                if constexpr (BEAM) {
                    stop = __ldcg(a.bar + 3) != 0;   // set by the finisher when the search ended
                } else if (rows_open(a) == 0) {
                    stop = 1;
                    if (blockIdx.x == 0 && tid == 0) decode_done(a, p + 1, 0, step + 1);
                }
            }
            if constexpr (BEAM) {
                if (!stop) snapshot_live((step + 1) & 1);   // the next position's live slots (the finisher placed them)
            }
            if (tid == 0) ctl[0] = stop;
            fence_proxy_async();   // generic accesses to the aliased buffers before the next step's bulk copies
            bar_all();   // hands the ring back to the producer; it reads the stop flag after this barrier
            if (stop) break;
            if (!BEAM && step + 1 == a.n_steps && blockIdx.x == 0 && tid == 0) decode_done(a, a.pos0 + a.n_steps, rows_open(a), a.n_steps);
        }
    }
    cl.sync();   // no CTA leaves while a peer may still address its shared memory
}

template <int D, int NT8, bool BEAM = false>
constexpr size_t dec6_smem() {
    using G = Geo<D>;
    return 1024 + (size_t)NSLOT * SLOT + (size_t)(G::KMAX / 64) * BX_SLAB +
           sizeof(float) * ((size_t)2 * G::PARAMS + 2 * G::CS * G::SEND + 2 * G::SEND + D + 192 + 64 + G::NS + 16 + 8 + 8 + 512 + 4 + NSLOT) +
           8 * (size_t)(2 * NSLOT + 6 + NCW * LG_NBUF) + 64 + (BEAM ? sizeof(int) * (4 * BM_LIVE + 2 + BM_NX) : 0);
}

template <int D, int NT8, typename KVT, bool BEAM = false>
bool launch6_t(const DecArgs& a, cudaStream_t st) {
    using G = Geo<D>;
    static_assert((size_t)2 * NT8 * (D / 32) * 32 * 16 + (size_t)NCW * 8 * NT8 * 16 <= sizeof(float) * (2 * G::PARAMS + 2 * G::CS * G::SEND), "logits scratch must fit the aliased buffers");
    const void* k = (const void*)dec6_kernel<D, NT8, KVT, BEAM>;
    const size_t smem = dec6_smem<D, NT8, BEAM>();
    static ClusterLaunch cl;   // per instantiation
    const int n_cl = cl.capacity(k, G::CS, NTH6, smem, "dec6");
    if (n_cl < 1) return false;
    static PerDeviceConfig wd;
    wd.ensure(1, [] {
        if (const char* e = getenv("WB200_WATCHDOG_MS")) {   // 0 = never trap
            const long long ms = atoll(e);
            const long long cyc = ms <= 0 ? (1LL << 62) : ms * 2000000LL;
            WB_CUDA(cudaMemcpyToSymbol(g_watchdog, &cyc, sizeof(cyc)));
        }
        return true;
    });
    // every launched cluster must be co-resident (grid barrier): launch what the device holds; rows beyond that are looped over
    void* args[] = {(void*)&a};
    cl.launch(k, G::CS, n_cl, NTH6, smem, args, st, "dec6");
    return true;
}

// ---- host: packed weights / parameter blocks of a model (built once per session) ----------------------------------------------
template <int D>
void build_pack_t(const Model& m, Dec6Pack& pk, cudaStream_t st) {
    using G = Geo<D>;
    const int L = m.dims.n_text_layer;
    pk.pack.alloc((size_t)L * G::CS * G::PACK);
    pk.params.alloc((size_t)L * G::CS * G::PARAMS);
    std::vector<PackSeg> ps;
    std::vector<ParamSeg> qs;
    std::vector<float> eps_h((size_t)L * 4, 0.0f);
    for (int l = 0; l < L; ++l) {
        const DecBlockW& B = m.dec[(size_t)l];
        eps_h[(size_t)l * 4] = B.attn_ln.eps; eps_h[(size_t)l * 4 + 1] = B.cross_ln.eps; eps_h[(size_t)l * 4 + 2] = B.mlp_ln.eps;
    }
    DevBuf<float> eps_d;
    eps_d.alloc(eps_h.size());
    WB_CUDA(cudaMemcpyAsync(eps_d.p, eps_h.data(), eps_h.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    for (int l = 0; l < L; ++l) {
        const DecBlockW& B = m.dec[(size_t)l];
        for (int h = 0; h < G::CS; ++h) {   // CTA h of a cluster owns attention head h
            const int64_t base = ((int64_t)l * G::CS + h) * G::PACK;
            const int64_t pb = ((int64_t)l * G::CS + h) * G::PARAMS;
            // q_h | k_h | v_h: three 64-row pieces of the fused [3d][d] matrix, d rows apart
            ps.push_back(PackSeg{B.qkv.w16, D, h * 64, 0, 192, D, 64, D, base + G::OFF_QKV});
            ps.push_back(PackSeg{B.out.w16, D, 0, h * 64, D, 64, D, 0, base + G::OFF_O});
            ps.push_back(PackSeg{B.cq.w16, D, h * 64, 0, 64, D, 64, 0, base + G::OFF_CQ});
            ps.push_back(PackSeg{B.cout.w16, D, 0, h * 64, D, 64, D, 0, base + G::OFF_CO});
            ps.push_back(PackSeg{B.mlp1.w16, D, h * G::NS, 0, G::NS, D, G::NS, 0, base + G::OFF_W1});
            ps.push_back(PackSeg{B.mlp2.w16, 4 * D, 0, h * G::NS, D, G::NS, D, 0, base + G::OFF_W2});
            qs.push_back(ParamSeg{B.attn_ln.g, D, pb + G::P_LN1G}); qs.push_back(ParamSeg{B.attn_ln.b, D, pb + G::P_LN1B});
            qs.push_back(ParamSeg{B.cross_ln.g, D, pb + G::P_LN2G}); qs.push_back(ParamSeg{B.cross_ln.b, D, pb + G::P_LN2B});
            qs.push_back(ParamSeg{B.mlp_ln.g, D, pb + G::P_LN3G}); qs.push_back(ParamSeg{B.mlp_ln.b, D, pb + G::P_LN3B});
            qs.push_back(ParamSeg{B.out.b, D, pb + G::P_BO}); qs.push_back(ParamSeg{B.cout.b, D, pb + G::P_BCO}); qs.push_back(ParamSeg{B.mlp2.b, D, pb + G::P_B2});
            for (int part = 0; part < 3; ++part) qs.push_back(ParamSeg{B.qkv.b + part * D + h * 64, 64, pb + G::P_BQKV + part * 64});
            qs.push_back(ParamSeg{B.cq.b + h * 64, 64, pb + G::P_BCQ});
            qs.push_back(ParamSeg{B.mlp1.b + h * G::NS, G::NS, pb + G::P_B1});
            qs.push_back(ParamSeg{eps_d.p + (size_t)l * 4, 4, pb + G::P_EPS});
        }
    }
    DevBuf<PackSeg> dps;
    DevBuf<ParamSeg> dqs;
    dps.alloc(ps.size());
    dqs.alloc(qs.size());
    WB_CUDA(cudaMemcpyAsync(dps.p, ps.data(), ps.size() * sizeof(PackSeg), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(dqs.p, qs.data(), qs.size() * sizeof(ParamSeg), cudaMemcpyHostToDevice, st));
    dec6_pack_kernel<<<dim3(32, (unsigned)std::min<size_t>(ps.size(), 1024)), 256, 0, st>>>(dps.p, (int)ps.size(), pk.pack.p);
    WB_LAUNCH_CHECK();
    dec6_param_kernel<<<(unsigned)std::min<size_t>(qs.size(), 2048), 128, 0, st>>>(dqs.p, (int)qs.size(), pk.params.p);
    WB_LAUNCH_CHECK();
    WB_CUDA(cudaStreamSynchronize(st));   // the descriptor arrays go out of scope
}

}  // namespace

// Returns false when this configuration is not covered.  The packed weights are built on the first launch.
//   greedy: k = 1, identity ancestry (a.anc == nullptr);
//   beam search (a.beam = B in 2..7): rows = n_win * B, prefill from position 0, ancestry tables anc / anc_alt, k = B.
bool launch_dec6(DecArgs a, const Model& m, Dec6Pack& pk, cudaStream_t st) {
    const bool beam = a.beam > 1;
    if (!m.fp16_exact || a.R > BM_LIVE || a.R < 1 || a.use_cur_tok || a.logits_out != nullptr) return false;
    if (!beam && (a.k != 1 || !a.greedy || a.anc != nullptr)) return false;
    if (beam && (a.beam > beamfx::MAX_BEAM || a.k != a.beam || a.greedy || a.R != a.n_win * a.beam || a.pos0 != 0 || a.max_depth < 1 ||
                 a.anc == nullptr || a.anc_alt == nullptr || a.slot_live == nullptr || a.bm_head == nullptr)) return false;
    if ((a.d != 128 && a.d != 384) || a.H * 64 != a.d || a.E_tiled == nullptr || a.t_max > 128) return false;
    if (pk.pack.p == nullptr) {
        if (a.d == 384) build_pack_t<384>(m, pk, st);
        else build_pack_t<128>(m, pk, st);
    }
    a.d6_pack = pk.pack.p;
    a.d6_params = pk.params.p;
#define WB_D6(DD, NT8_)                                                                                                  \
    (beam ? (a.kv_half ? launch6_t<DD, NT8_, __half, true>(a, st) : launch6_t<DD, NT8_, float, true>(a, st))             \
          : (a.kv_half ? launch6_t<DD, NT8_, __half>(a, st) : launch6_t<DD, NT8_, float>(a, st)))
    if (a.d == 384) return a.R <= 8 ? WB_D6(384, 1) : WB_D6(384, 3);
    return a.R <= 8 ? WB_D6(128, 1) : WB_D6(128, 3);
#undef WB_D6
}

}  // namespace wb
