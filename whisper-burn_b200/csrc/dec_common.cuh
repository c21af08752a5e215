// Device helpers shared by the persistent decoders decoder3.cu .. decoder6.cu: staging, GEMV and attention building blocks,
// and the one definition of the candidate ranking, the softmax state, the per-(CTA, row) record and the per-row finish.
// Internal; everything lives in an anonymous namespace of the including TU.
#pragma once
#include <algorithm>
#include <type_traits>
#include <cfloat>
#include <cuda_fp16.h>
#include <climits>

#include "../host/loop_rules.hpp"
#include "decoder.h"
#include "wb_internal.h"
#include "prims.cuh"

namespace wb {

namespace {

constexpr int NT = 256;
constexpr int NW = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void cvt8(const uint4& u, float (&w)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h[i]);
        w[2 * i] = f.x;
        w[2 * i + 1] = f.y;
    }
}
__device__ __forceinline__ unsigned int ld_acquire(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// ---- L2 eviction priorities -------------------------------------------------------------------------
// A persistent decoder reads the same streams at every position.  When their sum exceeds the L2 (H100: 50 MB), near-LRU
// replacement evicts every line of a cyclic stream before its reuse.  Per-instruction hints split the streams into
// lines to keep (evict_last) and lines read once per position (evict_first); no device-wide L2 carve-out is involved.
// A kernel that marks lines evict_last demotes them again before it exits (l2_demote), so no priority outlives the launch.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// read-only 16-byte / 1-byte loads with an L2 policy
__device__ __forceinline__ uint4 ldg_l2(const uint4* p, uint64_t pol) {
    uint4 v;
    asm("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ unsigned int ldg_l2(const uint8_t* p, uint64_t pol) {
    unsigned int v;
    asm("ld.global.nc.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}
// Back to normal priority: the 128-byte lines of [p, p + bytes) that are resident, line i handled by thread (i - first) % nthreads
// == tid of the calling grid (p need not be aligned: applypriority addresses the line that contains the address)
__device__ __forceinline__ void l2_demote(const void* p, size_t bytes, size_t tid, size_t nthreads) {
    if (p == nullptr) return;
    const uintptr_t b0 = reinterpret_cast<uintptr_t>(p) & ~uintptr_t(127), e = reinterpret_cast<uintptr_t>(p) + bytes;
    for (uintptr_t q = b0 + tid * 128; q < e; q += nthreads * 128)
        asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(q) : "memory");
}

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// optional stage trace (CTA 0, thread 0): pairs of (stage end, barrier end) nanosecond stamps
#define WB_TRACE()                                                                          \
    do {                                                                                    \
        if (a.trace && blockIdx.x == 0 && threadIdx.x == 0 && tr_n < a.trace_cap) a.trace[tr_n++] = gtime(); \
    } while (0)

// Grid barrier on a monotonic counter (zeroed by the host before the launch): arrive with a one-way
// red.release (no returned value to wait for), then poll until all CTAs of this round have arrived.
// All CTAs are co-resident (cooperative launch).  `gen` counts the barriers this CTA has passed.
__device__ __forceinline__ void grid_sync(unsigned int* bar, unsigned int& gen) {
    __syncthreads();
    if (threadIdx.x == 0) {
        ++gen;
        const unsigned int target = gen * gridDim.x;
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
        long long t0 = clock64();
        while (ld_acquire(bar) < target) {
            if (clock64() - t0 > 40000000000LL) __trap();   // ~20 s of SM clocks (profilers and sanitizers slow a launch down a lot): fail loudly instead of hanging the GPU
        }
    }
    __syncthreads();
}

// ---- input staging ---------------------------------------------------------------------------------
// LayerNorm (burn 0.9 form, prims.cuh) of rows [r0, r0+RC) of src (L2) into xs[RC][d]; warp per row.
// The row is fetched with ONE batch of independent 16-byte loads (d <= 1280 -> <= 10 per lane) and stays in
// registers through mean / variance / normalisation: a single L2 round trip per stage.
constexpr int LN_V4 = 10;
template <int RC>
__device__ __forceinline__ void stage_ln(const float* src, int r0, int R, int d, const float* __restrict__ g,
                                         const float* __restrict__ b, float eps, int eps_outside, float* xs) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nv = d / 4;
    for (int rr = warp; rr < RC; rr += NW) {
        float4* xr = reinterpret_cast<float4*>(xs + rr * d);
        const int r = r0 + rr;
        if (r >= R) {
            for (int c = lane; c < nv; c += 32) xr[c] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        const float4* s4 = reinterpret_cast<const float4*>(src + (int64_t)r * d);
        float4 v[LN_V4];
#pragma unroll
        for (int i = 0; i < LN_V4; ++i) {
            const int c = i * 32 + lane;
            v[i] = c < nv ? __ldcg(s4 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float sum = 0.0f;
#pragma unroll
        for (int i = 0; i < LN_V4; ++i) sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        sum = warp_sum(sum);
        const float mean = __fdiv_rn(sum, (float)d);
        float q = 0.0f;
#pragma unroll
        for (int i = 0; i < LN_V4; ++i) {
            const int c = i * 32 + lane;
            if (c < nv) {
                v[i].x = __fsub_rn(v[i].x, mean); v[i].y = __fsub_rn(v[i].y, mean);
                v[i].z = __fsub_rn(v[i].z, mean); v[i].w = __fsub_rn(v[i].w, mean);
                q = ln_sq_add4(q, v[i]);
            }
        }
        q = warp_sum(q);
        const float var = __fdiv_rn(q, (float)d);
        const float den = LN_DEN(var, eps, eps_outside);
#pragma unroll
        for (int i = 0; i < LN_V4; ++i) {
            const int c = i * 32 + lane;
            if (c < nv) {
                const float4 g4 = __ldg(reinterpret_cast<const float4*>(g) + c);
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(b) + c);
                xr[c] = ln_norm4(v[i], den, g4, b4);
            }
        }
    }
}

// same LayerNorm, source rows already in shared memory (src_s[rr][d])
template <int RC>
__device__ __forceinline__ void stage_ln_smem(const float* src_s, int r0, int R, int d, const float* __restrict__ g,
                                              const float* __restrict__ b, float eps, int eps_outside, float* xs) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int rr = warp; rr < RC; rr += NW) {
        float* xr = xs + rr * d;
        if (r0 + rr >= R) {
            for (int c = lane; c < d; c += 32) xr[c] = 0.0f;
            continue;
        }
        const float* s = src_s + rr * d;
        float sum = 0.0f;
        for (int c = lane; c < d; c += 32) sum += s[c];
        sum = warp_sum(sum);
        const float mean = __fdiv_rn(sum, (float)d);
        float q = 0.0f;
        for (int c = lane; c < d; c += 32) {
            q = ln_sq_add(q, __fsub_rn(s[c], mean));
        }
        q = warp_sum(q);
        const float var = __fdiv_rn(q, (float)d);
        const float den = LN_DEN(var, eps, eps_outside);
        for (int c = lane; c < d; c += 32)
            xr[c] = ln_norm<true>(__fsub_rn(s[c], mean), den, g, b, c);
    }
}

// copies rows [r0, r0+RC) of src[R][K] (L2) into xs[RC][K]; 8 independent 16-byte loads per thread in flight
template <int RC>
__device__ __forceinline__ void stage_copy(const float* src, int r0, int R, int K, float* xs) {
    const int n4 = RC * K / 4;
    for (int i0 = threadIdx.x; i0 < n4; i0 += NT * 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * NT;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < n4) {
                const int rr = (i * 4) / K, c = (i * 4) % K;
                if (r0 + rr < R) v[u] = __ldcg(reinterpret_cast<const float4*>(src + (int64_t)(r0 + rr) * K + c));
            }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * NT;
            if (i < n4) *reinterpret_cast<float4*>(xs + (int64_t)i * 4) = v[u];
        }
    }
}

// ---- weight-slice GEMV --------------------------------------------------------------------------------
// Every warp of the grid owns output features n = gw, gw + n_warps, ...; two features are in flight.
// emit(n, rr, value) is called by lane 0 semantics-free (all lanes hold the sums; lane rr handles row rr).
template <int RC>
__device__ __forceinline__ float dot8_acc(const float (&w)[8], const float* xs, float acc) {
    const float4 x0 = *reinterpret_cast<const float4*>(xs);
    const float4 x1 = *reinterpret_cast<const float4*>(xs + 4);
    acc = fmaf(w[0], x0.x, acc); acc = fmaf(w[1], x0.y, acc); acc = fmaf(w[2], x0.z, acc); acc = fmaf(w[3], x0.w, acc);
    acc = fmaf(w[4], x1.x, acc); acc = fmaf(w[5], x1.y, acc); acc = fmaf(w[6], x1.z, acc); acc = fmaf(w[7], x1.w, acc);
    return acc;
}

// dots of G weight rows (K elements each, full warp per row, lane-strided 16-byte vectors) with the RC
// staged rows; all G rows' loads are issued before any is consumed; results in all lanes.
template <typename WT, int RC, int G>
__device__ __forceinline__ void rows_dot(const WT* (&wrow)[G], int K, const float* xs, float (&acc)[G][RC]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int rr = 0; rr < RC; ++rr) acc[g][rr] = 0.0f;
    const int nv = K / 8;
    constexpr int U = (sizeof(WT) == 2) ? (G == 1 ? 6 : 3) : (G == 1 ? 3 : 2);   // vectors per lane and row in flight
    for (int v0 = 0; v0 < nv; v0 += 32 * U) {
        if constexpr (sizeof(WT) == 2) {
            uint4 raw[G][U];
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
                for (int i = 0; i < U; ++i) {
                    const int v = v0 + i * 32 + lane;
                    raw[g][i] = v < nv ? __ldg(reinterpret_cast<const uint4*>(wrow[g]) + v) : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
            for (int i = 0; i < U; ++i) {
                const int v = v0 + i * 32 + lane;
                if (v < nv) {
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        float w[8];
                        cvt8(raw[g][i], w);
#pragma unroll
                        for (int rr = 0; rr < RC; ++rr) acc[g][rr] = dot8_acc<RC>(w, xs + rr * K + v * 8, acc[g][rr]);
                    }
                }
            }
        } else {
            float4 ra[G][U], rb[G][U];
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
                for (int i = 0; i < U; ++i) {
                    const int v = v0 + i * 32 + lane;
                    if (v < nv) {
                        ra[g][i] = __ldg(reinterpret_cast<const float4*>(wrow[g]) + 2 * v);
                        rb[g][i] = __ldg(reinterpret_cast<const float4*>(wrow[g]) + 2 * v + 1);
                    } else {
                        ra[g][i] = make_float4(0.f, 0.f, 0.f, 0.f);
                        rb[g][i] = ra[g][i];
                    }
                }
#pragma unroll
            for (int i = 0; i < U; ++i) {
                const int v = v0 + i * 32 + lane;
                if (v < nv) {
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        const float w[8] = {ra[g][i].x, ra[g][i].y, ra[g][i].z, ra[g][i].w, rb[g][i].x, rb[g][i].y, rb[g][i].z, rb[g][i].w};
#pragma unroll
                        for (int rr = 0; rr < RC; ++rr) acc[g][rr] = dot8_acc<RC>(w, xs + rr * K + v * 8, acc[g][rr]);
                    }
                }
            }
        }
    }
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int rr = 0; rr < RC; ++rr) acc[g][rr] = warp_sum(acc[g][rr]);
}

// Weight-slice GEMV phase: output features n = gw, gw + n_gw, ... two at a time; emit(n, acc[RC]) in all lanes.
template <typename WT, int RC, typename Emit>
__device__ __forceinline__ void gemv_phase(const WT* W, int N, int K, const float* xs, int gw, int n_gw, Emit&& emit) {
    for (int n = gw; n < N; n += 2 * n_gw) {
        const int n2 = n + n_gw;
        if (n2 < N) {
            const WT* rows[2] = {W + (int64_t)n * K, W + (int64_t)n2 * K};
            float acc[2][RC];
            rows_dot<WT, RC, 2>(rows, K, xs, acc);
            emit(n, acc[0]);
            emit(n2, acc[1]);
        } else {
            const WT* rows[1] = {W + (int64_t)n * K};
            float acc[1][RC];
            rows_dot<WT, RC, 1>(rows, K, xs, acc);
            emit(n, acc[0]);
        }
    }
}

// 8 lanes per weight row: a warp instruction covers 4 consecutive rows, G such groups in flight; after the
// call every lane of sub-group `sub` holds acc[g][rr] of row (g*4 + sub).  Used by the logits stage.
template <typename WT, int RC, int G>
__device__ __forceinline__ void dot_groups(const WT* (&wrow)[G], const float* xs, int K, float (&acc)[G][RC]) {
    const int l = threadIdx.x & 7;
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int rr = 0; rr < RC; ++rr) acc[g][rr] = 0.0f;
#pragma unroll 6
    for (int k0 = l * 8; k0 < K; k0 += 64) {
        float w[G][8];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            if constexpr (sizeof(WT) == 2) {
                cvt8(__ldg(reinterpret_cast<const uint4*>(wrow[g] + k0)), w[g]);
            } else {
                const float4 a4 = __ldg(reinterpret_cast<const float4*>(wrow[g] + k0));
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(wrow[g] + k0) + 1);
                w[g][0] = a4.x; w[g][1] = a4.y; w[g][2] = a4.z; w[g][3] = a4.w;
                w[g][4] = b4.x; w[g][5] = b4.y; w[g][6] = b4.z; w[g][7] = b4.w;
            }
        }
#pragma unroll
        for (int rr = 0; rr < RC; ++rr)
#pragma unroll
            for (int g = 0; g < G; ++g) acc[g][rr] = dot8_acc<RC>(w[g], xs + rr * K + k0, acc[g][rr]);
    }
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int rr = 0; rr < RC; ++rr) {
            float v = acc[g][rr];
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            acc[g][rr] = v;
        }
}

template <int RC>
__device__ __forceinline__ float pick_row(const float (&acc)[RC], int rr) {
    float v = acc[0];
#pragma unroll
    for (int i = 1; i < RC; ++i) v = (rr == i) ? acc[i] : v;
    return v;
}

// ---- attention of one query row over keys, one warp, 4 lanes per key, online softmax ------------------
struct AttnAcc {
    float m, l, o[16];
};
// One key per 4-lane group, held in registers (lane l4 of the group owns dims l4*16 .. +16): score, online-softmax update.
__device__ __forceinline__ void attn_regs_step(const float (&q)[16], const float4 (&kk)[4], const float4 (&vv)[4], bool ok, AttnAcc& A) {
    float s = 0.0f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        s = fmaf(q[c * 4], kk[c].x, s); s = fmaf(q[c * 4 + 1], kk[c].y, s);
        s = fmaf(q[c * 4 + 2], kk[c].z, s); s = fmaf(q[c * 4 + 3], kk[c].w, s);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if (ok) {
        const float mn = fmaxf(A.m, s);
        const float corr = expf(A.m - mn);
        const float e = expf(s - mn);
        A.l = A.l * corr + e;
        A.m = mn;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            A.o[c * 4] = fmaf(e, vv[c].x, A.o[c * 4] * corr);
            A.o[c * 4 + 1] = fmaf(e, vv[c].y, A.o[c * 4 + 1] * corr);
            A.o[c * 4 + 2] = fmaf(e, vv[c].z, A.o[c * 4 + 2] * corr);
            A.o[c * 4 + 3] = fmaf(e, vv[c].w, A.o[c * 4 + 3] * corr);
        }
    }
}
// merge the 8 key sub-groups of a warp (all lanes end with the warp's m, l and their 16 dims of o)
__device__ __forceinline__ void attn_merge_subs(AttnAcc& A) {
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, A.m, off);
        const float l2 = __shfl_xor_sync(0xffffffffu, A.l, off);
        const float mn = fmaxf(A.m, m2);
        const float c1 = A.m > -INFINITY ? expf(A.m - mn) : 0.0f;
        const float c2 = m2 > -INFINITY ? expf(m2 - mn) : 0.0f;
        A.l = A.l * c1 + l2 * c2;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const float o2 = __shfl_xor_sync(0xffffffffu, A.o[c], off);
            A.o[c] = A.o[c] * c1 + o2 * c2;
        }
        A.m = mn;
    }
}
// swz >= 0: the keys come from the head-major cross K/V layout (encoder.cu ckv_relayout_kernel), whose 16-byte chunks are
// XOR-4 swizzled on odd positions (swz = absolute position of key 0); the lane then finds its 16 dims one block over.
template <typename KF, typename VF>
__device__ __forceinline__ void attn_warp(const float* q_smem, int n_keys, int first, int stride, KF&& kptr, VF&& vptr,
                                          AttnAcc& A, int swz = -1) {
    const int lane = threadIdx.x & 31, sub = lane >> 2, l4 = lane & 3;
    float q[16];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float4 t = *reinterpret_cast<const float4*>(q_smem + l4 * 16 + c * 4);
        q[c * 4] = t.x; q[c * 4 + 1] = t.y; q[c * 4 + 2] = t.z; q[c * 4 + 3] = t.w;
    }
    A.m = -INFINITY;
    A.l = 0.0f;
#pragma unroll
    for (int c = 0; c < 16; ++c) A.o[c] = 0.0f;
    constexpr int UK = 2;
    for (int jb = first; jb < n_keys; jb += stride * 8 * UK) {
        float4 kk[UK][4], vv[UK][4];
        bool ok[UK];
        using KT = typename std::remove_cv<typename std::remove_pointer<decltype(kptr(0))>::type>::type;
#pragma unroll
        for (int u = 0; u < UK; ++u) {
            const int j = jb + (u * 8 + sub) * stride;
            ok[u] = j < n_keys;
            if (ok[u]) {
                const int par = swz >= 0 ? ((swz + j) & 1) : 0;
                if constexpr (sizeof(KT) == 4) {
                    const float4* kp = reinterpret_cast<const float4*>(kptr(j)) + (l4 ^ par) * 4;
                    const float4* vp = reinterpret_cast<const float4*>(vptr(j)) + (l4 ^ par) * 4;
#pragma unroll
                    for (int c = 0; c < 4; ++c) { kk[u][c] = __ldcg(kp + c); vv[u][c] = __ldcg(vp + c); }
                } else {   // fp16 cache: 16 dims = 32 bytes = two 16-byte loads
                    const uint4* kp = reinterpret_cast<const uint4*>(kptr(j)) + (l4 ^ (2 * par)) * 2;
                    const uint4* vp = reinterpret_cast<const uint4*>(vptr(j)) + (l4 ^ (2 * par)) * 2;
                    uint4 kr[2], vr[2];
                    kr[0] = __ldcg(kp); kr[1] = __ldcg(kp + 1); vr[0] = __ldcg(vp); vr[1] = __ldcg(vp + 1);
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        float w[8];
                        cvt8(kr[c], w);
                        kk[u][2 * c] = make_float4(w[0], w[1], w[2], w[3]); kk[u][2 * c + 1] = make_float4(w[4], w[5], w[6], w[7]);
                        cvt8(vr[c], w);
                        vv[u][2 * c] = make_float4(w[0], w[1], w[2], w[3]); vv[u][2 * c + 1] = make_float4(w[4], w[5], w[6], w[7]);
                    }
                }
            } else {
#pragma unroll
                for (int c = 0; c < 4; ++c) { kk[u][c] = make_float4(0.f, 0.f, 0.f, 0.f); vv[u][c] = kk[u][c]; }
            }
        }
#pragma unroll
        for (int u = 0; u < UK; ++u) attn_regs_step(q, kk[u], vv[u], ok[u], A);
    }
    attn_merge_subs(A);
}

// Ring variant for long key ranges (cross attention over up to 1500 encoder positions): K/V go global -> shared
// memory with cp.async into a per-warp ring (lane-private slots, no registers held while in flight), NSTG-1 batches
// of 8 keys in flight per warp, so the loop runs at memory throughput instead of one memory latency per batch.
// ring: this warp's NSTG * 8 * NV2 * 32 uint4 (NV2 = 16-byte vectors of K plus V per lane and key: 8 fp32 / 4 fp16).
template <int NSTG, typename KF, typename VF>
__device__ __forceinline__ void attn_warp_ring(const float* q_smem, int n_keys, int first, int stride, KF&& kptr, VF&& vptr,
                                               uint4* ring, AttnAcc& A, int swz = -1) {
    using KT = typename std::remove_cv<typename std::remove_pointer<decltype(kptr(0))>::type>::type;
    constexpr int NV = sizeof(KT) == 4 ? 4 : 2;   // 16-byte vectors per lane and tensor (16 dims)
    const int lane = threadIdx.x & 31, sub = lane >> 2, l4 = lane & 3;
    float q[16];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float4 t = *reinterpret_cast<const float4*>(q_smem + l4 * 16 + c * 4);
        q[c * 4] = t.x; q[c * 4 + 1] = t.y; q[c * 4 + 2] = t.z; q[c * 4 + 3] = t.w;
    }
    A.m = -INFINITY;
    A.l = 0.0f;
#pragma unroll
    for (int c = 0; c < 16; ++c) A.o[c] = 0.0f;
    const int span = stride * 8;
    const int n_it = n_keys > first ? (n_keys - first + span - 1) / span : 0;
    auto issue = [&](int it) {
        const int j = first + (it * 8 + sub) * stride;
        if (it < n_it && j < n_keys) {
            uint4* dst = ring + (it % NSTG) * (2 * NV * 32) + lane;   // vector c of this lane at [c][lane]: conflict-free
            const int blk = swz >= 0 ? (l4 ^ (((swz + j) & 1) * (NV == 4 ? 1 : 2))) : l4;
            const uint4* kp = reinterpret_cast<const uint4*>(kptr(j)) + blk * NV;
            const uint4* vp = reinterpret_cast<const uint4*>(vptr(j)) + blk * NV;
#pragma unroll
            for (int c = 0; c < NV; ++c) {
                cp_async16(dst + c * 32, kp + c);
                cp_async16(dst + (NV + c) * 32, vp + c);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");   // always: keeps the group count uniform
    };
#pragma unroll
    for (int s = 0; s < NSTG - 1; ++s) issue(s);
#pragma unroll 1
    for (int it = 0; it < n_it; ++it) {
        issue(it + NSTG - 1);
        asm volatile("cp.async.wait_group %0;" ::"n"(NSTG - 1) : "memory");
        const int j = first + (it * 8 + sub) * stride;
        if (j < n_keys) {
            const uint4* src = ring + (it % NSTG) * (2 * NV * 32) + lane;
            float kf[16], vf[16];
            if constexpr (sizeof(KT) == 4) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint4 kk = src[c * 32], vv = src[(4 + c) * 32];
                    kf[c * 4] = __uint_as_float(kk.x); kf[c * 4 + 1] = __uint_as_float(kk.y); kf[c * 4 + 2] = __uint_as_float(kk.z); kf[c * 4 + 3] = __uint_as_float(kk.w);
                    vf[c * 4] = __uint_as_float(vv.x); vf[c * 4 + 1] = __uint_as_float(vv.y); vf[c * 4 + 2] = __uint_as_float(vv.z); vf[c * 4 + 3] = __uint_as_float(vv.w);
                }
            } else {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float w[8];
                    cvt8(src[c * 32], w);
#pragma unroll
                    for (int e = 0; e < 8; ++e) kf[c * 8 + e] = w[e];
                    cvt8(src[(2 + c) * 32], w);
#pragma unroll
                    for (int e = 0; e < 8; ++e) vf[c * 8 + e] = w[e];
                }
            }
            float s = 0.0f;
#pragma unroll
            for (int c = 0; c < 16; ++c) s = fmaf(q[c], kf[c], s);
            s += __shfl_xor_sync(0xfu << (lane & 28), s, 1);
            s += __shfl_xor_sync(0xfu << (lane & 28), s, 2);
            const float mn = fmaxf(A.m, s);
            const float corr = expf(A.m - mn);
            const float e = expf(s - mn);
            A.l = A.l * corr + e;
            A.m = mn;
#pragma unroll
            for (int c = 0; c < 16; ++c) A.o[c] = fmaf(e, vf[c], A.o[c] * corr);
        }
    }
    cp_async_wait_all();
    __syncwarp();
    attn_merge_subs(A);
}

// Bulk-copy variant for the head-major cross K/V layout (encoder.cu ckv_relayout_kernel): the unit's keys are ONE contiguous
// [n_keys][128] block, so a batch of keys (K and V rows) is a single cp.async.bulk (TMA engine, no tensor map) into this warp's
// ring, completion on the stage's mbarrier; NSTG-1 batches are in flight per warp.  A batch is 4 KB whatever the element type:
// 8 keys of fp32 or 16 keys of fp16 -- with 8-key (2 KB) fp16 batches the fp16 cache streamed at HALF the bytes per second of the
// fp32 one (decoder5.cu stage trace: 13.6 us vs 16.2 us for half the bytes): the stage is paced by batches, not by bytes.
// The warps of the unit take batches round-robin (wslot of nwarps).  Lane (sub, l4) handles key `sub` (and `sub + 8` of a 16-key
// batch: two independent score chains, one rescale of the running state) and the 16-byte chunks l4 + 4c of its K and V rows --
// with the layout's XOR-4 swizzle on odd positions the 8 lanes of a quarter warp hit 8 distinct bank groups.
// ring_count: batches this warp has pushed through its ring since kernel start (stage / parity bookkeeping).
template <typename KT>
__device__ __forceinline__ int attn_bulk_dim(int l4, int i) {   // which of the 64 head dims is o[i] / q[i] of lane l4
    constexpr int CE = 16 / (int)sizeof(KT);                    // elements per 16-byte chunk
    return (l4 + 4 * (i / CE)) * CE + i % CE;
}
template <typename KT>
struct AttnBulkGeom {
    static constexpr int ROWB = 128 * (int)sizeof(KT);   // bytes of one key: K row | V row of this head
    static constexpr int STGB = 4096;                    // bytes per batch / ring stage
    static constexpr int KPB = STGB / ROWB;              // keys per batch: 8 (fp32) or 16 (fp16)
};
// Batch bb of the unit's keys, the cnt-th batch through this warp's ring: its bytes expected on the stage's mbarrier and one bulk
// copy into the stage.  L2H: the copy carries the L2 policy l2pol (l2_policy_*).  Called by one lane.
template <int NSTG, typename KT, bool L2H>
__device__ __forceinline__ void attn_bulk_issue(const KT* base, int n_keys, int bb, unsigned int cnt, unsigned char* ring, uint64_t* mbar,
                                                uint64_t l2pol) {
    constexpr int ROWB = AttnBulkGeom<KT>::ROWB, STGB = AttnBulkGeom<KT>::STGB, KPB = AttnBulkGeom<KT>::KPB;
    const int slot = (int)(cnt % NSTG);
    const uint32_t bytes = (uint32_t)min(KPB, n_keys - bb * KPB) * ROWB;
    mbar_expect_tx(mbar + slot, bytes);
    if constexpr (L2H) bulk_g2s_l2(ring + slot * STGB, base + (int64_t)bb * KPB * 128, bytes, mbar + slot, l2pol);
    else bulk_g2s(ring + slot * STGB, base + (int64_t)bb * KPB * 128, bytes, mbar + slot);
}
// The first NSTG-1 batches of attn_warp_bulk, issued ahead of time (the K/V rows are static: nothing to wait for); the
// matching attn_warp_bulk call passes prefilled = true and the SAME base / n_keys / wslot / nwarps / ring_count.
template <int NSTG, typename KT, bool L2H = false>
__device__ __forceinline__ void attn_bulk_prefill(const KT* base, int n_keys, int wslot, int nwarps, unsigned char* ring, uint64_t* mbar,
                                                  unsigned int ring_count, uint64_t l2pol = 0) {
    constexpr int KPB = AttnBulkGeom<KT>::KPB;
    if ((threadIdx.x & 31) != 0) return;
    const int n_batches = (n_keys + KPB - 1) / KPB;
    const int n_it = n_batches > wslot ? (n_batches - wslot + nwarps - 1) / nwarps : 0;
#pragma unroll
    for (int it = 0; it < NSTG - 1; ++it)
        if (it < n_it) attn_bulk_issue<NSTG, KT, L2H>(base, n_keys, wslot + it * nwarps, ring_count + (unsigned int)it, ring, mbar, l2pol);
}
template <int NSTG, typename KT, bool L2H = false>
__device__ __forceinline__ void attn_warp_bulk(const float* q_smem, const KT* base, int n_keys, int wslot, int nwarps, int swz,
                                               unsigned char* ring, uint64_t* mbar, unsigned int& ring_count, AttnAcc& A,
                                               bool prefilled = false, uint64_t l2pol = 0) {
    constexpr int CE = 16 / (int)sizeof(KT), NC = 16 / CE;      // chunk elements; chunks per lane and tensor
    constexpr int ROWB = AttnBulkGeom<KT>::ROWB, STGB = AttnBulkGeom<KT>::STGB, KPB = AttnBulkGeom<KT>::KPB;
    const int lane = threadIdx.x & 31, sub = lane >> 2, l4 = lane & 3;
    float q[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) q[i] = q_smem[attn_bulk_dim<KT>(l4, i)];
    A.m = -INFINITY;
    A.l = 0.0f;
#pragma unroll
    for (int c = 0; c < 16; ++c) A.o[c] = 0.0f;
    const int n_batches = (n_keys + KPB - 1) / KPB;
    const int n_it = n_batches > wslot ? (n_batches - wslot + nwarps - 1) / nwarps : 0;
    auto issue = [&](int it) {
        if (it < n_it && lane == 0) attn_bulk_issue<NSTG, KT, L2H>(base, n_keys, wslot + it * nwarps, ring_count + (unsigned int)it, ring, mbar, l2pol);
    };
    auto load16 = [&](const unsigned char* p16, int par, float (&f)[16]) {   // this lane's 16 dims of one K or V row
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int phys = (l4 + 4 * c) ^ (4 * par);
            const uint4 u = *reinterpret_cast<const uint4*>(p16 + phys * 16);
            if constexpr (sizeof(KT) == 4) {
                f[c * 4] = __uint_as_float(u.x); f[c * 4 + 1] = __uint_as_float(u.y); f[c * 4 + 2] = __uint_as_float(u.z); f[c * 4 + 3] = __uint_as_float(u.w);
            } else {
                float w[8];
                cvt8(u, w);
#pragma unroll
                for (int e = 0; e < 8; ++e) f[c * 8 + e] = w[e];
            }
        }
    };
    if (!prefilled) {
#pragma unroll
        for (int s = 0; s < NSTG - 1; ++s) issue(s);
    }
    const unsigned qmask = 0xfu << (lane & 28);
#pragma unroll 1
    for (int it = 0; it < n_it; ++it) {
        __syncwarp();                 // every lane is done with the slot that is refilled now (consumed one iteration ago)
        issue(it + NSTG - 1);
        const unsigned int cnt = ring_count + (unsigned int)it;
        const int slot = (int)(cnt % NSTG);
        mbar_wait(mbar + slot, (cnt / NSTG) & 1);
        const int bb = wslot + it * nwarps;
        const int j0 = bb * KPB + sub;
        if (j0 < n_keys) {
            const unsigned char* row0 = ring + slot * STGB + sub * ROWB;
            const int par0 = (swz + j0) & 1;
            if constexpr (KPB == 8) {
                float kf[16], vf[16];
                load16(row0, par0, kf);
                load16(row0 + ROWB / 2, par0, vf);
                float s = 0.0f;
#pragma unroll
                for (int c = 0; c < 16; ++c) s = fmaf(q[c], kf[c], s);
                s += __shfl_xor_sync(qmask, s, 1);
                s += __shfl_xor_sync(qmask, s, 2);
                const float mn = fmaxf(A.m, s);
                const float corr = expf(A.m - mn);
                const float e = expf(s - mn);
                A.l = A.l * corr + e;
                A.m = mn;
#pragma unroll
                for (int c = 0; c < 16; ++c) A.o[c] = fmaf(e, vf[c], A.o[c] * corr);
            } else {
                // keys sub and sub + 8 of the batch: two score chains, one rescale
                const int j1 = j0 + 8;
                const bool v1 = j1 < n_keys;
                const unsigned char* row1 = row0 + 8 * ROWB;
                const int par1 = (swz + j1) & 1;
                float s0, s1 = -INFINITY;
                {
                    float k0[16], k1[16];
                    load16(row0, par0, k0);
                    if (v1) load16(row1, par1, k1);
                    float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
                    for (int c = 0; c < 16; ++c) a0 = fmaf(q[c], k0[c], a0);
                    s0 = a0;
                    if (v1) {
#pragma unroll
                        for (int c = 0; c < 16; ++c) a1 = fmaf(q[c], k1[c], a1);
                        s1 = a1;
                    }
                }
                s0 += __shfl_xor_sync(qmask, s0, 1);
                s0 += __shfl_xor_sync(qmask, s0, 2);
                if (v1) {   // uniform over the four lanes of a key
                    s1 += __shfl_xor_sync(qmask, s1, 1);
                    s1 += __shfl_xor_sync(qmask, s1, 2);
                }
                const float mn = fmaxf(A.m, fmaxf(s0, s1));
                const float corr = expf(A.m - mn);
                const float e0 = expf(s0 - mn), e1 = expf(s1 - mn);   // s1 = -inf without a second key: e1 = 0
                A.l = A.l * corr + (e0 + e1);
                A.m = mn;
                asm volatile("" ::: "memory");   // keep the V loads behind the scores (register pressure)
                float vv[16];
                load16(row0 + ROWB / 2, par0, vv);
#pragma unroll
                for (int c = 0; c < 16; ++c) A.o[c] = fmaf(e0, vv[c], A.o[c] * corr);
                if (v1) {
                    load16(row1 + ROWB / 2, par1, vv);
#pragma unroll
                    for (int c = 0; c < 16; ++c) A.o[c] = fmaf(e1, vv[c], A.o[c]);
                }
            }
        }
    }
    ring_count += (unsigned int)n_it;
    __syncwarp();
    attn_merge_subs(A);   // same l4 = same dims
}

// block-level merge of the 8 warps' partial attention results; out[64] / ML valid after the trailing __syncthreads()
__device__ __forceinline__ void attn_cta_tail(const AttnAcc& A, float* wm, float* wl, float* wo, float* out, float* ML) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (lane < 4) {
#pragma unroll
        for (int c = 0; c < 16; ++c) wo[warp * 64 + lane * 16 + c] = A.o[c];
    }
    if (lane == 0) { wm[warp] = A.m; wl[warp] = A.l; }
    __syncthreads();
    if (tid < 64) {
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < NW; ++w) M = fmaxf(M, wm[w]);
        float L = 0.0f, o = 0.0f;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
            const float m = wm[w];
            const float sc = m > -INFINITY ? expf(m - M) : 0.0f;
            L += sc * wl[w];
            o += sc * wo[w * 64 + tid];
        }
        out[tid] = o;
        if (tid == 0) { ML[0] = M; ML[1] = L; }
    }
    __syncthreads();
}

// one (query row, head) unit handled by the 8 warps of a CTA (keys strided over warps); returns the merged
// (M, L) and the unnormalised output in out[64] (shared memory), valid after the trailing __syncthreads().
template <typename KF, typename VF>
__device__ __forceinline__ void attn_cta(const float* q_smem, int n_keys, KF&& kptr, VF&& vptr, float* wm, float* wl,
                                         float* wo, float* out, float* ML, int swz = -1) {
    const int warp = threadIdx.x >> 5;
    AttnAcc A;
    attn_warp(q_smem, n_keys, warp, NW, kptr, vptr, A, swz);
    attn_cta_tail(A, wm, wl, wo, out, ML);
}

// ---- activation planes of the mma.sync products (fp16 hi/lo split of prims.cuh; see decoder5.cu) -------------
// Fragment-order planes: element (row, col) of an activation matrix [rows][K] lives in the uint4
//   ((row / 8) * (K / 32) + col / 32) * 32 + (row % 8) * 4 + (col % 32) / 8,   half (col % 8)
// i.e. lane (g = row % 8, t) of the MMA finds the 8 halves x[row][chunk*32 + t*8 .. +8) in ONE 16-byte word.
__device__ __forceinline__ int plane_idx(int nchunks, int row, int col) {
    return ((row >> 3) * nchunks + (col >> 5)) * 32 + (row & 7) * 4 + ((col & 31) >> 3);
}
__device__ __forceinline__ void store_frag(uint4* xhi, uint4* xlo, int nchunks, int row, int col, const float4 v) {
    uint2 hi, lo;
    hl_split4(v, hi, lo);
    const int idx = plane_idx(nchunks, row, col), half = (col & 7) >> 2;
    reinterpret_cast<uint2*>(xhi + idx)[half] = hi;
    reinterpret_cast<uint2*>(xlo + idx)[half] = lo;
}

// ---- top candidates --------------------------------------------------------------------------------------
// The ranking of vocabulary candidates, the only place it is written (DESIGN.md section 2): the higher value first, the
// lower id on equal values.  An empty candidate is (-inf, INT_MAX).
__device__ __forceinline__ bool cand_better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

// one xor-shuffle step of a warp arg-max: (bv, bi) becomes the better of this lane's and lane ^ off's
__device__ __forceinline__ void cand_xor(float& bv, int& bi, int off) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (cand_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
}
// arg-max over the warp: every lane ends with the warp's best (bv, bi)
__device__ __forceinline__ void warp_best(float& bv, int& bi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cand_xor(bv, bi, o);
}

template <int KC>
struct Cand {
    float v[KC];
    int i[KC];
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int k = 0; k < KC; ++k) { v[k] = -INFINITY; i[k] = INT_MAX; }
    }
    __device__ __forceinline__ void push(float val, int idx) {   // keep the KC best
        if (!cand_better(val, idx, v[KC - 1], i[KC - 1])) return;
        v[KC - 1] = val;
        i[KC - 1] = idx;
#pragma unroll
        for (int k = KC - 1; k > 0; --k) {
            if (cand_better(v[k], i[k], v[k - 1], i[k - 1])) {
                const float tv = v[k]; v[k] = v[k - 1]; v[k - 1] = tv;
                const int ti = i[k]; i[k] = i[k - 1]; i[k - 1] = ti;
            }
        }
    }
};

// The same list in shared memory, DEC_KC entries sorted best first; false when (v, n) stays out
__device__ __forceinline__ bool cand_insert(float* lv, int* li, float v, int n) {
    if (!cand_better(v, n, lv[DEC_KC - 1], li[DEC_KC - 1])) return false;
    int k = DEC_KC - 1;
    for (; k > 0 && cand_better(v, n, lv[k - 1], li[k - 1]); --k) { lv[k] = lv[k - 1]; li[k] = li[k - 1]; }
    lv[k] = v;
    li[k] = n;
    return true;
}

// ---- softmax state: running max m and sum of exp(v - m) -----------------------------------------------
// one more finite value v
__device__ __forceinline__ void softmax_add(float& m, float& s, float v) {
    if (v > m) { s = s * expf(m - v) + 1.0f; m = v; }
    else s += expf(v - m);
}
// the state (m2, s2) of other values; an empty state has m = -inf
__device__ __forceinline__ void softmax_merge(float& m, float& s, float m2, float s2) {
    const float mn = fmaxf(m, m2);
    s = (m > -INFINITY ? s * expf(m - mn) : 0.0f) + (m2 > -INFINITY ? s2 * expf(m2 - mn) : 0.0f);
    m = mn;
}

// ---- one record per (CTA, row) --------------------------------------------------------------------------
// The vocabulary stage leaves, per (CTA or slice c, row r), a record at o = c * R + r: lg_m / lg_s (max, sum-exp) and the
// best candidates, lg_v / lg_i[o] for a top-1 record, lg_v / lg_i[o * KC + k] for a KC list.
// (max, sum-exp) of n per-warp records rec[w * ld] = {max, sum-exp, ...}, folded in record order
__device__ __forceinline__ float2 fold_softmax(const float* rec, int n, int ld) {
    float M = -INFINITY;
    for (int w = 0; w < n; ++w) M = fmaxf(M, rec[w * ld]);
    float S = 0.0f;
    for (int w = 0; w < n; ++w)
        if (rec[w * ld] > -INFINITY) S += rec[w * ld + 1] * expf(rec[w * ld] - M);
    return make_float2(M, S);
}
// the top-1 record o from n per-warp records rec[w * ld] = {max, sum-exp, best value, best id as float bits}
__device__ __forceinline__ void fold_records_top1(const DecArgs& a, const float* rec, int n, int ld, int64_t o) {
    const float2 ms = fold_softmax(rec, n, ld);
    float bv = -INFINITY;
    int bi = INT_MAX;
    for (int w = 0; w < n; ++w) {
        const int ci = __float_as_int(rec[w * ld + 3]);
        if (cand_better(rec[w * ld + 2], ci, bv, bi)) { bv = rec[w * ld + 2]; bi = ci; }
    }
    a.lg_m[o] = ms.x;
    a.lg_s[o] = ms.y;
    a.lg_v[o] = bv;
    a.lg_i[o] = bi;
}
// the KC-list record o from n per-warp records rec[w * ld] = {max, sum-exp, KC values, KC ids as float bits}, sorted
// lists of which the first nk entries can matter
template <int KC>
__device__ __forceinline__ void fold_records(const DecArgs& a, const float* rec, int n, int ld, int nk, int64_t o) {
    const float2 ms = fold_softmax(rec, n, ld);
    Cand<KC> best;
    best.init();
    for (int w = 0; w < n; ++w)
        for (int k = 0; k < nk; ++k) best.push(rec[w * ld + 2 + k], __float_as_int(rec[w * ld + 2 + KC + k]));
    a.lg_m[o] = ms.x;
    a.lg_s[o] = ms.y;
#pragma unroll
    for (int k = 0; k < KC; ++k) { a.lg_v[o * KC + k] = best.v[k]; a.lg_i[o * KC + k] = best.i[k]; }
}

// whether the vocabulary stage at position p masks the special ids (DecArgs::mask_mode): position p produces token p + 1,
// and the beam search masks them while the sequence has at most 5 tokens (transcribe.rs:271-275).  A macro: the same
// expression behind a __forceinline__ function compiles to different predicate code in every decoder.
#define SPECIAL_MASKED(a, p) \
    ((a).is_special != nullptr && ((a).mask_mode == MASK_ALWAYS || ((a).mask_mode == MASK_SHORT && (p) + 1 <= 5)))

// ---- per-row finish: log-probs (v - max) - lse of the candidates, lse from the NP records of the row (DESIGN.md section 2)
// greedy bookkeeping of row r at position p (beam.rs:9-37 with beam_size 1): the token and its rounded log-prob lp, the
// length, EOT.  A row whose position p + 1 is still inside its prompt commits nothing (its token is in the buffer, its
// log-prob 0); a row is finished by EOT or once it holds prompt_len + max_depth ids.
// the most ids row r may hold, its prompt length + max_depth (DecArgs::lengths): a greedy row is finished when it holds them;
// a beam window's search starts at position id_limit(slot 0) - max_depth - 1
__device__ __forceinline__ int id_limit(const DecArgs& a, int r) { return __ldg(a.lengths + a.Rmax + r); }
__device__ __forceinline__ void greedy_commit(const DecArgs& a, int r, int p, int id, float lp) {
    // lengths[r] holds the prompt length until the first commit, then p + 2 < p' + 2: the test passes from then on.  The
    // limit is read at its use (an L1 hit) rather than held: the finishers run at the decoders' register limit
    if (!a.greedy || __ldcg(a.finished + r) || p + 1 < __ldcg(a.lengths + r)) return;
    a.tokens[(int64_t)r * a.t_max + p + 1] = id;
    a.token_lp[(int64_t)r * a.t_max + p + 1] = lp;
    a.lengths[r] = p + 2;
    if (id == a.eot || p + 2 >= id_limit(a, r)) a.finished[r] = 1;
}
// The greedy loop's rules (DecArgs::loop_rules, host/loop_rules.hpp) for row r after greedy_commit put `id` at p + 1: the EOT
// test on the raw logits of `id` (`top`) and of EOT, then the repetition cut over tokens[0, p + 2), lane l taking windows
// i = l (mod 32).  Only for a row that was open before the commit.  The EOT test only finishes the row: the host appends the
// EOT that follows (Session::greedy_decode).  The cut writes EOT at `end`, with a NaN log-prob (no step chose it), and
// finishes the row.  Called by a whole warp.
__device__ __forceinline__ void loop_finish(const DecArgs& a, int r, int p, int id, float top) {
    if (id == a.eot) return;   // finished by greedy_commit; the EOT test holds and appends nothing
    const int lane = threadIdx.x & 31;
    if (loop::eot_stop(__ldcg(a.eot_logit + r), top)) {
        if (lane == 0) a.finished[r] = 1;
        return;
    }
    int* row = a.tokens + (int64_t)r * a.t_max;
    const int n = p + 2;
    auto tok = [&](int j) { return j == p + 1 ? id : __ldcg(row + j); };
    const int end = loop::repeat_cut(n, [&](int base) {
        const int i = base + lane;
        return __ballot_sync(0xffffffffu, i + 2 * loop::REPEAT_WINDOW <= n && loop::window_repeats(tok, n, i));
    });
    if (end >= 0 && lane == 0) {
        row[end] = a.eot;
        a.token_lp[(int64_t)r * a.t_max + end] = __int_as_float(0x7fffffff);
        a.lengths[r] = end + 1;
        a.finished[r] = 1;
    }
}
// rows whose search is still open: every row, or in a greedy search those that have not produced EOT
__device__ __forceinline__ int rows_open(const DecArgs& a) {
    int live = 0;
    for (int r = 0; r < a.R; ++r) live += (a.greedy && __ldcg(a.finished + r)) ? 0 : 1;
    return live;
}
// where a launch stopped: the next position, the searches still open and the steps run (written by one thread)
__device__ __forceinline__ void decode_done(const DecArgs& a, int pos, int n_open, int steps) {
    *a.pos = pos;
    *a.n_unfinished = n_open;
    *a.steps_done = steps;
}

// Warp per row: the max and lse of the row's NP <= 32 * NPL records, record lane + 32 k in rm[k] / rs[k] of this lane
template <int NPL>
__device__ __forceinline__ float row_lse(const float (&rm)[NPL], const float (&rs)[NPL], int NP, float& mx) {
    const int lane = threadIdx.x & 31;
    mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < NPL; ++k)
        if (lane + 32 * k < NP) mx = fmaxf(mx, rm[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float se = 0.0f;
#pragma unroll
    for (int k = 0; k < NPL; ++k)
        if (lane + 32 * k < NP && rm[k] > -INFINITY) se += rs[k] * expf(rm[k] - mx);
    return logf(warp_sum(se));
}
// Warp per row, k = 1: the best candidate of row r from its NP <= 32 * NPL top-1 records, all loads issued before any use
// (one L2 round trip) -> topk_id / topk_lp [r], then the greedy bookkeeping
template <int NPL>
__device__ __forceinline__ void finish_row_top1(const DecArgs& a, int r, int p, int NP) {
    const int lane = threadIdx.x & 31, R = a.R;
    float rm[NPL], rs[NPL], rv[NPL];
    int ri[NPL];
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
        const int64_t o = (int64_t)min(lane + 32 * k, NP - 1) * R + r;
        rm[k] = __ldcg(a.lg_m + o);
        rs[k] = __ldcg(a.lg_s + o);
        rv[k] = __ldcg(a.lg_v + o);
        ri[k] = __ldcg(a.lg_i + o);
    }
    const bool loop_open = a.loop_rules && !__ldcg(a.finished + r);   // read before the commit below
    float mx;
    const float lse = row_lse<NPL>(rm, rs, NP, mx);
    float bv = -INFINITY;
    int bi = INT_MAX;
#pragma unroll
    for (int k = 0; k < NPL; ++k)
        if (lane + 32 * k < NP && ri[k] != INT_MAX && cand_better(rv[k], ri[k], bv, bi)) { bv = rv[k]; bi = ri[k]; }
    warp_best(bv, bi);
    if (lane == 0) {
        a.topk_id[r] = bi == INT_MAX ? -1 : bi;
        const float lp = __fsub_rn(__fsub_rn(bv, mx), lse);
        a.topk_lp[r] = lp;
        greedy_commit(a, r, p, bi, lp);
    }
    if (loop_open) loop_finish(a, r, p, bi, bv);   // bv: the raw logit of bi (no mask in loop mode)
}
// CTA per row, the k best candidates of row r from its NP KC-list records -> topk_id / topk_lp [r][k]; candidate 0 goes
// to the greedy bookkeeping.  s_f / s_i: NW floats / ints of shared scratch.  Called by the whole CTA.
template <int KC>
__device__ __forceinline__ void finish_row_topk(const DecArgs& a, int r, int p, int NP, float* s_f, int* s_i) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, R = a.R;
    const bool loop_open = a.loop_rules && !__ldcg(a.finished + r);   // read before the commit below
    int id0 = -1;
    float mx = -INFINITY;
    for (int c = tid; c < NP; c += NT) mx = fmaxf(mx, __ldcg(a.lg_m + (int64_t)c * R + r));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_f[warp] = mx;
    __syncthreads();
    mx = s_f[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) mx = fmaxf(mx, s_f[w]);
    __syncthreads();
    float se = 0.0f;
    for (int c = tid; c < NP; c += NT) {
        const float m = __ldcg(a.lg_m + (int64_t)c * R + r);
        if (m > -INFINITY) se += __ldcg(a.lg_s + (int64_t)c * R + r) * expf(m - mx);
    }
    se = warp_sum(se);
    if (lane == 0) s_f[warp] = se;
    __syncthreads();
    se = 0.0f;
#pragma unroll
    for (int w = 0; w < NW; ++w) se += s_f[w];
    const float lse = logf(se);
    __syncthreads();
    float prev_v = INFINITY;
    int prev_i = -1;
    for (int kk = 0; kk < a.k; ++kk) {   // the best candidate ranked after the previous one
        float bv = -INFINITY;
        int bi = INT_MAX;
        for (int c = tid; c < NP * KC; c += NT) {
            const int part = c / KC, k = c % KC;
            const int idx = __ldcg(a.lg_i + ((int64_t)part * R + r) * KC + k);
            if (idx == INT_MAX) continue;
            const float v = __fsub_rn(__fsub_rn(__ldcg(a.lg_v + ((int64_t)part * R + r) * KC + k), mx), lse);
            if (cand_better(prev_v, prev_i, v, idx) && cand_better(v, idx, bv, bi)) { bv = v; bi = idx; }
        }
        warp_best(bv, bi);
        if (lane == 0) { s_f[warp] = bv; s_i[warp] = bi; }
        __syncthreads();
        bv = s_f[0];
        bi = s_i[0];
#pragma unroll
        for (int w = 1; w < NW; ++w)
            if (cand_better(s_f[w], s_i[w], bv, bi)) { bv = s_f[w]; bi = s_i[w]; }
        __syncthreads();
        if (tid == 0) {
            a.topk_id[(int64_t)r * a.k + kk] = bi == INT_MAX ? -1 : bi;
            a.topk_lp[(int64_t)r * a.k + kk] = bv;
            if (kk == 0) greedy_commit(a, r, p, bi, bv);
        }
        if (kk == 0) id0 = bi;
        prev_v = bv;
        prev_i = bi;
    }
    // the raw logit of candidate 0 is the row's max mx: the records' maxima run over the same values as their candidates
    if (loop_open && warp == 0) loop_finish(a, r, p, id0, mx);
}

// ---- ticket finish (decoder4, decoder6): every CTA takes a ticket after publishing its records; the CTA that takes the last
// ticket of round n finishes the step and releases the flag the others wait on.  bar[1]: tickets, bar[2]: flag (the
// rounds released so far); both zeroed by the host before the launch.  Called by one thread.
__device__ __forceinline__ bool last_ticket(unsigned int* bar, unsigned int n) {
    __threadfence();
    return atomicAdd(bar + 1, 1u) == n * gridDim.x - 1;
}
__device__ __forceinline__ void release_flag(unsigned int* bar, unsigned int gen) {
    __threadfence();
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(bar + 2), "r"(gen) : "memory");
}
// watchdog: SM clocks the wait may last before the kernel traps (fail loudly instead of hanging the GPU)
__device__ __forceinline__ void wait_flag(const unsigned int* bar, unsigned int gen, long long watchdog) {
    const long long t0 = clock64();
    while (ld_acquire(bar + 2) < gen)
        if (clock64() - t0 > watchdog) __trap();
}


}  // namespace

}  // namespace wb
