// PTX primitives of the tensor-core and async-copy kernels, each defined once: shared-memory addresses, mbarriers,
// asynchronous copies, the m16n8k16 MMA, the erf GELU, the LayerNorm arithmetic and the fp16 hi/lo split of fp32 activations.
// Internal; everything lives in an anonymous namespace of the including TU.
#pragma once
#include <cstdint>
#include <cuda_fp16.h>

namespace wb {

namespace {

// ---- shared memory and mbarriers ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
// after the mbar_init calls: the barriers are visible to the async proxy and to the other CTAs of the cluster
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
// true once the phase of the mbarrier at shared address addr with this parity has completed
__device__ __forceinline__ bool mbar_try_wait(uint32_t addr, uint32_t parity) {
    uint32_t done;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    return done != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    while (!mbar_try_wait(addr, parity)) {
    }
}
// the same wait, trapping after `clocks` SM clocks (fail loudly instead of hanging the GPU)
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity, long long clocks) {
    const uint32_t addr = smem_u32(bar);
    const long long t0 = clock64();
    while (!mbar_try_wait(addr, parity))
        if (clock64() - t0 > clocks) __trap();
}

// ---- asynchronous copies -----------------------------------------------------------------------------
// 16-byte cp.async global -> shared (L2 only); completion with cp_async_wait_all() or cp.async.wait_group
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// the same with an L2 policy (l2_policy_* in dec_common.cuh)
__device__ __forceinline__ void cp_async16_l2(void* dst, const void* src, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// 1-D bulk copy global -> shared (TMA engine, no tensor map), completion counted on an mbarrier of this CTA
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
// the same with an L2 policy
__device__ __forceinline__ void bulk_g2s_l2(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
                 : "memory");
}
// shared address addr of this CTA -> the same location in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
// orders this thread's generic-proxy shared-memory accesses before the async-proxy ones (bulk copies, wgmma) that follow
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- math ----------------------------------------------------------------------------------------------
// D[16 x 8] += A[16 x 16] * B[16 x 8], fp16 operands, fp32 accumulate
__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// burn activation::gelu (erf form): x * (erf(x / sqrt2) + 1) / 2, evaluated in that order
__device__ __forceinline__ float gelu_erf(float x) {
    const float t = __fadd_rn(erff(__fdiv_rn(x, 1.41421356237309504880f)), 1.0f);
    return __fdiv_rn(__fmul_rn(x, t), 2.0f);
}

// ---- LayerNorm arithmetic ------------------------------------------------------------------------------
// burn 0.9 nn::LayerNorm (layer_norm in oracle/model.py): mean, biased variance of dv = x - mean, then dv / den * gamma + beta,
// every op rounded on its own as the reference issues them as separate tensor ops (no FMA contraction).  Each kernel keeps its
// own loads, reduction order and row mapping; only the arithmetic below is shared.
// LN_DEN: burn 0.9 divides by sqrt(var) + eps (eps_outside, the default); later burn by sqrt(var + eps).  A macro, so that
// eps is read after the eps_outside test, inside the branch, as the kernels always have: an inline function reads it ahead,
// which reschedules decoder5's LayerNorm stage.
#define LN_DEN(var, eps, eps_outside) ((eps_outside) ? __fadd_rn(__fsqrt_rn(var), (eps)) : __fsqrt_rn(__fadd_rn((var), (eps))))
// the centred square sum: q += dv * dv; the float4 form adds x, y, z, w in that order
__device__ __forceinline__ float ln_sq_add(float q, float dv) { return __fadd_rn(q, __fmul_rn(dv, dv)); }
__device__ __forceinline__ float ln_sq_add4(float q, const float4 dv) {
    q = ln_sq_add(q, dv.x); q = ln_sq_add(q, dv.y);
    q = ln_sq_add(q, dv.z); return ln_sq_add(q, dv.w);
}
// the normalisation dv / den * gamma + beta.  The scalar form reads g[c] and b[c] itself, after the divide, where the kernels
// have always read them (gamma and beta passed in by value are loaded, and scheduled, ahead of it); LDG reads them through the
// read-only data cache (__ldg: global memory only).  The float4 form takes the vectors every caller loads ahead of it.
template <bool LDG = false>
__device__ __forceinline__ float ln_norm(float dv, float den, const float* g, const float* b, int c) {
    return __fadd_rn(__fmul_rn(__fdiv_rn(dv, den), LDG ? __ldg(g + c) : g[c]), LDG ? __ldg(b + c) : b[c]);
}
__device__ __forceinline__ float4 ln_norm4(const float4 dv, float den, const float4 g, const float4 b) {
    float4 o;
    o.x = __fadd_rn(__fmul_rn(__fdiv_rn(dv.x, den), g.x), b.x);
    o.y = __fadd_rn(__fmul_rn(__fdiv_rn(dv.y, den), g.y), b.y);
    o.z = __fadd_rn(__fmul_rn(__fdiv_rn(dv.z, den), g.z), b.z);
    o.w = __fadd_rn(__fmul_rn(__fdiv_rn(dv.w, den), g.w), b.w);
    return o;
}
// decoder4's LayerNorm (ln_warp) is the one exception to the separate roundings above, for the headline decoder's speed: the
// square sum contracts into fmaf, and the normalisation multiplies by rinv = 1 / den (<= 1.5 ulp from the divide) and
// contracts the beta add, fmaf(dv * rinv, g, b).  The eps placement (LN_DEN) is the same.
__device__ __forceinline__ float ln_sq_fma4(float q, const float4 dv) {
    q = fmaf(dv.x, dv.x, q); q = fmaf(dv.y, dv.y, q);
    q = fmaf(dv.z, dv.z, q); return fmaf(dv.w, dv.w, q);
}
__device__ __forceinline__ float4 ln_norm4_rcp(const float4 dv, float rinv, const float4 g, const float4 b) {
    return make_float4(fmaf(__fmul_rn(dv.x, rinv), g.x, b.x), fmaf(__fmul_rn(dv.y, rinv), g.y, b.y),
                       fmaf(__fmul_rn(dv.z, rinv), g.z, b.z), fmaf(__fmul_rn(dv.w, rinv), g.w, b.w));
}

// ---- fp16 hi/lo split of fp32 activations -------------------------------------------------------------
// The reference computes in f32, so one fp16 pass is not accurate enough for the tensor cores.  Every weight of a released
// Whisper checkpoint is fp16-representable, so the weights are EXACT in fp16; an fp32 activation x travels as a PAIR of fp16
// values
//     x = hi + lo / HL_SCALE,   hi = fp16(x),   lo = fp16((x - hi) * HL_SCALE)
// (22 mantissa bits; the scaling keeps lo normal).  Every product hi * w, lo * w is exact in an fp32 accumulator; the hi and
// lo products accumulate separately and are rejoined by hl_join.  Scalar, pair and quad forms: the packed ones convert two
// values per instruction.
constexpr float HL_SCALE = 2048.0f;
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ void hl_split(float x, __half& hi, __half& lo) {
    const __half h = __float2half_rn(x);
    hi = h;
    lo = __float2half_rn((x - __half2float(h)) * HL_SCALE);
}
__device__ __forceinline__ void hl_split_pair(float x, float y, __half2& hi, __half2& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 f = __half22float2(h);
    hi = h;
    lo = __floats2half2_rn((x - f.x) * HL_SCALE, (y - f.y) * HL_SCALE);
}
__device__ __forceinline__ void hl_split4(const float4 v, uint2& hi, uint2& lo) {
    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    const __half2 l01 = __floats2half2_rn((v.x - f01.x) * HL_SCALE, (v.y - f01.y) * HL_SCALE);
    const __half2 l23 = __floats2half2_rn((v.z - f23.x) * HL_SCALE, (v.w - f23.y) * HL_SCALE);
    hi = make_uint2(h2_bits(h01), h2_bits(h23));
    lo = make_uint2(h2_bits(l01), h2_bits(l23));
}
__device__ __forceinline__ float hl_join(float hi, float lo) { return fmaf(lo, 1.0f / HL_SCALE, hi); }

}  // namespace

}  // namespace wb
