// Tile helpers of the tensor-core attention kernels (enc_attn_tc.cu) and the alignment scores (align.cu): [64][64] fp16 tiles in
// shared memory with XOR-swizzled 16-byte chunks, their ldmatrix loads, the m16n8k16 MMA on fragment arrays and the hi/lo split
// of fp32 pairs into fragment registers.  Internal; everything lives in an anonymous namespace of the including TU.
#pragma once
#include <cuda_fp16.h>

#include "prims.cuh"

namespace wb {

namespace {

constexpr int TQ = 64, TK = 64, HD = 64;
constexpr int TILE_B = 64 * 128;   // one [64][64] fp16 tile = 8 KB (rows of 128 bytes)

__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool ok) {
    const int sz = ok ? 16 : 0;   // zero-fill out-of-range rows
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
// tile [64 rows][64 halves]: 16-byte chunk c of row r sits at r * 128 + ((c ^ (r & 7)) << 4)  (conflict-free ldmatrix)
__device__ __forceinline__ uint32_t tile_off(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }
__device__ __forceinline__ void ldsm4(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr));
}
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr));
}
__device__ __forceinline__ void mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) { mma16816(c, a[0], a[1], a[2], a[3], b0, b1); }
// two fp32 values -> fp16 hi pair and fp16 lo pair, as the A / B fragment registers of an MMA
__device__ __forceinline__ void split2(float x, float y, uint32_t& hi, uint32_t& lo) {
    __half2 h, l;
    hl_split_pair(x, y, h, l);
    hi = h2_bits(h);
    lo = h2_bits(l);
}

}  // namespace

}  // namespace wb
