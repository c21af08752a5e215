// Micro-benchmarks behind the persistent-decoder design choices (decoder5.cu / dec_common.cuh), one CTA per SM, cooperative launch:
//   bar   : latency of grid-barrier variants (with the stores + fence a real stage ends with)
//   stage : barrier + every CTA staging the SAME activation planes (73 KB for small.en, 24 rows) from L2 into shared memory:
//           cp.async in identical order / rotated per CTA / bulk copies (TMA engine) / rotated bulk copies
//   pf    : streaming a 45 / 89 MB block (one layer's cross K/V of 24 small.en windows, fp16 / fp32) cold from HBM vs after a
//           cp.async.bulk.prefetch.L2 issued a dozen barriers earlier (the latency-bound stages that precede cross attention)
// Build: make -C scripts/ubench      Run: scripts/ubench/build/grid_ubench  (prints one line per measurement)
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                                  \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) {                                                               \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                           \
        }                                                                                      \
    } while (0)

constexpr int NT = 256;

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned int ld_acquire(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned int ld_relaxed(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// V0: red.release + ld.acquire polling on the same counter (dec_common.cuh grid_sync)
// V1: red.release + relaxed polling, one acquire fence at the end
// V2: ticket (atom.acq_rel) + flag on another line written by the last arriver; the others poll the flag
// V3: V0 with the counter polled by lane 0 of warp 0 while all OTHER warps skip the leading __syncthreads via a named barrier
//     arrive (bar.arrive) -- only thread 0 waits for them (bar.sync count NT), nobody else blocks twice
// V4: two-level: one CTA per SM arrives on one of 8 group counters (stride 128 B); the last of a group (ticket) arrives on the top
//     counter; everybody polls the top counter
template <int V>
__device__ __forceinline__ void gsync(unsigned int* bar, unsigned int& gen) {
    if (V == 3) {
        if (threadIdx.x < 32) {
            asm volatile("bar.sync 1, %0;" ::"r"(NT) : "memory");
            if (threadIdx.x == 0) {
                ++gen;
                const unsigned int target = gen * gridDim.x;
                asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
                while (ld_acquire(bar) < target) {}
            }
        } else {
            asm volatile("bar.arrive 1, %0;" ::"r"(NT) : "memory");
        }
        __syncthreads();
        return;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        ++gen;
        const unsigned int target = gen * gridDim.x;
        if (V == 0) {
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
            while (ld_acquire(bar) < target) {}
        } else if (V == 1) {
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
            while (ld_relaxed(bar) < target) {}
            asm volatile("fence.acq_rel.gpu;" ::: "memory");
        } else if (V == 2) {
            unsigned int old;
            asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(bar) : "memory");
            if (old == target - 1) {
                asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(bar + 64), "r"(gen) : "memory");
            } else {
                while (ld_acquire(bar + 64) < gen) {}
            }
        } else if (V == 4) {
            const unsigned int grp = blockIdx.x & 7u;
            const unsigned int gsz = (gridDim.x - grp + 7u) / 8u;
            unsigned int old;
            asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(bar + 32 * (1 + grp)) : "memory");
            if (old == gen * gsz - 1) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
            while (ld_acquire(bar) < gen * 8u) {}
        }
    }
    __syncthreads();
}

template <int V>
__global__ void __launch_bounds__(NT, 1) bar_kernel(unsigned int* bar, float* sink, int iters, int stores, unsigned long long* out) {
    unsigned int gen = 0;
    gsync<V>(bar, gen);
    const unsigned long long t0 = gtime();
    for (int it = 0; it < iters; ++it) {
        for (int s = 0; s < stores; ++s) sink[((size_t)(blockIdx.x * stores + s) * NT + threadIdx.x)] = (float)it;
        gsync<V>(bar, gen);
    }
    const unsigned long long t1 = gtime();
    if (blockIdx.x == 0 && threadIdx.x == 0) out[0] = t1 - t0;
}

// ---- staging
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
template <int MODE>
__global__ void __launch_bounds__(NT, 1) stage_kernel(unsigned int* bar, const uint4* planes, int n16, int iters, float* sink, unsigned long long* out) {
    extern __shared__ __align__(128) unsigned char smraw[];
    uint4* dst = reinterpret_cast<uint4*>(smraw + 64);
    uint64_t* mb = reinterpret_cast<uint64_t*>(smraw);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mb)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    unsigned int gen = 0, ph = 0;
    float acc = 0.0f;
    gsync<0>(bar, gen);
    const unsigned long long t0 = gtime();
    for (int it = 0; it < iters; ++it) {
        if (MODE == 0) {
            for (int i = threadIdx.x; i < n16; i += NT) cp_async16(dst + i, planes + i);
            asm volatile("cp.async.wait_all;" ::: "memory");
        } else if (MODE == 1) {
            const int rot = (int)(((long long)blockIdx.x * n16 / gridDim.x) & ~(NT - 1));
            for (int i = threadIdx.x; i < n16; i += NT) {
                int j = i + rot;
                if (j >= n16) j -= n16;
                cp_async16(dst + j, planes + j);
            }
            asm volatile("cp.async.wait_all;" ::: "memory");
        } else {
            constexpr int PIECE = 512;   // uint4 per bulk copy (8 KB)
            const int np = (n16 + PIECE - 1) / PIECE;
            if (threadIdx.x == 0) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mb)), "r"((uint32_t)n16 * 16u) : "memory");
                const int rot = MODE == 3 ? (int)((blockIdx.x * np) / gridDim.x) : 0;
                for (int q = 0; q < np; ++q) {
                    int pz = q + rot;
                    if (pz >= np) pz -= np;
                    const int cnt = min(PIECE, n16 - pz * PIECE);
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst + pz * PIECE)),
                                 "l"(planes + pz * PIECE), "r"((uint32_t)cnt * 16u), "r"(smem_u32(mb))
                                 : "memory");
                }
            }
            uint32_t done = 0;
            while (!done) {
                asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(done) : "r"(smem_u32(mb)), "r"(ph) : "memory");
            }
            ph ^= 1u;
        }
        __syncthreads();
        acc += reinterpret_cast<const float*>(dst)[(threadIdx.x * 37 + it) % (n16 * 4)];
        gsync<0>(bar, gen);
    }
    const unsigned long long t1 = gtime();
    if (acc == 12345.678f) sink[0] = acc;
    if (blockIdx.x == 0 && threadIdx.x == 0) out[0] = t1 - t0;
}

// ---- L2 prefetch ahead of a streaming stage
__global__ void __launch_bounds__(NT, 1) pf_kernel(unsigned int* bar, const uint4* buf, size_t chunk16, int n_chunks, int reps, int nbar, int do_pf,
                                                   float* sink, unsigned long long* out) {
    unsigned int gen = 0;
    unsigned int x = 0;
    unsigned long long t_stream = 0, t_total0 = 0;
    gsync<0>(bar, gen);
    t_total0 = gtime();
    for (int rep = 0; rep < reps; ++rep) {
        for (int c = 0; c < n_chunks; ++c) {
            const uint4* base = buf + (size_t)c * chunk16;
            if (do_pf && threadIdx.x < 32) {
                // this CTA's 1/grid slice, 16 KB pieces, one piece per lane and round
                const size_t per = (chunk16 + gridDim.x - 1) / gridDim.x;
                const size_t b0 = (size_t)blockIdx.x * per, b1 = min(chunk16, b0 + per);
                for (size_t o = b0 + (size_t)threadIdx.x * 1024; o < b1; o += 32 * 1024) {
                    const uint32_t bytes = (uint32_t)(min((size_t)1024, b1 - o) * 16);
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + o), "r"(bytes) : "memory");
                }
            }
            for (int b = 0; b < nbar; ++b) gsync<0>(bar, gen);
            const unsigned long long t0 = gtime();
            // stream the chunk: grid-strided 16-byte loads, 8 in flight per thread
            const size_t stride = (size_t)gridDim.x * NT;
            size_t i = (size_t)blockIdx.x * NT + threadIdx.x;
            for (; i + 7 * stride < chunk16; i += 8 * stride) {
                uint4 v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[k].x), "=r"(v[k].y), "=r"(v[k].z), "=r"(v[k].w) : "l"(base + i + k * stride));
#pragma unroll
                for (int k = 0; k < 8; ++k) x ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
            }
            gsync<0>(bar, gen);
            t_stream += gtime() - t0;
        }
    }
    const unsigned long long t1 = gtime();
    if (x == 0x12345u) sink[0] = 1.0f;
    if (blockIdx.x == 0 && threadIdx.x == 0) { out[0] = t_stream; out[1] = t1 - t_total0; }
}

template <typename K, typename... A>
static void coop(K k, int grid, size_t smem, A... args) {
    void* p[] = {(void*)&args...};
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaLaunchCooperativeKernel((void*)k, dim3(grid), dim3(NT), p, smem, 0));
    CK(cudaDeviceSynchronize());
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int grid = prop.multiProcessorCount;
    printf("device %s, %d SMs\n", prop.name, grid);
    unsigned int* bar;
    float* sink;
    unsigned long long* out;
    CK(cudaMalloc(&bar, 4096));
    CK(cudaMalloc(&sink, (size_t)grid * 64 * NT * 4));
    CK(cudaMallocManaged(&out, 64));
    const size_t big_smem = 120 * 1024;   // forces one CTA per SM
    const int iters = 2000;
#define BAR(V, ST)                                                           \
    do {                                                                     \
        CK(cudaMemset(bar, 0, 4096));                                        \
        coop(bar_kernel<V>, grid, big_smem, bar, sink, iters, ST, out);      \
        printf("bar V%d stores/thread %d: %.3f us / barrier\n", V, ST, out[0] / 1000.0 / iters); \
    } while (0)
    for (int st : {0, 1, 4}) {
        BAR(0, st); BAR(1, st); BAR(2, st); BAR(3, st); BAR(4, st);
    }
    // staging: 24 rows (NT8 = 3), d = 768: 2 planes x 3 x 24 chunks x 32 x 16 B = 73728 B; d = 1024 (medium): 98304 B; 1/3 slab of d=768
    uint4* planes;
    CK(cudaMalloc(&planes, 1 << 20));
    CK(cudaMemset(planes, 1, 1 << 20));
    for (int bytes : {24576, 73728, 98304}) {
        const int n16 = bytes / 16;
#define STAGE(M)                                                                              \
    do {                                                                                      \
        CK(cudaMemset(bar, 0, 4096));                                                         \
        coop(stage_kernel<M>, grid, (size_t)bytes + 1024, bar, (const uint4*)planes, n16, iters, sink, out); \
        printf("stage mode %d, %d B per CTA: %.3f us / (staging + barrier)\n", M, bytes, out[0] / 1000.0 / iters); \
    } while (0)
        STAGE(0); STAGE(1); STAGE(2); STAGE(3);
    }
    // L2 prefetch
    for (size_t mb : {45, 89}) {
        const size_t chunk16 = mb * 1000 * 1000 / 16;
        const int n_chunks = 12;
        uint4* buf;
        CK(cudaMalloc(&buf, chunk16 * 16 * n_chunks));
        CK(cudaMemset(buf, 3, chunk16 * 16 * n_chunks));
        for (int nbar : {12, 24}) {
            for (int pf : {0, 1}) {
                CK(cudaMemset(bar, 0, 4096));
                coop(pf_kernel, grid, big_smem, bar, (const uint4*)buf, chunk16, n_chunks, 3, nbar, pf, sink, out);
                printf("pf chunk %zu MB, %d barriers ahead, prefetch %d: stream %.2f us / chunk (%.0f GB/s), total %.2f us / chunk\n", mb, nbar, pf,
                       out[0] / 1000.0 / (3 * n_chunks), (double)chunk16 * 16 / (out[0] / (3.0 * n_chunks)), out[1] / 1000.0 / (3 * n_chunks));
            }
        }
        CK(cudaFree(buf));
    }
    return 0;
}
