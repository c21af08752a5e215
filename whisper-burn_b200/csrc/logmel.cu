// Fused log-mel frontend for sm_90a  (reference: src/audio.rs:34-56 prep_audio, :284-367 stfft).
//
// One CTA turns 32 STFT frames of one window into 32 token-major rows of 80 log-mel values:
//   reflect-pad + framing (audio.rs:296-346)  -> staged once in shared memory (hop-row layout,
//       row stride 161 so that the 160-sample hop does not alias one bank)
//   windowed real DFT (audio.rs:349-364)      -> dense 402x400 fp32 product against the
//       reference's own f32-angle basis (NOT an FFT: the reference's twiddles are inexact and
//       parity is defined against them), basis streamed through shared memory in 16-sample stages,
//       8 freq x 4 frame register tile per thread
//   power, drop last frame (audio.rs:40-42)   -> registers -> shared
//   mel projection (audio.rs:44-46)           -> sparse triangular taps only
//   log10(max(.,1e-10)) (audio.rs:48)         -> written once, coalesced (80 contiguous floats/row)
//   global max (audio.rs:50)                  -> warp/block reduce + one atomicMax per CTA
// A second tiny kernel applies max(x, max-8) and (x+4)/4 in place (audio.rs:52-53).
// Algorithmic HBM bytes per window: 4*n_samples in + 4*80*n_frames out (SURVEY.md 8d).
#include <climits>

#include "wb_internal.h"

namespace wb {

namespace {

constexpr int FR = 32;                  // frames per CTA
constexpr int JC = 16;                  // samples per basis stage
constexpr int XROW = 161;               // smem stride of one hop row (160 samples + 1 pad)
constexpr int NHOP = FR + 2;            // hop rows touched by FR frames: (FR-1)*160 + 400 samples
constexpr int NSAMP = (FR - 1) * HOP + N_FFT;
constexpr int XS_FLOATS = (NHOP * XROW + 3) / 4 * 4;   // keeps the stage buffer 16-byte aligned
constexpr int PS_STRIDE = FR + 1;
constexpr int STAGE_FLOATS = KPAD * PS_STRIDE;   // >= JC * 2 * KPAD, shared by basis stage and power tile
constexpr int LOGMEL_THREADS = 256;
constexpr size_t LOGMEL_SMEM = (size_t)(XS_FLOATS + STAGE_FLOATS) * sizeof(float);
static_assert(STAGE_FLOATS >= JC * 2 * KPAD, "stage buffer too small");

__device__ __forceinline__ int float_to_ordered(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int i) {
    return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff);
}

__global__ void __launch_bounds__(LOGMEL_THREADS)
logmel_raw_kernel(const float* __restrict__ wave, const LogMelWindow* __restrict__ wins,
                  const float* __restrict__ basis_t, const float* __restrict__ mel_filt,
                  const int* __restrict__ mel_range, float* __restrict__ mel_rows, int* __restrict__ max_slots) {
    extern __shared__ __align__(16) float smem[];
    float* xs = smem;
    float* stage = smem + XS_FLOATS;
    __shared__ int s_max;

    const LogMelWindow win = wins[blockIdx.y];
    const int t0 = blockIdx.x * FR;
    if (t0 >= win.n_frames) return;
    const int tid = threadIdx.x;
    const int n = win.n_samples;
    const float* x = wave + win.wave_off;
    if (tid == 0) s_max = INT_MIN;

    // ---- stage the samples of FR frames; reflect padding of 200 (audio.rs:296-306)
    const int p0 = t0 * HOP - N_FFT / 2;
    for (int s = tid; s < NSAMP; s += LOGMEL_THREADS) {
        int p = p0 + s;
        if (p < 0) p = -p;
        else if (p >= n) p = 2 * (n - 1) - p;
        float v = (p >= 0 && p < n) ? __ldg(x + p) : 0.0f;   // out of range only for frames that are never stored
        xs[(s / HOP) * XROW + (s % HOP)] = v;
    }

    const int tk = tid >> 3;   // 0..31 : 8 frequency rows each (26 groups cover 208)
    const int tf = tid & 7;    // 0..7  : 4 frames each
    const bool active = tk < KPAD / 8;
    float re[8][4], im[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int f = 0; f < 4; ++f) re[i][f] = im[i][f] = 0.0f;

    const float4* basis4 = reinterpret_cast<const float4*>(basis_t);
    float4* stage4 = reinterpret_cast<float4*>(stage);
    constexpr int ROW4 = 2 * KPAD / 4;   // float4 per basis row
    for (int c = 0; c < N_FFT / JC; ++c) {
        __syncthreads();   // previous stage consumed (and xs visible on the first pass)
        for (int i = tid; i < JC * ROW4; i += LOGMEL_THREADS) stage4[i] = __ldg(basis4 + (size_t)c * JC * ROW4 + i);
        __syncthreads();
        if (active) {
#pragma unroll 4
            for (int jj = 0; jj < JC; ++jj) {
                const int j = c * JC + jj;
                const int h = j / HOP, r = j - h * HOP;
                float xv[4];
#pragma unroll
                for (int f = 0; f < 4; ++f) xv[f] = xs[(tf * 4 + f + h) * XROW + r];
                const float4 c0 = *reinterpret_cast<const float4*>(stage + jj * 2 * KPAD + tk * 8);
                const float4 c1 = *reinterpret_cast<const float4*>(stage + jj * 2 * KPAD + tk * 8 + 4);
                const float4 s0 = *reinterpret_cast<const float4*>(stage + jj * 2 * KPAD + KPAD + tk * 8);
                const float4 s1 = *reinterpret_cast<const float4*>(stage + jj * 2 * KPAD + KPAD + tk * 8 + 4);
                const float cc[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
                const float ss[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int f = 0; f < 4; ++f) {
                        re[i][f] = fmaf(cc[i], xv[f], re[i][f]);
                        im[i][f] = fmaf(ss[i], xv[f], im[i][f]);
                    }
            }
        }
    }
    __syncthreads();
    // ---- power spectrum re^2 + im^2 (audio.rs:40), each term rounded like powf(2.0) + add
    if (active) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int k = tk * 8 + i;
#pragma unroll
            for (int f = 0; f < 4; ++f)
                stage[k * PS_STRIDE + tf * 4 + f] = __fadd_rn(__fmul_rn(re[i][f], re[i][f]), __fmul_rn(im[i][f], im[i][f]));
        }
    }
    __syncthreads();
    // ---- mel projection + log10 (audio.rs:44-48)
    const float LN10 = 2.30258509299404568402f;   // fl32(ln 10), helper.rs:24-27
    float lmax = -3.0e38f;
    for (int idx = tid; idx < N_MELS * FR; idx += LOGMEL_THREADS) {
        const int m = idx % N_MELS, f = idx / N_MELS;
        const int t = t0 + f;
        if (t >= win.n_frames) continue;   // also drops the reference's last frame (audio.rs:42)
        const int lo = mel_range[2 * m], hi = mel_range[2 * m + 1];
        float acc = 0.0f;
        for (int k = lo; k < hi; ++k) acc = fmaf(__ldg(mel_filt + m * N_FREQ + k), stage[k * PS_STRIDE + f], acc);
        float d = __fsub_rn(acc, 1.0e-10f);        // tensor_max_scalar: relu(x - m) + m  (helper.rs:8-10)
        d = d > 0.0f ? d : 0.0f;
        const float v = __fadd_rn(d, 1.0e-10f);
        const float lg = __fdiv_rn(logf(v), LN10);
        if (t < win.n_store) mel_rows[win.out_off + (int64_t)t * N_MELS + m] = lg;
        lmax = fmaxf(lmax, lg);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    if ((tid & 31) == 0) atomicMax(&s_max, float_to_ordered(lmax));
    __syncthreads();
    if (tid == 0) atomicMax(max_slots + win.max_slot, s_max);
}

// max(x, max-8) via relu identity, then (x + 4) / 4   (audio.rs:50-53, helper.rs:8-10)
__global__ void logmel_finalize_kernel(const LogMelWindow* __restrict__ wins, float* __restrict__ mel_rows,
                                       const int* __restrict__ max_slots) {
    const LogMelWindow win = wins[blockIdx.y];
    const int total = win.n_store * N_MELS;
    const float mx = ordered_to_float(max_slots[win.max_slot]);
    const float m8 = (float)((double)mx - 8.0);
    float* p = mel_rows + win.out_off;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        float d = __fsub_rn(p[i], m8);
        d = d > 0.0f ? d : 0.0f;
        const float v = __fadd_rn(d, m8);
        p[i] = __fdiv_rn(__fadd_rn(v, 4.0f), 4.0f);
    }
}

__global__ void rows_to_chan_kernel(const float* __restrict__ rows, float* __restrict__ chan, int n_frames) {
    __shared__ float tile[32][N_MELS + 1];
    const int t0 = blockIdx.x * 32;
    for (int i = threadIdx.x; i < 32 * N_MELS; i += blockDim.x) {
        const int f = i / N_MELS, m = i % N_MELS;
        tile[f][m] = (t0 + f < n_frames) ? rows[(int64_t)(t0 + f) * N_MELS + m] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * N_MELS; i += blockDim.x) {
        const int m = i / 32, f = i % 32;
        if (t0 + f < n_frames) chan[(int64_t)m * n_frames + t0 + f] = tile[f][m];
    }
}

__global__ void chan_to_rows_kernel(const float* __restrict__ chan, float* __restrict__ rows, int n_frames,
                                    int64_t chan_stride) {
    __shared__ float tile[32][N_MELS + 1];
    const int t0 = blockIdx.x * 32;
    for (int i = threadIdx.x; i < 32 * N_MELS; i += blockDim.x) {
        const int m = i / 32, f = i % 32;
        tile[f][m] = (t0 + f < n_frames) ? chan[(int64_t)m * chan_stride + t0 + f] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * N_MELS; i += blockDim.x) {
        const int f = i / N_MELS, m = i % N_MELS;
        if (t0 + f < n_frames) rows[(int64_t)(t0 + f) * N_MELS + m] = tile[f][m];
    }
}

}  // namespace

void launch_logmel(const Model& m, const float* wave, const LogMelWindow* win_dev, int n_windows, int max_frames,
                   float* mel_rows, int* max_slots, int n_slots, cudaStream_t st) {
    static PerDeviceConfig cfg;
    cfg.ensure(LOGMEL_SMEM, [&] {
        WB_CUDA(cudaFuncSetAttribute(logmel_raw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LOGMEL_SMEM));
        return true;
    });
    WB_CUDA(cudaMemsetAsync(max_slots, 0x80, sizeof(int) * n_slots, st));   // very negative ordered key
    dim3 grid((max_frames + FR - 1) / FR, n_windows);
    logmel_raw_kernel<<<grid, LOGMEL_THREADS, LOGMEL_SMEM, st>>>(wave, win_dev, m.basis_t, m.mel_filt, m.mel_range,
                                                                   mel_rows, max_slots);
    WB_LAUNCH_CHECK();
    dim3 grid2((max_frames * N_MELS + 255) / 256 > 64 ? 64 : (max_frames * N_MELS + 255) / 256, n_windows);
    logmel_finalize_kernel<<<grid2, 256, 0, st>>>(win_dev, mel_rows, max_slots);
    WB_LAUNCH_CHECK();
}

void launch_rows_to_chan(const float* rows, float* chan, int n_frames, cudaStream_t st) {
    rows_to_chan_kernel<<<(n_frames + 31) / 32, 256, 0, st>>>(rows, chan, n_frames);
    WB_LAUNCH_CHECK();
}

void launch_chan_to_rows(const float* chan, float* rows, int n_frames, int64_t chan_stride, cudaStream_t st) {
    chan_to_rows_kernel<<<(n_frames + 31) / 32, 256, 0, st>>>(chan, rows, n_frames, chan_stride);
    WB_LAUNCH_CHECK();
}

}  // namespace wb
