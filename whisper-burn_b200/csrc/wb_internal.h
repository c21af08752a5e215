// Internal declarations shared by the translation units of libwhisper_b200.so.
// Nothing here is part of the C ABI (include/whisper_b200.h).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/whisper_b200.h"

namespace wb {

// ---- errors -----------------------------------------------------------------------------
struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
void set_last_error(const std::string& m);
[[noreturn]] void fail(int code, const std::string& m);

#define WB_CUDA(expr)                                                                           \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess)                                                                  \
            ::wb::fail(_e == cudaErrorMemoryAllocation ? WB_ERR_OOM : WB_ERR_CUDA,              \
                       std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" + \
                           std::to_string(__LINE__) + ")");                                     \
    } while (0)

#define WB_REQUIRE(cond, msg)                                   \
    do {                                                        \
        if (!(cond)) ::wb::fail(WB_ERR_INVALID_ARG, (msg));     \
    } while (0)

// kernels launched by this library (bench.py's gpu_launches)
extern thread_local int64_t g_launch_count;
#define WB_LAUNCH_CHECK()                     \
    do {                                      \
        ++::wb::g_launch_count;               \
        WB_CUDA(cudaPeekAtLastError());       \
    } while (0)

// ---- per-device launch configuration cache -----------------------------------------------------
// cudaFuncSetAttribute / occupancy results belong to a DEVICE: one slot per device ordinal, guarded by a mutex
// (a process may create models on several devices and sessions from several host threads).
struct PerDeviceConfig {
    std::mutex mu;
    size_t value[16] = {};
    // runs configure() when the current device has not been configured for `want` yet; returns what configure() returned
    template <typename F>
    bool ensure(size_t want, F&& configure) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return configure();
        std::lock_guard<std::mutex> lock(mu);
        if (value[dev] == want) return true;
        if (!configure()) return false;
        value[dev] = want;
        return true;
    }
};

// Launches of a persistent cluster kernel (decoder4.cu, decoder6.cu), one object per kernel instance.  The kernel synchronises
// its whole grid, so every cluster it launches must be co-resident: capacity() asks the device once how many clusters it holds,
// launch() asks the driver to enforce that (cooperative cluster launch).  A driver that rejects the cooperative attribute gets
// plain cluster launches from then on, whose co-residency rests on the occupancy query; so does WB200_NO_COOP (profilers
// cannot replay cooperative cluster launches).
struct ClusterLaunch {
    std::mutex mu;
    int clusters[16] = {};   // per device ordinal: 0 not queried, > 0 co-resident clusters, -1 the kernel does not fit
    bool plain[16] = {};     // per device ordinal: launch without the cooperative attribute
    static cudaLaunchConfig_t config(int cs, int n_clusters, int threads, size_t smem, cudaStream_t st, cudaLaunchAttribute (&attr)[2]) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(n_clusters * cs);
        cfg.blockDim = dim3(threads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cs;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        attr[1].id = cudaLaunchAttributeCooperative;
        attr[1].val.cooperative = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        return cfg;
    }
    // co-resident clusters of `cs` CTAs on the current device; 0 when the kernel does not fit it
    int capacity(const void* k, int cs, int threads, size_t smem, const char* name) {
        int dev = 0;
        WB_CUDA(cudaGetDevice(&dev));
        if (dev < 0 || dev >= 16) return 0;
        std::lock_guard<std::mutex> lock(mu);
        if (clusters[dev] == 0) {
            clusters[dev] = -1;
            if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
                (cs > 8 && cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess)) {
                cudaGetLastError();
                return 0;
            }
            cudaLaunchAttribute attr[2];
            const cudaLaunchConfig_t cfg = config(cs, 1, threads, smem, nullptr, attr);
            int n = 0;
            const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, k, &cfg);
            if (getenv("WB200_VERBOSE")) fprintf(stderr, "[wb] %s: cluster %d, smem %zu B, max active clusters %d (%s)\n", name, cs, smem, n, cudaGetErrorString(e));
            if (e != cudaSuccess || n < 1) {
                cudaGetLastError();
                return 0;
            }
            clusters[dev] = n;
            plain[dev] = getenv("WB200_NO_COOP") != nullptr;
        }
        return std::max(clusters[dev], 0);
    }
    // n_clusters clusters of `cs` CTAs; args as for cudaLaunchKernel
    void launch(const void* k, int cs, int n_clusters, int threads, size_t smem, void** args, cudaStream_t st, const char* name) {
        int dev = 0;
        WB_CUDA(cudaGetDevice(&dev));
        std::lock_guard<std::mutex> lock(mu);
        cudaLaunchAttribute attr[2];
        cudaLaunchConfig_t cfg = config(cs, n_clusters, threads, smem, st, attr);
        if (!plain[dev]) {
            cfg.numAttrs = 2;
            const cudaError_t e = cudaLaunchKernelExC(&cfg, k, args);
            if (e == cudaSuccess) {
                WB_LAUNCH_CHECK();
                return;
            }
            cudaGetLastError();
            plain[dev] = true;
            cfg.numAttrs = 1;
            if (getenv("WB200_VERBOSE")) fprintf(stderr, "[wb] %s: cooperative cluster launch rejected (%s), using a plain cluster launch\n", name, cudaGetErrorString(e));
        }
        WB_CUDA(cudaLaunchKernelExC(&cfg, k, args));
        WB_LAUNCH_CHECK();
    }
};

// ---- device buffer ----------------------------------------------------------------------
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
    void alloc(size_t count) {
        release();
        if (count == 0) return;
        WB_CUDA(cudaMalloc((void**)&p, count * sizeof(T)));
        n = count;
    }
    void ensure(size_t count) {
        if (count > n) alloc(count);
    }
    void zero(cudaStream_t st) {
        if (p) WB_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), st));
    }
};

// ---- constant tables of the frontend (host-built, f32 op order of audio.rs) ----------------
constexpr int N_FFT = 400, HOP = 160, N_MELS = 80, N_FREQ = 201;
constexpr int KPAD = 208;                 // 201 padded to a multiple of 8
struct FrontendTables {
    std::vector<float> hann;              // [400]            audio.rs:272-278
    std::vector<float> basis_t;           // [400][2*KPAD]    audio.rs:349-364, transposed: [j][cos k.. | sin k..]
    std::vector<float> mel_filt;          // [80][201]        audio.rs:67-143
    int mel_lo[N_MELS], mel_hi[N_MELS];   // non-zero tap range of every filter
};
const FrontendTables& frontend_tables();

// ---- model ----------------------------------------------------------------------------------
struct LinearW {       // y = x @ W + b, stored transposed: w[n][k] (k contiguous)
    float* w32 = nullptr;   // fp32 [N][K]   (encoder GEMMs, and decoder when !fp16_exact)
    __half* w16 = nullptr;  // fp16 [N][K]   (decoder GEMVs when fp16_exact)
    float* b = nullptr;     // [N] (never null; zeros when the reference has no bias)
    int n = 0, k = 0;
};
struct LayerNormW {
    float* g = nullptr;
    float* b = nullptr;
    float eps = 1e-5f;
};
struct EncBlockW {
    LayerNormW attn_ln, mlp_ln;
    LinearW qkv;        // [3d][d]  rows: q | k | v
    LinearW out, mlp1, mlp2;
};
struct DecBlockW {
    LayerNormW attn_ln, cross_ln, mlp_ln;
    LinearW qkv;        // self-attention q | k | v
    LinearW out;
    LinearW cq;         // cross query
    LinearW ckv;        // cross k | v  [2d][d]  (applied to the encoder output once per window)
    LinearW cout, mlp1, mlp2;
};

struct Model {
    wb_dims dims{};
    int device = 0;
    bool finalized = false;
    bool fp16_exact = false;
    int ln_eps_outside = 1;     // burn 0.9: (x-mean)/(sqrt(var)+eps)
    std::map<std::string, std::pair<std::vector<int64_t>, std::vector<float>>> host;  // until finalize

    std::vector<void*> allocs;  // everything cudaMalloc'ed for weights
    // frontend tables
    float* basis_t = nullptr;   // [400][416]
    float* mel_filt = nullptr;  // [80][201]
    int* mel_range = nullptr;   // [80][2]
    // encoder
    LinearW conv1;              // [d][3*80]   k = kk*80 + c
    LinearW conv2;              // [d][3*d]    k = kk*d + c
    float* enc_pos = nullptr;   // [n_audio_ctx][d]
    std::vector<EncBlockW> enc;
    LayerNormW ln_post;
    // decoder
    float* tok_emb32 = nullptr;   // [V][d] (always kept: embedding lookup + fp32 logits path)
    __half* tok_emb16 = nullptr;  // [V][d] when fp16_exact
    __half* tok_emb16_tiled = nullptr;   // [ceil(V/16)][2][16][d/2] half-tiles for decoder4.cu (d = 128 / 384 only)
    float* dec_pos = nullptr;     // [n_text_ctx][d]
    std::vector<DecBlockW> dec;
    LayerNormW dec_ln;
    float* zero_bias = nullptr;   // [max(4d, V)] zeros

    ~Model();
};

// ---- GEMM (gemm.cu) -------------------------------------------------------------------------
// C[g][m][n] = epilogue( sum_k A[g][m][k] * B[n][k] ), fp32.  Rows are grouped (one group per
// audio window) so that A rows may overlap (lda < K: the conv stems read a sliding 3-row
// window of a token-major buffer); plain GEMMs use one group.
struct GemmGroup {
    int64_t a_off;   // element offset of the group's first A row
    int64_t c_off;   // element offset of the group's first C row (also residual)
    int rows;
};
enum { ACT_NONE = 0, ACT_GELU = 1 };
struct GemmParams {
    const float* A = nullptr;
    int64_t lda = 0;
    const float* B = nullptr;      // [N][K]
    float* C = nullptr;
    int64_t ldc = 0;
    int N = 0, K = 0;
    const float* bias = nullptr;   // [N] or null
    int act = ACT_NONE;
    float scale = 1.0f;            // applied to columns < scale_cols after bias (q/k pre-scaling)
    int scale_cols = 0;
    const float* residual = nullptr;  // same layout as C, or null
    const float* pos = nullptr;       // [rows][N] added after activation, indexed by the row inside the group
    const GemmGroup* groups = nullptr;   // device array
    int n_groups = 1;
    int max_rows = 0;                 // max rows over groups
};
void launch_gemm(const GemmParams& p, cudaStream_t st);

// ---- tensor-core GEMM on fp16 hi/lo planes (gemm_f16.cu) ----------------------------------------------------
// A = A_hi + A_lo / 2048 (fp16 planes, row-major [rows][lda]), B = fp16 [N][K] (exact weights); see gemm_f16.cu.
struct GemmF16Params {
    const __half *A_hi = nullptr, *A_lo = nullptr;
    int64_t lda = 0;
    const __half* B = nullptr;        // [N][K]
    float* C = nullptr;               // fp32 result rows, or null
    __half *P_hi = nullptr, *P_lo = nullptr;   // fp16 planes of the result, or null
    int64_t ldc = 0;
    int N = 0, K = 0;
    const float* bias = nullptr;
    int act = ACT_NONE;
    float scale = 1.0f;
    int scale_cols = 0;
    const float* residual = nullptr;
    const float* pos = nullptr;
    const GemmGroup* groups = nullptr;
    int n_groups = 1;
    int max_rows = 0;
};
bool gemm_f16_supported(const GemmF16Params& p);
// Tensor maps and launch geometry of one GEMM site, built once per (site, geometry) instead of per launch
class GemmF16Plan {
public:
    GemmF16Plan();
    ~GemmF16Plan();
    GemmF16Plan(const GemmF16Plan&) = delete;
    GemmF16Plan& operator=(const GemmF16Plan&) = delete;
    void build(const GemmF16Params& p, int64_t a_group_stride, int a_rows_total_per_group);
    void launch(cudaStream_t st) const;
    bool matches(int max_rows, int n_groups) const { return impl != nullptr && key_rows == max_rows && key_groups == n_groups; }
private:
    struct Impl;
    Impl* impl = nullptr;
    int key_rows = -1, key_groups = -1;
};
void launch_split_f16(const float* src, __half* hi, __half* lo, int64_t n, cudaStream_t st);
// Logits GEMM of token scoring (gemm_f16.cu, LogitArgs): rows x E^T over E = the fp16 token embedding [V][K], reduced per
// (row, 128-column tile) to the tile max, sum of exp(x - max) and arg-max, plus each row's target logit; no logits are stored.
struct LogitStatsParams {
    const __half *A_hi = nullptr, *A_lo = nullptr;   // [rows][K] planes of the final LayerNorm
    const __half* E = nullptr;                       // [V][K]
    int rows = 0, K = 0, V = 0;
    const int* target = nullptr;                     // [rows]
    const uint8_t* row_mask = nullptr;               // [rows] or null
    const uint8_t* is_special = nullptr;             // [V]
    float *tile_m = nullptr, *tile_s = nullptr, *tgt_logit = nullptr;   // [rows][logit_stats_tiles(V)], [rows]
    int* tile_i = nullptr;
};
int logit_stats_tiles(int V);
void launch_logit_stats(const LogitStatsParams& p, cudaStream_t st);

// ---- frontend (logmel.cu) ---------------------------------------------------------------------
struct LogMelWindow {
    int64_t wave_off;   // element offset into the wave buffer
    int n_samples;
    int n_frames;       // n_samples / 160 frames enter the max of audio.rs:50
    int n_store;        // frames written out (<= n_frames; mels_to_text clips, transcribe.rs:171-173)
    int max_slot;       // windows sharing a slot share the global max of audio.rs:50
    int64_t out_off;    // element offset of frame 0's row in the token-major output (row = 80 floats)
};
// raw pass: log10(max(mel,1e-10)) token-major + per-slot max; finalize: clamp/normalise in place.
void launch_logmel(const Model& m, const float* wave, const LogMelWindow* win_dev, int n_windows,
                   int max_frames, float* mel_rows, int* max_slots, int n_slots, cudaStream_t st);
// token-major rows [n][80] -> channel-major [80][n] (the reference's [B,80,F] layout) and back
void launch_rows_to_chan(const float* rows, float* chan, int n_frames, cudaStream_t st);
void launch_chan_to_rows(const float* chan, float* rows, int n_frames, int64_t chan_stride, cudaStream_t st);

// ---- resampling to 16 kHz (resample.cu) -------------------------------------------------------------
// up / down of sample_rate -> 16 kHz after dividing by their gcd; false unless sample_rate >= 1 and max(up, down) <= 1024
bool resample_ratio(int64_t sample_rate, int& up, int& down);
// ceil(n_frames * up / down) (wb_resampled_length); -1 for an unsupported rate or n_frames < 0
int64_t resampled_length(int64_t n_frames, int64_t sample_rate);
// resample_poly's filter, scaled by up: 2 * 10 * max(up, down) + 1 f64 taps, or [1] for up = down = 1
std::vector<double> resample_taps(int up, int down);
struct ResampleDesc {   // one waveform of a resample launch
    int64_t in_off, n;        // first interleaved input sample, frames
    int64_t out_off, n_out;   // first output sample, outputs
    int64_t taps_off, tile0;  // its filter in the taps buffer, its first output tile
    int channels, up, down, half;
};
struct ResampleBufs {   // device buffers of resample_waveforms, grown to the largest call
    DevBuf<float> in, out;
    DevBuf<double> taps;
    DevBuf<ResampleDesc> desc;
};
// Uploads n_waveforms interleaved host waveforms (frames x channels at sample_rates[w]; every rate supported) and resamples
// all of them to 16 kHz mono in one launch: waveform w lands in b.out at out_off[w], n_out[w] samples.  Synchronises st.
void resample_waveforms(ResampleBufs& b, const float* const* in, const int64_t* n_frames, const int64_t* channels,
                        const int64_t* sample_rates, int64_t n_waveforms, std::vector<int64_t>& out_off,
                        std::vector<int64_t>& n_out, cudaStream_t st);

// ---- encoder pieces (encoder.cu) -----------------------------------------------------------------
// head-major re-layout of one layer's cross K|V rows (see encoder.cu)
void launch_ckv_relayout(const float* src, void* dst, bool dst_half, const int64_t* win_row_off, const int* win_T, int n_windows,
                         int64_t M, int d, cudaStream_t st);
// LayerNorm of rows [rows][d] into fp32 rows y, or, with planes y_hi / y_lo, into fp16 hi/lo planes (and into y as well when
// it is non-null)
void launch_layernorm(const float* x, float* y, __half* y_hi, __half* y_lo, const LayerNormW& ln, int rows, int d, int eps_outside,
                      cudaStream_t st);
struct AttnWindow {
    int64_t row_off;   // first packed row of the window
    int T;
};
// non-causal multi-head attention over packed rows; qkv [rows][3d] (q,k pre-scaled), out [rows][d]
void launch_encoder_attention(const float* qkv, float* out, const AttnWindow* win_dev, int n_windows, int max_T, int d, int n_head,
                              cudaStream_t st);
// tensor-core version on fp16 hi/lo planes (enc_attn_tc.cu): q | k | v planes [rows][3d] -> output planes [rows][d]
void launch_encoder_attention_tc(const __half* qkv_hi, const __half* qkv_lo, __half* out_hi, __half* out_lo, const AttnWindow* win_dev,
                                 int n_windows, int max_T, int d, int n_head, cudaStream_t st);
// token scoring (enc_attn_tc.cu): causal self attention over the packed rows of each sequence (q | k | v planes [rows][3d];
// kv_f16: K and V enter as their fp16 rounding), and cross attention of each sequence's cross-query planes [rows][d] over its
// window's head-major cross K/V of one layer (Session::ckv / ckv16)
void launch_causal_attention_tc(const __half* qkv_hi, const __half* qkv_lo, __half* out_hi, __half* out_lo, const AttnWindow* seq_dev,
                                int n_seqs, int max_T, int d, int n_head, bool kv_f16, cudaStream_t st);
void launch_cross_attention_tc(const __half* q_hi, const __half* q_lo, const void* ckv_layer, bool kv_f16, __half* out_hi, __half* out_lo,
                               const AttnWindow* seq_dev, const int* seq_win_dev, const int64_t* win_row_off_dev, const int* win_T_dev,
                               int n_seqs, int max_T, int d, int n_head, cudaStream_t st);

}  // namespace wb
