// Token alignment (wb_session_align_tokens, wb_align_dtw): openai-whisper's find_alignment (whisper/timing.py) on this project's
// rows.  Times come from a separate teacher-forced pass over a finished transcript; the decoders and the ids they emit are not
// touched.  Per group of whole sequences (at most SCORE_GROUP_ROWS rows, one row per position, score.cu's grouping):
//   decoder_pass (score.cu) over every position, stopping after the cross-query GEMM of the last layer holding a selected head;
//   after each such layer's cross-query GEMM, for its selected heads:
//     align_qk_kernel       q . k of each position against the window's first C scaled keys (the head-major cross K the
//                           decoders read; fp16 keys under WB_KV_F16), 3-term hi/lo mma.sync as enc_attn_tc.cu
//     align_softmax_kernel  softmax over the C columns (crop first, then exp(x - max) / sum)
//     align_stats_kernel    per column: mean and biased std over the sequence's L positions (f64)
//     align_filter_kernel   (w - mean) / std (0 where std = 0), width-7 median along the columns with reflect padding (none
//                           when C <= 3), summed into each kept row [first - 1, L - 2] of the matrix in ascending head order;
//                           after the last layer divided by the head count
//   align_dtw_kernel        one CTA per sequence: DTW on -matrix over the anti-diagonals, 2-bit trace in shared memory, then
//                           the backtrace (host/dtw.hpp) -> start / end per aligned id.
// Workspace: the weights of one layer's selected heads of one group, [heads][rows][Cmax] f32 (at most n_text_head x 4096 x
// n_audio_ctx x 4 B: 295 MB for small.en's 12 heads, 492 MB for 20 heads), their column statistics, the group's matrices.
#include <algorithm>
#include <cmath>

#include "../host/dtw.hpp"
#include "attn_tile.cuh"
#include "session.h"

namespace wb {

namespace {

constexpr int AQ_THREADS = 128;
constexpr int DTW_MAX_ROWS = 448;                 // one thread per matrix row
constexpr int DTW_DIAG = DTW_MAX_ROWS + 1;        // floats per anti-diagonal buffer (rows 1 .. 448)
constexpr int DTW_BLOCK = 8;                      // anti-diagonals per register prefetch block
constexpr size_t DTW_SMEM_MAX = 227 * 1024;       // an H100 CTA's shared memory

size_t dtw_smem(int64_t N, int64_t C) { return (size_t)3 * DTW_DIAG * sizeof(float) + (size_t)N * ((C + 15) / 16) * sizeof(uint32_t); }

// w[hs][row_off + r][c] = q_r . k_c of head heads[hs] for every position r < L and column c < C of sequence blockIdx.z
template <typename KVT>
__global__ void __launch_bounds__(AQ_THREADS)
align_qk_kernel(const __half* __restrict__ q_hi, const __half* __restrict__ q_lo, const KVT* __restrict__ ckv, const AlignSeq* __restrict__ seqs,
                const int* __restrict__ heads, const int64_t* __restrict__ win_row_off, const int* __restrict__ win_T, int d, int64_t rows,
                int ldw, float* __restrict__ w) {
    constexpr bool KV16 = sizeof(KVT) == 2;
    __shared__ __align__(128) uint8_t sm[4 * TILE_B];   // Q hi, Q lo, K hi, K lo
    const AlignSeq sq = seqs[blockIdx.z];
    const int q0 = blockIdx.x * TQ;
    if (q0 >= sq.L) return;
    const int hs = blockIdx.y, h = heads[hs], tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int Tk = win_T[sq.win];
    const KVT* blk = ckv + win_row_off[sq.win] * 2 * (int64_t)d + (int64_t)h * Tk * 128;   // as cross_attn_tc_kernel reads it
    const uint32_t sQ = smem_u32(sm), sK = sQ + 2 * TILE_B;
    for (int i = tid; i < 64 * 8; i += AQ_THREADS) {
        const int r = i >> 3, c = i & 7;
        const bool ok = q0 + r < sq.L;
        const int64_t off = (sq.row_off + (ok ? q0 + r : 0)) * (int64_t)d + h * HD + c * 8;
        cp16(sQ + tile_off(r, c), q_hi + off, ok);
        cp16(sQ + TILE_B + tile_off(r, c), q_lo + off, ok);
    }
    uint32_t qh[4][4], ql[4][4];
    float* wq = w + ((int64_t)hs * rows + sq.row_off) * ldw;
    for (int k0 = 0; k0 < sq.C; k0 += TK) {
        for (int i = tid; i < 64 * 8; i += AQ_THREADS) {   // keys k0 .. k0 + 63: the first 64 elements of each position
            const int r = i >> 3, c = i & 7, j = k0 + r;
            const bool ok = j < sq.C;
            const uint32_t dst = sK + tile_off(r, c);
            const KVT* row = blk + (int64_t)(ok ? j : 0) * 128;
            if constexpr (KV16) {
                cp16(dst, row + ((c ^ (4 * (j & 1))) << 3), ok);
            } else {
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
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        if (k0 == 0) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const int r = warp * 16 + (lane & 15), c = ks * 2 + (lane >> 4);
                ldsm4(sQ + tile_off(r, c), qh[ks][0], qh[ks][1], qh[ks][2], qh[ks][3]);
                ldsm4(sQ + TILE_B + tile_off(r, c), ql[ks][0], ql[ks][1], ql[ks][2], ql[ks][3]);
            }
        }
        float s_m[8][4], s_c[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) { s_m[i][j] = 0.0f; s_c[i][j] = 0.0f; }
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
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
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int q = q0 + warp * 16 + g + 8 * e;
            if (q >= sq.L) continue;
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int b = 0; b < 2; ++b) {
                    const int key = k0 + i * 8 + 2 * t + b;
                    if (key < sq.C) wq[(int64_t)q * ldw + key] = hl_join(s_m[i][2 * e + b], s_c[i][2 * e + b]);
                }
        }
        __syncthreads();   // every warp is done with the K tile before the next one overwrites it
    }
}

// softmax over the C columns of every position: one warp per (head, position)
__global__ void align_softmax_kernel(const AlignSeq* __restrict__ seqs, int64_t rows, int ldw, float* __restrict__ w) {
    const AlignSeq sq = seqs[blockIdx.z];
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= sq.L) return;
    float* x = w + ((int64_t)blockIdx.y * rows + sq.row_off + r) * ldw;
    float mx = -INFINITY, s = 0.0f;
    for (int c = lane; c < sq.C; c += 32) mx = fmaxf(mx, x[c]);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    for (int c = lane; c < sq.C; c += 32) s = __fadd_rn(s, expf(__fsub_rn(x[c], mx)));
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    for (int c = lane; c < sq.C; c += 32) x[c] = __fdiv_rn(expf(__fsub_rn(x[c], mx)), s);
}

// stats[hs][seq][c] = (mean, biased std) of column c over the sequence's L positions, in f64
__global__ void align_stats_kernel(const AlignSeq* __restrict__ seqs, int n_seqs, int64_t rows, int ldw, const float* __restrict__ w,
                                   double* __restrict__ stats) {
    const AlignSeq sq = seqs[blockIdx.z];
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= sq.C) return;
    const float* x = w + ((int64_t)blockIdx.y * rows + sq.row_off) * ldw + c;
    double sum = 0.0, sq_sum = 0.0;
    for (int r = 0; r < sq.L; ++r) sum += (double)x[(int64_t)r * ldw];
    const double mean = sum / sq.L;
    for (int r = 0; r < sq.L; ++r) {
        const double dv = (double)x[(int64_t)r * ldw] - mean;
        sq_sum += dv * dv;
    }
    double* o = stats + (((int64_t)blockIdx.y * n_seqs + blockIdx.z) * ldw + c) * 2;
    o[0] = mean;
    o[1] = sqrt(sq_sum / sq.L);
}

// matrix[k][c] += median filter of the normalised weights of each head of this layer (ascending), rows k = 0 .. N-1 of the
// sequence (position first - 1 + k); last: then divided by n_total
__global__ void align_filter_kernel(const AlignSeq* __restrict__ seqs, int n_seqs, int n_heads, int64_t rows, int ldw,
                                    const float* __restrict__ w, const double* __restrict__ stats, bool last, int n_total,
                                    float* __restrict__ mat) {
    const AlignSeq sq = seqs[blockIdx.z];
    const int c = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y, C = sq.C;
    if (c >= C || k >= sq.L - sq.first) return;
    float* out = mat + sq.mat_off + (int64_t)k * C + c;
    float acc = *out;
    for (int hs = 0; hs < n_heads; ++hs) {
        const float* x = w + ((int64_t)hs * rows + sq.row_off + sq.first - 1 + k) * ldw;
        const double* st = stats + ((int64_t)hs * n_seqs + blockIdx.z) * ldw * 2;
        auto norm = [&](int cc) {
            const double sd = st[2 * cc + 1];
            return sd == 0.0 ? 0.0f : (float)(((double)x[cc] - st[2 * cc]) / sd);
        };
        float v;
        if (C <= 3) {
            v = norm(c);
        } else {
            float a[7];
#pragma unroll
            for (int u = 0; u < 7; ++u) {
                int cc = c - 3 + u;
                cc = cc < 0 ? -cc : cc >= C ? 2 * (C - 1) - cc : cc;   // torch reflect padding (scipy "mirror")
                a[u] = norm(cc);
            }
#pragma unroll
            for (int i = 0; i < 6; ++i)
#pragma unroll
                for (int j = 0; j < 6 - i; ++j) {
                    const float lo = fminf(a[j], a[j + 1]), hi = fmaxf(a[j], a[j + 1]);
                    a[j] = lo;
                    a[j + 1] = hi;
                }
            v = a[3];
        }
        acc = __fadd_rn(acc, v);
    }
    if (last) acc = __fdiv_rn(acc, (float)n_total);
    *out = acc;
}

// DTW of sequence blockIdx.x's matrix (N = L - first rows, C columns at mat_off) -> start / end at out_off.  Thread i - 1 owns
// row i and walks it one cell per anti-diagonal s = i + j, prefetching its row of the matrix DTW_BLOCK cells ahead.
__global__ void __launch_bounds__(DTW_MAX_ROWS)
align_dtw_kernel(const float* __restrict__ mat, const AlignSeq* __restrict__ seqs, const int64_t* __restrict__ out_off, int* __restrict__ start,
                 int* __restrict__ end) {
    extern __shared__ __align__(16) uint8_t dsm[];
    float* diag = reinterpret_cast<float*>(dsm);                           // [3][DTW_DIAG]: cost of row i on diagonals s % 3
    uint32_t* trace = reinterpret_cast<uint32_t*>(diag + 3 * DTW_DIAG);   // [N][W]: 2-bit codes, 16 cells per word
    const AlignSeq sq = seqs[blockIdx.x];
    const int N = sq.L - sq.first, C = sq.C, W = (C + 15) / 16, i = threadIdx.x + 1;
    const bool mine = i <= N;
    const float* x = mat + sq.mat_off + (int64_t)(i - 1) * C;
    float cur[DTW_BLOCK], nxt[DTW_BLOCK];
    auto load = [&](float (&buf)[DTW_BLOCK], int s0) {
#pragma unroll
        for (int u = 0; u < DTW_BLOCK; ++u) {
            const int j = s0 + u - i;
            buf[u] = mine && j >= 1 && j <= C ? -x[j - 1] : 0.0f;
        }
    };
    load(cur, 2);
    uint32_t word = 0;
    for (int s0 = 2; s0 <= N + C; s0 += DTW_BLOCK) {
        load(nxt, s0 + DTW_BLOCK);
#pragma unroll
        for (int u = 0; u < DTW_BLOCK; ++u) {
            const int s = s0 + u, j = s - i;
            if (s > N + C) break;
            if (mine && j >= 1 && j <= C) {
                const float* d1 = diag + ((s - 1) % 3) * DTW_DIAG;
                const float c0 = i == 1 ? (j == 1 ? 0.0f : INFINITY) : j == 1 ? INFINITY : diag[((s - 2) % 3) * DTW_DIAG + i - 1];
                const float c1 = i == 1 ? INFINITY : d1[i - 1];
                const float c2 = j == 1 ? INFINITY : d1[i];
                float c;
                const int code = dtw::pick(c0, c1, c2, c);
                diag[(s % 3) * DTW_DIAG + i] = __fadd_rn(cur[u], c);
                word |= (uint32_t)code << (2 * ((j - 1) & 15));
                if (((j - 1) & 15) == 15 || j == C) {
                    trace[(i - 1) * W + ((j - 1) >> 4)] = word;
                    word = 0;
                }
            }
            __syncthreads();   // three buffers: diagonal s - 2 is overwritten at s + 1, after this barrier
        }
#pragma unroll
        for (int u = 0; u < DTW_BLOCK; ++u) cur[u] = nxt[u];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        auto tr = [&](int ii, int jj) { return (int)((trace[(ii - 1) * W + ((jj - 1) >> 4)] >> (2 * ((jj - 1) & 15))) & 3u); };
        const int64_t o = out_off[blockIdx.x];
        dtw::backtrace(N, C, tr, start + o, end + o);
    }
}

PerDeviceConfig g_dtw_smem;

void launch_dtw(const float* mat, const AlignSeq* seqs_dev, const int64_t* out_off_dev, int n_seqs, int max_N, size_t smem, int* start,
                int* end, cudaStream_t st) {
    cudaError_t err = cudaSuccess;
    if (!g_dtw_smem.ensure(DTW_SMEM_MAX, [&] {
            err = cudaFuncSetAttribute(align_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DTW_SMEM_MAX);
            return err == cudaSuccess;
        })) {
        cudaGetLastError();
        fail(WB_ERR_CUDA, std::string("align DTW: the device refuses 227 KB of dynamic shared memory per CTA: ") + cudaGetErrorString(err));
    }
    const int threads = (max_N + 31) / 32 * 32;
    align_dtw_kernel<<<n_seqs, threads, smem, st>>>(mat, seqs_dev, out_off_dev, start, end);
    WB_LAUNCH_CHECK();
}

}  // namespace

bool dtw_fits(int64_t N, int64_t C) { return N >= 1 && N <= DTW_MAX_ROWS && C >= 1 && C <= INT32_MAX / 2 && dtw_smem(N, C) <= DTW_SMEM_MAX; }

void Session::align_tokens(int64_t n_seqs, const int32_t* window_of_seq, const int64_t* toks, const int64_t* lens, const int64_t* first,
                           int64_t n_heads, const int32_t* heads, int32_t* start_out, int32_t* end_out, float* matrix_out,
                           int64_t matrix_capacity) {
    if (!encoded) fail(WB_ERR_STATE, "align_tokens: no window encoded yet");
    const wb_dims& D = m->dims;
    const int d = D.n_text_state, H = D.n_text_head, L = D.n_text_layer, V = D.n_vocab;
    WB_REQUIRE(n_seqs >= 1, "align_tokens: n_seqs must be >= 1");
    std::vector<int64_t> off((size_t)n_seqs + 1, 0), aoff((size_t)n_seqs + 1, 0), moff((size_t)n_seqs + 1, 0);
    std::vector<int> cols((size_t)n_seqs);
    for (int64_t i = 0; i < n_seqs; ++i) {
        WB_REQUIRE(lens[i] >= 2 && lens[i] <= D.n_text_ctx, "align_tokens: sequence length outside [2, n_text_ctx]");
        WB_REQUIRE(first[i] >= 1 && first[i] <= lens[i] - 1, "align_tokens: first outside [1, len - 1]");
        WB_REQUIRE(window_of_seq[i] >= 0 && window_of_seq[i] < n_windows, "align_tokens: window outside the encoded ones");
        const int C = std::max(1, win_F[(size_t)window_of_seq[i]] / 2);   // openai: num_frames // 2
        cols[(size_t)i] = C;
        off[(size_t)i + 1] = off[(size_t)i] + lens[i];
        aoff[(size_t)i + 1] = aoff[(size_t)i] + lens[i] - first[i];
        moff[(size_t)i + 1] = moff[(size_t)i] + (lens[i] - first[i]) * C;
    }
    for (int64_t p = 0; p < off[(size_t)n_seqs]; ++p) WB_REQUIRE(toks[p] >= 0 && toks[p] < V, "align_tokens: token outside [0, n_vocab)");
    WB_REQUIRE(n_heads >= 0 && n_heads <= (int64_t)L * H, "align_tokens: n_heads outside [0, n_text_layer * n_text_head]");
    WB_REQUIRE(n_heads == 0 || heads, "align_tokens: null heads");
    std::vector<uint8_t> sel((size_t)L * H, 0);   // [layer][head]: selected
    for (int64_t k = 0; k < n_heads; ++k) {
        const int l = heads[2 * k], h = heads[2 * k + 1];
        WB_REQUIRE(l >= 0 && l < L && h >= 0 && h < H, "align_tokens: head outside the model");
        WB_REQUIRE(!sel[(size_t)l * H + h], "align_tokens: head listed twice");
        sel[(size_t)l * H + h] = 1;
    }
    if (n_heads == 0)   // openai's fallback: every head of the second half of the decoder layers
        for (int l = L / 2; l < L; ++l) std::fill(sel.begin() + (size_t)l * H, sel.begin() + (size_t)(l + 1) * H, 1);
    WB_REQUIRE(!matrix_out || matrix_capacity >= moff[(size_t)n_seqs], "align_tokens: matrix_capacity below the matrices' size");
    if (!m->fp16_exact) fail(WB_ERR_UNSUPPORTED, "align_tokens: the weights are not fp16-exact (the decoder pass runs on the tensor cores only)");
    for (int64_t i = 0; i < n_seqs; ++i)
        if (!dtw_fits(lens[i] - first[i], cols[(size_t)i]))
            fail(WB_ERR_UNSUPPORTED, "align_tokens: the DTW trace of a sequence does not fit one CTA's shared memory");

    // selected heads, ascending, by layer
    std::vector<int> hlist, hoff((size_t)L + 1, 0);
    int l_last = 0, n_total = 0, nh_max = 0;
    for (int l = 0; l < L; ++l) {
        for (int h = 0; h < H; ++h)
            if (sel[(size_t)l * H + h]) hlist.push_back(h);
        hoff[(size_t)l + 1] = (int)hlist.size();
        const int nh = hoff[(size_t)l + 1] - hoff[(size_t)l];
        if (nh) l_last = l;
        nh_max = std::max(nh_max, nh);
    }
    n_total = (int)hlist.size();
    ScoreWs& w = score_ws;
    AlignWs& a = align_ws;
    a.heads.ensure(hlist.size());
    WB_CUDA(cudaMemcpyAsync(a.heads.p, hlist.data(), hlist.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    const bool kv16 = kv_dtype == WB_KV_F16;

    for (int64_t s0 = 0; s0 < n_seqs;) {
        // ---- one group of whole sequences, every position a row
        int64_t s1 = s0, P = 0;
        while (s1 < n_seqs && (s1 == s0 || P + lens[s1] <= SCORE_GROUP_ROWS)) P += lens[s1++];
        const int n = (int)(s1 - s0);
        std::vector<int> tok((size_t)P), pos((size_t)P), win((size_t)n);
        std::vector<AttnWindow> aw((size_t)n);
        std::vector<AlignSeq> as((size_t)n);
        std::vector<int64_t> oo((size_t)n);
        int max_L = 0, max_N = 0, Cmax = 0;
        size_t smem = 0;
        for (int64_t i = s0, r = 0; i < s1; ++i) {
            const int Li = (int)lens[i], z = (int)(i - s0);
            aw[(size_t)z] = AttnWindow{r, Li};
            win[(size_t)z] = window_of_seq[i];
            as[(size_t)z] = AlignSeq{r, moff[(size_t)i] - moff[(size_t)s0], Li, (int)first[i], cols[(size_t)i], window_of_seq[i]};
            oo[(size_t)z] = aoff[(size_t)i] - aoff[(size_t)s0];
            max_L = std::max(max_L, Li);
            max_N = std::max(max_N, Li - (int)first[i]);
            Cmax = std::max(Cmax, cols[(size_t)i]);
            smem = std::max(smem, dtw_smem(Li - (int)first[i], cols[(size_t)i]));
            for (int j = 0; j < Li; ++j, ++r) {
                tok[(size_t)r] = (int)toks[off[(size_t)i] + j];
                pos[(size_t)r] = j;
            }
        }
        const int64_t n_mat = moff[(size_t)s1] - moff[(size_t)s0], n_ids = aoff[(size_t)s1] - aoff[(size_t)s0];
        w.tok.ensure((size_t)P); w.pos.ensure((size_t)P); w.seq_win.ensure((size_t)n); w.seqs.ensure((size_t)n);
        a.seqs.ensure((size_t)n); a.out_off.ensure((size_t)n); a.start.ensure((size_t)n_ids); a.end.ensure((size_t)n_ids);
        a.w.ensure((size_t)nh_max * P * Cmax); a.stats.ensure((size_t)nh_max * n * Cmax * 2); a.mat.ensure((size_t)n_mat);
        WB_CUDA(cudaMemcpyAsync(w.tok.p, tok.data(), tok.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.pos.p, pos.data(), pos.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.seq_win.p, win.data(), win.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.seqs.p, aw.data(), aw.size() * sizeof(AttnWindow), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(a.seqs.p, as.data(), as.size() * sizeof(AlignSeq), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(a.out_off.p, oo.data(), oo.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemsetAsync(a.mat.p, 0, (size_t)n_mat * sizeof(float), st));

        // ---- the pass, with the head weights of each layer that holds a selected head
        decoder_pass((int)P, n, max_L, l_last + 1, false, [&](int l) {
            const int nh = hoff[(size_t)l + 1] - hoff[(size_t)l];
            if (nh == 0) return;
            const int* hl = a.heads.p + hoff[(size_t)l];
            const dim3 qk_grid((max_L + TQ - 1) / TQ, nh, n);
            if (kv16)
                align_qk_kernel<__half><<<qk_grid, AQ_THREADS, 0, st>>>(w.qkv_h.p, w.qkv_l.p, ckv16.p + (size_t)l * Mcap * 2 * d, a.seqs.p, hl,
                                                                       d_win_row_off.p, d_win_T.p, d, P, Cmax, a.w.p);
            else
                align_qk_kernel<float><<<qk_grid, AQ_THREADS, 0, st>>>(w.qkv_h.p, w.qkv_l.p, ckv.p + (size_t)l * Mcap * 2 * d, a.seqs.p, hl,
                                                                      d_win_row_off.p, d_win_T.p, d, P, Cmax, a.w.p);
            WB_LAUNCH_CHECK();
            align_softmax_kernel<<<dim3((max_L + 7) / 8, nh, n), 256, 0, st>>>(a.seqs.p, P, Cmax, a.w.p);
            WB_LAUNCH_CHECK();
            align_stats_kernel<<<dim3((Cmax + 127) / 128, nh, n), 128, 0, st>>>(a.seqs.p, n, P, Cmax, a.w.p, a.stats.p);
            WB_LAUNCH_CHECK();
            align_filter_kernel<<<dim3((Cmax + 127) / 128, max_N, n), 128, 0, st>>>(a.seqs.p, n, nh, P, Cmax, a.w.p, a.stats.p, l == l_last,
                                                                                  n_total, a.mat.p);
            WB_LAUNCH_CHECK();
        });
        launch_dtw(a.mat.p, a.seqs.p, a.out_off.p, n, max_N, smem, a.start.p, a.end.p, st);

        WB_CUDA(cudaMemcpyAsync(start_out + aoff[(size_t)s0], a.start.p, (size_t)n_ids * sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(end_out + aoff[(size_t)s0], a.end.p, (size_t)n_ids * sizeof(int), cudaMemcpyDeviceToHost, st));
        if (matrix_out)
            WB_CUDA(cudaMemcpyAsync(matrix_out + moff[(size_t)s0], a.mat.p, (size_t)n_mat * sizeof(float), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaStreamSynchronize(st));   // the host vectors above are in flight until here
        s0 = s1;
    }
}

void align_dtw(const float* matrix, int64_t N, int64_t C, int32_t* start_out, int32_t* end_out) {
    DevBuf<float> mat;
    DevBuf<AlignSeq> seq;
    DevBuf<int64_t> oo;
    DevBuf<int> start, end;
    mat.alloc((size_t)(N * C)); seq.alloc(1); oo.alloc(1); start.alloc((size_t)N); end.alloc((size_t)N);
    const AlignSeq as{0, 0, (int)N + 1, 1, (int)C, 0};
    const int64_t zero = 0;
    WB_CUDA(cudaMemcpy(mat.p, matrix, (size_t)(N * C) * sizeof(float), cudaMemcpyHostToDevice));
    WB_CUDA(cudaMemcpy(seq.p, &as, sizeof(as), cudaMemcpyHostToDevice));
    WB_CUDA(cudaMemcpy(oo.p, &zero, sizeof(zero), cudaMemcpyHostToDevice));
    launch_dtw(mat.p, seq.p, oo.p, 1, (int)N, dtw_smem(N, C), start.p, end.p, nullptr);
    WB_CUDA(cudaMemcpy(start_out, start.p, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost));
    WB_CUDA(cudaMemcpy(end_out, end.p, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost));
}

}  // namespace wb
