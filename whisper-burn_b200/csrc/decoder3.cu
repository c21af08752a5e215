// Persistent cooperative decoder ("megakernel") for sm_90a.
//
// Reference math: TextDecoder::forward src/model/mod.rs:131-157, ResidualDecoderAttentionBlock::forward
// :345-350, MultiHead{Self,Cross}Attention::forward :428-436 / :482-490, qkv_attention :493-533,
// MLP::forward :376-382, and the search closure beamsearch_next src/transcribe.rs:253-307 (special-token
// mask :271-275, log_softmax :276); greedy = beam::beam_search with beam_size 1 (src/beam.rs:9-37).
//
// Why one kernel: at the batch sizes of this workload (3 rows for BASELINE configs[1]) a decoder step
// is ~60 MB of L2-resident weight/KV traffic but a chain of ~35 dependent stages; as separate kernels
// each stage costs a launch + drain + cold prologue (measured 10-35 us each, profiles/).  Here ONE
// cooperative launch (one CTA per SM, all co-resident) runs prompt prefill and every greedy step; the
// stages are separated by a grid barrier (atomic arrive + generation flag in L2, ~1 us) and every stage
// spreads its output features over all warps of the grid (weight-slice GEMV: a warp owns whole output
// features, reads each weight row once for all rows of the batch, fp32 accumulate, no cross-CTA
// reduction).  Per layer: LN+QKV | self-attention | out-proj+residual | LN+Q | cross-attention (split
// over keys) | merge+out-proj+residual | LN+MLP1+GELU | MLP2+residual; then LN+logits with fused
// special-token mask / online softmax / top-k candidates per warp, and a per-row finish.
//
// Everything another CTA wrote during the launch is read with ld.global.cg (L2), never through L1.
#include <cooperative_groups.h>

#include "dec_common.cuh"

namespace wb {

namespace {

// =====================================================================================================
template <typename WT, int RC, int KC, typename KVT>
__global__ void __launch_bounds__(NT, 1)
dec3_kernel(const DecArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int d = a.d, H = a.H, L = a.L, V = a.V, R = a.R, t_max = a.t_max;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gw = blockIdx.x * NW + warp, n_gw = gridDim.x * NW;
    float* xs = sm;                         // [RC][4d] staged activations
    float* qs = xs + RC * 4 * d;            // [64] query of the current attention unit
    float* wm = qs + 64;                    // [NW]
    float* wl = wm + NW;                    // [NW]
    float* wo = wl + NW;                    // [NW][64]
    float* ao = wo + NW * 64;               // [64]
    float* ML = ao + 64;                    // [2]
    float* red = ML + 2;                    // logits merge scratch: [NW][RC][2 + 2*KC]; also cross merge weights
    unsigned int gen = 0;
    int tr_n = 0;
    WB_TRACE();
    const float scale = a.qk_scale;
    const int S = a.n_splits;

    for (int step = 0; step < a.n_steps; ++step) {
        const int p = a.pos0 + step;
        const bool want_logits = p >= a.logits_from;
        // embed: x[r] = tok_emb[token] + pos_emb[p] (mod.rs:141-146) is formed by EVERY CTA in shared memory for
        // the first LayerNorm (no extra barrier); rows are published to a.x by the CTAs r % grid for the residual adds.
        for (int l = 0; l < L; ++l) {
            const DecLayer& W = a.layers[l];
            KVT* kcl = reinterpret_cast<KVT*>(a.kc) + (size_t)l * a.Rmax * t_max * d;
            KVT* vcl = reinterpret_cast<KVT*>(a.vc) + (size_t)l * a.Rmax * t_max * d;
            // ================= P1: q | k | v = LN(x) Wqkv + b   (mod.rs:429-431)
            for (int r0 = 0; r0 < R; r0 += RC) {
                if (l == 0) {
                    float* emb_s = xs + RC * d;   // scratch behind the LN rows (xs holds RC*4d floats)
                    int* tok_s = reinterpret_cast<int*>(wm);
                    if (tid < RC) tok_s[tid] = (r0 + tid < R) ? (a.use_cur_tok ? __ldcg(a.cur_tok + r0 + tid)
                                                                               : __ldcg(a.tokens + (int64_t)(r0 + tid) * t_max + p)) : 0;
                    __syncthreads();
                    const float* pe = a.pos_emb + (int64_t)p * d;
                    for (int i = tid; i < RC * d / 4; i += NT) {   // all rows' embedding loads are independent
                        const int rr = (i * 4) / d, c = (i * 4) % d, r = r0 + rr;
                        if (r >= R) continue;
                        const float4 e4 = __ldg(reinterpret_cast<const float4*>(a.tok_emb + (int64_t)tok_s[rr] * d + c));
                        const float4 p4 = __ldg(reinterpret_cast<const float4*>(pe + c));
                        const float4 v = make_float4(__fadd_rn(e4.x, p4.x), __fadd_rn(e4.y, p4.y), __fadd_rn(e4.z, p4.z), __fadd_rn(e4.w, p4.w));
                        *reinterpret_cast<float4*>(emb_s + rr * d + c) = v;
                        if (r % gridDim.x == blockIdx.x) *reinterpret_cast<float4*>(a.x + (int64_t)r * d + c) = v;
                    }
                    __syncthreads();
                    stage_ln_smem<RC>(emb_s, r0, R, d, W.ln1_g, W.ln1_b, W.ln1_eps, a.eps_outside, xs);
                } else {
                    stage_ln<RC>(a.x, r0, R, d, W.ln1_g, W.ln1_b, W.ln1_eps, a.eps_outside, xs);
                }
                __syncthreads();
                gemv_phase<WT, RC>(reinterpret_cast<const WT*>(W.Wqkv), 3 * d, d, xs, gw, n_gw, [&](int n, const float (&acc)[RC]) {
                    if (lane < RC && r0 + lane < R) {
                        const int r = r0 + lane;
                        float v = __fadd_rn(pick_row<RC>(acc, lane), __ldg(W.bqkv + n));
                        if (n < 2 * d) v = __fmul_rn(v, scale);
                        if (n < d) a.q[(int64_t)r * d + n] = v;
                        else if (n < 2 * d) kcl[((int64_t)r * t_max + p) * d + (n - d)] = (KVT)v;     // fp16 cache: round-to-nearest
                        else vcl[((int64_t)r * t_max + p) * d + (n - 2 * d)] = (KVT)v;
                    }
                });
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P2: self attention over positions 0..p of the row's ancestry (mask == causal)
            for (int u = blockIdx.x; u < R * H; u += gridDim.x) {
                const int r = u / H, h = u % H;
                if (tid < 16) *reinterpret_cast<float4*>(qs + tid * 4) = __ldcg(reinterpret_cast<const float4*>(a.q + (int64_t)r * d + h * 64) + tid);
                __syncthreads();
                const int* anc = a.anc ? a.anc + (int64_t)r * t_max : nullptr;
                const KVT* kb = kcl + h * 64;
                const KVT* vb = vcl + h * 64;
                auto kp = [&](int j) { return kb + ((int64_t)((anc && j < p) ? __ldcg(anc + j) : r) * t_max + j) * d; };
                auto vp = [&](int j) { return vb + ((int64_t)((anc && j < p) ? __ldcg(anc + j) : r) * t_max + j) * d; };
                attn_cta(qs, p + 1, kp, vp, wm, wl, wo, ao, ML);
                if (tid < 64) a.att[(int64_t)r * d + h * 64 + tid] = __fdiv_rn(ao[tid], ML[1]);
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P3: x += att Wo + bo   (mod.rs:435, :346)
            for (int r0 = 0; r0 < R; r0 += RC) {
                stage_copy<RC>(a.att, r0, R, d, xs);
                __syncthreads();
                gemv_phase<WT, RC>(reinterpret_cast<const WT*>(W.Wo), d, d, xs, gw, n_gw, [&](int n, const float (&acc)[RC]) {
                    if (lane < RC && r0 + lane < R) {
                        float* xp = a.x + (int64_t)(r0 + lane) * d + n;
                        *xp = __fadd_rn(__ldcg(xp), __fadd_rn(pick_row<RC>(acc, lane), __ldg(W.bo + n)));
                    }
                });
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P4: cross query = LN(x) Wq + b   (mod.rs:483)
            for (int r0 = 0; r0 < R; r0 += RC) {
                stage_ln<RC>(a.x, r0, R, d, W.ln2_g, W.ln2_b, W.ln2_eps, a.eps_outside, xs);
                __syncthreads();
                gemv_phase<WT, RC>(reinterpret_cast<const WT*>(W.Wcq), d, d, xs, gw, n_gw, [&](int n, const float (&acc)[RC]) {
                    if (lane < RC && r0 + lane < R)
                        a.q[(int64_t)(r0 + lane) * d + n] = __fmul_rn(__fadd_rn(pick_row<RC>(acc, lane), __ldg(W.bcq + n)), scale);
                });
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P5: cross attention, split over the window's encoder positions (K/V projected once per window)
            {
                const KVT* ckvl = reinterpret_cast<const KVT*>(a.ckv) + (size_t)l * a.Mcap * 2 * d;
                for (int u = blockIdx.x; u < R * H * S; u += gridDim.x) {
                    const int sp = u % S, h = (u / S) % H, r = u / (S * H);
                    if (tid < 16) *reinterpret_cast<float4*>(qs + tid * 4) = __ldcg(reinterpret_cast<const float4*>(a.q + (int64_t)r * d + h * 64) + tid);
                    __syncthreads();
                    const int w = __ldcg(a.row_window + r);
                    const int T = a.win_T[w];
                    const int per = (T + S - 1) / S;
                    const int kb0 = sp * per;
                    const int nk = max(0, min(T, kb0 + per) - kb0);
                    const KVT* kbase = ckvl + a.win_row_off[w] * (int64_t)(2 * d) + ((int64_t)h * T + kb0) * 128;   // head-major K | V rows
                    auto kp = [&](int j) { return kbase + j * 128; };
                    auto vp = [&](int j) { return kbase + j * 128 + 64; };
                    attn_cta(qs, nk, kp, vp, wm, wl, wo, ao, ML, kb0);
                    const int64_t o = ((int64_t)r * H + h) * S + sp;
                    if (tid < 64) a.part_o[o * 64 + tid] = ao[tid];
                    if (tid == 0) { a.part_m[o] = nk > 0 ? ML[0] : -INFINITY; a.part_l[o] = ML[1]; }
                    __syncthreads();
                }
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P6: x += merge(cross partials) Wo + bo   (mod.rs:489, :347)
            for (int r0 = 0; r0 < R; r0 += RC) {
                float* wn = red;   // [RC][H][S] normalised split weights
                for (int i = tid; i < RC * H; i += NT) {
                    const int rr = i / H, h = i % H, r = r0 + rr;
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
                for (int i = tid; i < RC * d / 4; i += NT) {   // 4 consecutive dims of one (row, head)
                    const int rr = (i * 4) / d, c = (i * 4) % d, r = min(r0 + rr, R - 1);
                    const int h = c / 64;
                    const float4* po = reinterpret_cast<const float4*>(a.part_o + (((int64_t)r * H + h) * S) * 64 + (c & 63));
                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
                    for (int s = 0; s < S; ++s) {
                        const float4 v = __ldcg(po + s * 16);
                        const float wgt = wn[(rr * H + h) * S + s];
                        acc.x = fmaf(wgt, v.x, acc.x); acc.y = fmaf(wgt, v.y, acc.y);
                        acc.z = fmaf(wgt, v.z, acc.z); acc.w = fmaf(wgt, v.w, acc.w);
                    }
                    *reinterpret_cast<float4*>(xs + rr * d + c) = acc;
                }
                __syncthreads();
                gemv_phase<WT, RC>(reinterpret_cast<const WT*>(W.Wco), d, d, xs, gw, n_gw, [&](int n, const float (&acc)[RC]) {
                    if (lane < RC && r0 + lane < R) {
                        float* xp = a.x + (int64_t)(r0 + lane) * d + n;
                        *xp = __fadd_rn(__ldcg(xp), __fadd_rn(pick_row<RC>(acc, lane), __ldg(W.bco + n)));
                    }
                });
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P7: hid = gelu(LN(x) W1 + b1)   (mod.rs:377-378)
            for (int r0 = 0; r0 < R; r0 += RC) {
                stage_ln<RC>(a.x, r0, R, d, W.ln3_g, W.ln3_b, W.ln3_eps, a.eps_outside, xs);
                __syncthreads();
                gemv_phase<WT, RC>(reinterpret_cast<const WT*>(W.W1), 4 * d, d, xs, gw, n_gw, [&](int n, const float (&acc)[RC]) {
                    if (lane < RC && r0 + lane < R)
                        a.hid[(int64_t)(r0 + lane) * 4 * d + n] = gelu_erf(__fadd_rn(pick_row<RC>(acc, lane), __ldg(W.b1 + n)));
                });
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= P8: x += hid W2 + b2   (mod.rs:379, :348)
            for (int r0 = 0; r0 < R; r0 += RC) {
                stage_copy<RC>(a.hid, r0, R, 4 * d, xs);
                __syncthreads();
                gemv_phase<WT, RC>(reinterpret_cast<const WT*>(W.W2), d, 4 * d, xs, gw, n_gw, [&](int n, const float (&acc)[RC]) {
                    if (lane < RC && r0 + lane < R) {
                        float* xp = a.x + (int64_t)(r0 + lane) * d + n;
                        *xp = __fadd_rn(__ldcg(xp), __fadd_rn(pick_row<RC>(acc, lane), __ldg(W.b2 + n)));
                    }
                });
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
        }
        if (want_logits) {
            // ================= logits = LN(x) tok_emb^T (mod.rs:155-156) + mask + online softmax + candidates.
            // 8 lanes per vocabulary row, 8 rows per warp step; lane (sub, l8) tracks batch row l8.
            const bool use_mask = SPECIAL_MASKED(a, p);
            const int eot_cap = a.loop_rules ? a.eot : -1;   // the id whose logit the greedy loop's EOT test reads
            const WT* E = reinterpret_cast<const WT*>(a.E);
            const int sub = lane >> 3, l8 = lane & 7;
            for (int r0 = 0; r0 < R; r0 += RC) {
                stage_ln<RC>(a.x, r0, R, d, a.lnf_g, a.lnf_b, a.lnf_eps, a.eps_outside, xs);
                __syncthreads();
                float m_run = -INFINITY, s_run = 0.0f;
                Cand<KC> cand;
                cand.init();
                const int n_blk = (V + 7) / 8;
                for (int blk = gw; blk < n_blk; blk += n_gw) {
                    const int n0 = blk * 8;
                    const WT* rows[2];
                    int nn[2];
#pragma unroll
                    for (int g = 0; g < 2; ++g) {
                        nn[g] = n0 + g * 4 + sub;
                        rows[g] = E + (int64_t)min(nn[g], V - 1) * d;
                    }
                    float acc[2][RC];
                    dot_groups<WT, RC, 2>(rows, xs, d, acc);
                    if (l8 < RC && r0 + l8 < R) {
#pragma unroll
                        for (int g = 0; g < 2; ++g) {
                            if (nn[g] < V) {
                                const float raw = pick_row<RC>(acc[g], l8);
                                if (a.logits_out) a.logits_out[(int64_t)(r0 + l8) * V + nn[g]] = raw;
                                const float v = (use_mask && a.is_special[nn[g]]) ? __fadd_rn(raw, -INFINITY) : raw;
                                if (v > -INFINITY) softmax_add(m_run, s_run, v);
                                cand.push(v, nn[g]);
                                if (nn[g] == eot_cap) a.eot_logit[r0 + l8] = v;
                            }
                        }
                    }
                }
                // merge: 4 sub-groups x 8 warps hold a state for every batch row -> one record per (CTA, row)
                if (l8 < RC) {
                    float* rec = red + ((warp * 4 + sub) * RC + l8) * (2 + 2 * KC);
                    rec[0] = m_run;
                    rec[1] = s_run;
#pragma unroll
                    for (int k = 0; k < KC; ++k) { rec[2 + k] = cand.v[k]; rec[2 + KC + k] = __int_as_float(cand.i[k]); }
                }
                __syncthreads();
                if (tid < RC && r0 + tid < R)
                    fold_records<KC>(a, red + tid * (2 + 2 * KC), NW * 4, RC * (2 + 2 * KC), KC, (int64_t)blockIdx.x * R + r0 + tid);
                __syncthreads();
            }
            WB_TRACE();
        grid_sync(a.bar, gen);
        WB_TRACE();
            // ================= finish: log_softmax of the candidates, k best, greedy bookkeeping
            for (int r = blockIdx.x; r < R; r += gridDim.x) finish_row_topk<KC>(a, r, p, gridDim.x, wm, reinterpret_cast<int*>(wl));
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

size_t dec3_smem_bytes(int d, int H, int S, int RC, int KC) {
    size_t red = std::max((size_t)NW * 4 * RC * (2 + 2 * KC), (size_t)RC * H * S);
    return sizeof(float) * ((size_t)RC * 4 * d + 64 + 2 * NW + NW * 64 + 64 + 2 + red + 8);
}

template <typename WT, int RC, int KC, typename KVT>
void launch_t(const DecArgs& a, int n_ctas, cudaStream_t st) {
    const size_t smem = dec3_smem_bytes(a.d, a.H, a.n_splits, RC, KC);
    auto k = dec3_kernel<WT, RC, KC, KVT>;
    static PerDeviceConfig cfg;   // per instantiation
    cfg.ensure(smem, [&] {
        WB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int per_sm = 0;
        WB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, NT, smem));
        if (per_sm < 1) fail(WB_ERR_UNSUPPORTED, "decoder megakernel does not fit on an SM");
        return true;
    });
    void* args[] = {(void*)&a};
    WB_CUDA(cudaLaunchCooperativeKernel((void*)k, dim3(n_ctas), dim3(NT), args, smem, st));
    WB_LAUNCH_CHECK();
}

}  // namespace

void launch_dec3(const DecArgs& a, int n_ctas, bool w_half, cudaStream_t st) {
    const bool big = a.R > 4;
    const bool wide = a.k > 1;
#define WB_D3(WT)                                                        \
    do {                                                                 \
        if (a.kv_half) {                                                 \
            if (!big && !wide) launch_t<WT, 4, 2, __half>(a, n_ctas, st);        \
            else if (!big && wide) launch_t<WT, 4, 8, __half>(a, n_ctas, st);    \
            else if (big && !wide) launch_t<WT, 8, 2, __half>(a, n_ctas, st);    \
            else launch_t<WT, 8, 8, __half>(a, n_ctas, st);                      \
        } else {                                                         \
            if (!big && !wide) launch_t<WT, 4, 2, float>(a, n_ctas, st);         \
            else if (!big && wide) launch_t<WT, 4, 8, float>(a, n_ctas, st);     \
            else if (big && !wide) launch_t<WT, 8, 2, float>(a, n_ctas, st);     \
            else launch_t<WT, 8, 8, float>(a, n_ctas, st);                       \
        }                                                                \
    } while (0)
    if (w_half) WB_D3(__half);
    else WB_D3(float);
#undef WB_D3
}

}  // namespace wb
