// Teacher-forced token scoring (wb_session_score_tokens): Whisper::forward_decoder (mod.rs:131-157) and log_softmax
// (transcribe.rs:276) at every position of many token sequences, against windows the session has encoded.
//
// Every input token is known up front, so unlike the persistent decoders (one position per step, latency-bound GEMVs) this
// pass runs all positions of all sequences at once: the packed rows of the sequences are the M dimension of tensor-core GEMMs,
// as the encoder's windows are.  Row p of sequence i is its position j; only positions 0 .. len - 2 are rows, since the last
// position's logits predict nothing and, the self attention being causal, no earlier position reads it.
//   embed (score_embed_kernel) -> per layer: attn_ln -> q|k|v GEMM -> causal self attention -> out GEMM + residual ->
//   cross_attn_ln -> cross-query GEMM -> cross attention over the window's cached cross K/V -> cross-out GEMM + residual ->
//   mlp_ln -> mlp1 (GELU) -> mlp2 + residual -> final LayerNorm -> logits GEMM with the statistics epilogue ->
//   score_combine_kernel: log-prob of each row's target and its arg-max.
// decoder_pass (embed and the layer loop) is shared with token alignment (align.cu), which builds a row for every position and
// stops after the cross-query GEMM of the last layer it reads.
// Numerics as the encoder's (DESIGN.md section 3): fp32 activations travel as fp16 hi/lo planes into fp16-exact weights, fp32
// accumulation; the self and cross K/V of WB_KV_F16 sessions enter as their fp16 rounding, as in the persistent decoders.
#include <climits>
#include <cmath>

#include "session.h"

namespace wb {

namespace {

// x[r] = tok_emb[token] + pos_emb[position]  (mod.rs:141-146), f32 add
__global__ void score_embed_kernel(const int* __restrict__ tok, const int* __restrict__ pos, const float* __restrict__ tok_emb,
                                   const float* __restrict__ pos_emb, float* __restrict__ x, int rows, int d) {
    const int64_t n4 = (int64_t)rows * d / 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(i * 4 / d), c = (int)(i * 4 % d);
        const float4 e = __ldg(reinterpret_cast<const float4*>(tok_emb + (int64_t)tok[r] * d + c));
        const float4 p = __ldg(reinterpret_cast<const float4*>(pos_emb + (int64_t)pos[r] * d + c));
        reinterpret_cast<float4*>(x)[i] = make_float4(__fadd_rn(e.x, p.x), __fadd_rn(e.y, p.y), __fadd_rn(e.z, p.z), __fadd_rn(e.w, p.w));
    }
}

// One warp per row: the tile statistics of the logits GEMM -> (x_t - M) - log(sum_k s_k exp(m_k - M)) and the arg-max (tiles
// cover ascending id ranges, so the lowest id among equal tile maxima is the lowest id overall)
__global__ void score_combine_kernel(const float* __restrict__ tile_m, const float* __restrict__ tile_s, const int* __restrict__ tile_i,
                                     const float* __restrict__ tgt_logit, const int* __restrict__ target, const uint8_t* __restrict__ row_mask,
                                     const uint8_t* __restrict__ is_special, int n_tiles, int rows, float* __restrict__ lp, int* __restrict__ am) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    float M = -INFINITY, S = 0.0f;
    int bi = INT_MAX;
    for (int k = lane; k < n_tiles; k += 32) {
        const int64_t o = (int64_t)row * n_tiles + k;
        const float m = tile_m[o], s = tile_s[o];
        if (m > M) { S = S * expf(M - m) + s; M = m; bi = tile_i[o]; }
        else if (m > -INFINITY) S += s * expf(m - M);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        const float oM = __shfl_xor_sync(0xffffffffu, M, o), oS = __shfl_xor_sync(0xffffffffu, S, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oM > M) { S = S * expf(M - oM) + oS; M = oM; bi = oi; }
        else if (oM > -INFINITY) { S += oS * expf(oM - M); if (oM == M && oi < bi) bi = oi; }
    }
    if (lane == 0) {
        const int t = target[row];
        const bool excluded = row_mask != nullptr && row_mask[row] && is_special[t];   // transcribe.rs:271-275
        lp[row] = excluded ? -INFINITY : __fsub_rn(__fsub_rn(tgt_logit[row], M), logf(S));
        am[row] = bi;
    }
}

}  // namespace

void Session::decoder_pass(int M, int n, int max_T, int n_layers, bool full, const std::function<void(int)>& after_cross_query) {
    const wb_dims& D = m->dims;
    const int d = D.n_text_state, H = D.n_text_head, L = D.n_text_layer;
    const bool kv16 = kv_dtype == WB_KV_F16;
    ScoreWs& w = score_ws;
    if (w.plans.empty()) {
        w.plans.resize((size_t)6 * L);
        for (auto& pl : w.plans) pl.reset(new GemmF16Plan());
    }
    auto gemm = [&](size_t site, const GemmF16Params& p) {
        GemmF16Plan& pl = *w.plans[site];
        pl.build(p, 0, p.max_rows);   // the workspace may have moved since the last call
        pl.launch(st);
    };
    const size_t Pd = (size_t)M * d;
    w.x.ensure(Pd); w.xn_h.ensure(Pd); w.xn_l.ensure(Pd); w.att_h.ensure(Pd); w.att_l.ensure(Pd);
    w.qkv_h.ensure(3 * Pd); w.qkv_l.ensure(3 * Pd); w.hid_h.ensure(4 * Pd); w.hid_l.ensure(4 * Pd);

    const float qk_scale = (float)std::pow((double)d / (double)H, -0.25);   // mod.rs:503
    {
        const int64_t n4 = (int64_t)M * d / 4;
        score_embed_kernel<<<(int)std::min<int64_t>((n4 + 255) / 256, 132 * 8), 256, 0, st>>>(w.tok.p, w.pos.p, m->tok_emb32, m->dec_pos, w.x.p, M, d);
        WB_LAUNCH_CHECK();
    }
    for (int l = 0; l < n_layers; ++l) {
        const DecBlockW& B = m->dec[(size_t)l];
        const size_t site = (size_t)6 * l;
        GemmF16Params p;
        // x = x + attn(attn_ln(x), causal mask)   (mod.rs:345, 428-436)
        launch_layernorm(w.x.p, nullptr, w.xn_h.p, w.xn_l.p, B.attn_ln, M, d, m->ln_eps_outside, st);
        p.A_hi = w.xn_h.p; p.A_lo = w.xn_l.p; p.lda = d; p.B = B.qkv.w16; p.P_hi = w.qkv_h.p; p.P_lo = w.qkv_l.p; p.ldc = 3 * d;
        p.N = 3 * d; p.K = d; p.bias = B.qkv.b; p.scale = qk_scale; p.scale_cols = 2 * d; p.max_rows = M;
        gemm(site, p);
        launch_causal_attention_tc(w.qkv_h.p, w.qkv_l.p, w.att_h.p, w.att_l.p, w.seqs.p, n, max_T, d, H, kv16, st);
        p = GemmF16Params{};
        p.A_hi = w.att_h.p; p.A_lo = w.att_l.p; p.lda = d; p.B = B.out.w16; p.C = w.x.p; p.ldc = d; p.N = d; p.K = d;
        p.bias = B.out.b; p.residual = w.x.p; p.max_rows = M;
        gemm(site + 1, p);
        // x = x + cross_attn(cross_attn_ln(x), xa)   (mod.rs:347, 482-490); K/V: the window's cached head-major block
        launch_layernorm(w.x.p, nullptr, w.xn_h.p, w.xn_l.p, B.cross_ln, M, d, m->ln_eps_outside, st);
        p = GemmF16Params{};
        p.A_hi = w.xn_h.p; p.A_lo = w.xn_l.p; p.lda = d; p.B = B.cq.w16; p.P_hi = w.qkv_h.p; p.P_lo = w.qkv_l.p; p.ldc = d;
        p.N = d; p.K = d; p.bias = B.cq.b; p.scale = qk_scale; p.scale_cols = d; p.max_rows = M;
        gemm(site + 2, p);
        if (after_cross_query) after_cross_query(l);
        if (!full && l == n_layers - 1) break;
        const void* ckv_l = kv16 ? (const void*)(ckv16.p + (size_t)l * Mcap * 2 * d) : (const void*)(ckv.p + (size_t)l * Mcap * 2 * d);
        launch_cross_attention_tc(w.qkv_h.p, w.qkv_l.p, ckv_l, kv16, w.att_h.p, w.att_l.p, w.seqs.p, w.seq_win.p, d_win_row_off.p,
                                  d_win_T.p, n, max_T, d, H, st);
        p = GemmF16Params{};
        p.A_hi = w.att_h.p; p.A_lo = w.att_l.p; p.lda = d; p.B = B.cout.w16; p.C = w.x.p; p.ldc = d; p.N = d; p.K = d;
        p.bias = B.cout.b; p.residual = w.x.p; p.max_rows = M;
        gemm(site + 3, p);
        // x = x + mlp(mlp_ln(x))   (mod.rs:348, 376-382)
        launch_layernorm(w.x.p, nullptr, w.xn_h.p, w.xn_l.p, B.mlp_ln, M, d, m->ln_eps_outside, st);
        p = GemmF16Params{};
        p.A_hi = w.xn_h.p; p.A_lo = w.xn_l.p; p.lda = d; p.B = B.mlp1.w16; p.P_hi = w.hid_h.p; p.P_lo = w.hid_l.p; p.ldc = 4 * d;
        p.N = 4 * d; p.K = d; p.bias = B.mlp1.b; p.act = ACT_GELU; p.max_rows = M;
        gemm(site + 4, p);
        p = GemmF16Params{};
        p.A_hi = w.hid_h.p; p.A_lo = w.hid_l.p; p.lda = 4 * d; p.B = B.mlp2.w16; p.C = w.x.p; p.ldc = d; p.N = d; p.K = 4 * d;
        p.bias = B.mlp2.b; p.residual = w.x.p; p.max_rows = M;
        gemm(site + 5, p);
    }
}

void Session::score_tokens(int64_t n_seqs, const int32_t* window_of_seq, const int64_t* toks, const int64_t* lens, bool apply_mask,
                           const uint8_t* is_special_host, float* lp_out, int64_t* argmax_out) {
    if (!encoded) fail(WB_ERR_STATE, "score_tokens: no window encoded yet");
    const wb_dims& D = m->dims;
    const int d = D.n_text_state, L = D.n_text_layer, V = D.n_vocab;
    WB_REQUIRE(n_seqs >= 1, "score_tokens: n_seqs must be >= 1");
    WB_REQUIRE(!apply_mask || is_special_host, "score_tokens: apply_special_mask needs is_special");
    std::vector<int64_t> off((size_t)n_seqs + 1, 0);
    for (int64_t i = 0; i < n_seqs; ++i) {
        WB_REQUIRE(lens[i] >= 1 && lens[i] <= D.n_text_ctx, "score_tokens: sequence length outside [1, n_text_ctx]");
        WB_REQUIRE(window_of_seq[i] >= 0 && window_of_seq[i] < n_windows, "score_tokens: window outside the encoded ones");
        off[(size_t)i + 1] = off[(size_t)i] + lens[i];
    }
    for (int64_t p = 0; p < off[(size_t)n_seqs]; ++p) WB_REQUIRE(toks[p] >= 0 && toks[p] < V, "score_tokens: token outside [0, n_vocab)");
    if (!m->fp16_exact) fail(WB_ERR_UNSUPPORTED, "score_tokens: the weights are not fp16-exact (the scoring pass runs on the tensor cores only)");

    const int n_tiles = logit_stats_tiles(V);
    ScoreWs& w = score_ws;
    if (apply_mask) {
        w.special.ensure((size_t)V);
        WB_CUDA(cudaMemcpyAsync(w.special.p, is_special_host, (size_t)V, cudaMemcpyHostToDevice, st));
    }

    for (int64_t s0 = 0; s0 < n_seqs;) {
        // ---- one group of whole sequences: host descriptors of its rows
        int64_t s1 = s0, P = 0;
        while (s1 < n_seqs && (s1 == s0 || P + lens[s1] - 1 <= SCORE_GROUP_ROWS)) P += lens[s1++] - 1;
        const int n = (int)(s1 - s0);
        std::vector<int> tok((size_t)P), pos((size_t)P), tgt((size_t)P), win((size_t)n);
        std::vector<uint8_t> rmask((size_t)P);
        std::vector<AttnWindow> seqs((size_t)n);
        int max_T = 0;
        for (int64_t i = s0, r = 0; i < s1; ++i) {
            const int T = (int)lens[i] - 1;
            seqs[(size_t)(i - s0)] = AttnWindow{r, T};
            win[(size_t)(i - s0)] = window_of_seq[i];
            max_T = std::max(max_T, T);
            for (int j = 0; j < T; ++j, ++r) {
                tok[(size_t)r] = (int)toks[off[(size_t)i] + j];
                tgt[(size_t)r] = (int)toks[off[(size_t)i] + j + 1];
                pos[(size_t)r] = j;
                rmask[(size_t)r] = apply_mask && j + 1 <= 5 ? 1 : 0;   // the prefix of target j + 1 has j + 1 <= 5 tokens
            }
        }
        for (int64_t i = s0; i < s1; ++i) { lp_out[off[(size_t)i]] = 0.0f; if (argmax_out) argmax_out[off[(size_t)i]] = -1; }
        if (P == 0) { s0 = s1; continue; }

        // ---- workspace
        w.tok.ensure((size_t)P); w.pos.ensure((size_t)P); w.target.ensure((size_t)P); w.am.ensure((size_t)P);
        w.row_mask.ensure((size_t)P); w.seq_win.ensure((size_t)n); w.seqs.ensure((size_t)n);
        w.tgt_logit.ensure((size_t)P); w.lp.ensure((size_t)P);
        w.tile_m.ensure((size_t)P * n_tiles); w.tile_s.ensure((size_t)P * n_tiles); w.tile_i.ensure((size_t)P * n_tiles);
        WB_CUDA(cudaMemcpyAsync(w.tok.p, tok.data(), tok.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.pos.p, pos.data(), pos.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.target.p, tgt.data(), tgt.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.row_mask.p, rmask.data(), rmask.size(), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.seq_win.p, win.data(), win.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaMemcpyAsync(w.seqs.p, seqs.data(), seqs.size() * sizeof(AttnWindow), cudaMemcpyHostToDevice, st));

        // ---- the pass
        const int M = (int)P;
        decoder_pass(M, n, max_T, L, true, nullptr);
        // logits = ln(x) tok_emb^T (mod.rs:153-156), reduced to per-tile statistics, then combined per row
        launch_layernorm(w.x.p, nullptr, w.xn_h.p, w.xn_l.p, m->dec_ln, M, d, m->ln_eps_outside, st);
        LogitStatsParams lsp;
        lsp.A_hi = w.xn_h.p; lsp.A_lo = w.xn_l.p; lsp.E = m->tok_emb16; lsp.rows = M; lsp.K = d; lsp.V = V;
        lsp.target = w.target.p; lsp.row_mask = apply_mask ? w.row_mask.p : nullptr; lsp.is_special = w.special.p;
        lsp.tile_m = w.tile_m.p; lsp.tile_s = w.tile_s.p; lsp.tile_i = w.tile_i.p; lsp.tgt_logit = w.tgt_logit.p;
        launch_logit_stats(lsp, st);
        score_combine_kernel<<<(M + 7) / 8, 256, 0, st>>>(w.tile_m.p, w.tile_s.p, w.tile_i.p, w.tgt_logit.p, w.target.p,
                                                          apply_mask ? w.row_mask.p : nullptr, w.special.p, n_tiles, M, w.lp.p, w.am.p);
        WB_LAUNCH_CHECK();

        std::vector<float> lp((size_t)P);
        std::vector<int> am((size_t)P);
        WB_CUDA(cudaMemcpyAsync(lp.data(), w.lp.p, lp.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(am.data(), w.am.p, am.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaStreamSynchronize(st));   // the host vectors above are in flight until here
        for (int64_t i = s0, r = 0; i < s1; ++i)
            for (int64_t j = 1; j < lens[i]; ++j, ++r) {
                lp_out[off[(size_t)i] + j] = lp[(size_t)r];
                if (argmax_out) argmax_out[off[(size_t)i] + j] = am[(size_t)r];
            }
        s0 = s1;
    }
}

}  // namespace wb
