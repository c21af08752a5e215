// Session: device buffers + the launch sequences of the hot path
//   prep_audio (audio.rs:34-56) -> mel padding (transcribe.rs:161-177) -> forward_encoder
//   (mod.rs:228-260) -> cross K/V (mod.rs:484-485, hoisted out of the step loop) -> decoder steps.
// Windows of one call are batched: encoder rows of all windows are packed back to back.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "session.h"

namespace wb {

int window_mel_frames(int n_audio_ctx, int window_mode) {
    WB_REQUIRE(window_mode == WB_WINDOWS_REFERENCE || window_mode == WB_WINDOWS_NATIVE,
               "window_mode must be WB_WINDOWS_REFERENCE or WB_WINDOWS_NATIVE");
    return window_mode == WB_WINDOWS_NATIVE ? 2 * n_audio_ctx : n_audio_ctx;
}

int64_t window_samples(int n_audio_ctx, int window_mode) {
    return wb_max_waveform_samples(window_mel_frames(n_audio_ctx, window_mode) - MEL_PADDING);   // transcribe.rs:32-34
}

Session::Session(Model* model, int64_t max_w, int64_t max_b, int64_t max_text_len, int kv, int mode) : m(model) {
    if (!m || !m->finalized) fail(WB_ERR_STATE, "session: model not finalized");
    const wb_dims& D = m->dims;
    WB_REQUIRE(max_w >= 1 && max_b >= 1 && max_w * max_b <= 4096, "session: bad max_windows / max_beams");
    WB_REQUIRE(max_text_len >= 2 && max_text_len <= D.n_text_ctx, "session: max_text_len must be in [2, n_text_ctx]");
    WB_REQUIRE(kv == WB_KV_F32 || kv == WB_KV_F16, "session: kv_dtype must be WB_KV_F32 or WB_KV_F16");
    WB_CUDA(cudaSetDevice(m->device));
    max_windows = (int)max_w;
    max_beams = (int)max_b;
    t_max = (int)max_text_len;
    kv_dtype = kv;
    window_mode = mode;
    mel_limit = window_mel_frames(D.n_audio_ctx, mode);
    Rmax = max_windows * max_beams;
    TmS = mel_limit + 2;
    Tcap = (mel_limit - 1) / 2 + 1;
    Mcap = (int64_t)max_windows * Tcap;
    const int d = D.n_audio_state, H = D.n_text_head, L = D.n_text_layer, V = D.n_vocab;
    WB_REQUIRE(max_beams <= DEC_KC - 1, "session: max_beams must be <= 7 (candidates kept per record by the persistent decoders)");
    if (const char* e = getenv("WB200_DECODER"); e && e[0]) {   // run every launch on this decoder (comparisons, tests)
        only_decoder = atoi(e);
        WB_REQUIRE(only_decoder >= 3 && only_decoder <= 6, "session: WB200_DECODER must be 3, 4, 5 or 6");
    }

    WB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    for (auto& e : ev) WB_CUDA(cudaEventCreate(&e));
    d_lmwin.alloc(max_windows); d_g1.alloc(max_windows); d_g2.alloc(max_windows); d_awin.alloc(max_windows);
    d_win_row_off.alloc(max_windows); d_win_T.alloc(max_windows);
    max_slots.alloc(max_windows);
    mel_rows.alloc((size_t)max_windows * TmS * N_MELS);
    x.alloc(Mcap * d);
    xa.alloc(Mcap * d);
    if (kv == WB_KV_F16) ckv16.alloc((size_t)L * Mcap * 2 * d); else ckv.alloc((size_t)L * Mcap * 2 * d);
    use_tc = m->fp16_exact;   // fp16-exact weights (released checkpoints): tensor-core encoder on fp16 hi/lo planes; else fp32 CUDA cores
    if (use_tc) {
        const size_t nm = (size_t)max_windows * TmS * N_MELS, nh = (size_t)max_windows * TmS * d;
        mel_h.alloc(nm); mel_l.alloc(nm); h1_h.alloc(nh); h1_l.alloc(nh);
        xn_h.alloc(Mcap * d); xn_l.alloc(Mcap * d); qkv_h.alloc(Mcap * 3 * d); qkv_l.alloc(Mcap * 3 * d);
        att_h.alloc(Mcap * d); att_l.alloc(Mcap * d); hid_h.alloc(Mcap * 4 * d); hid_l.alloc(Mcap * 4 * d);
        xa_h.alloc(Mcap * d); xa_l.alloc(Mcap * d);
        enc_plans.resize((size_t)2 + 4 * D.n_audio_layer + L);
        for (auto& pl : enc_plans) pl.reset(new GemmF16Plan());
    } else {
        h1.alloc((size_t)max_windows * TmS * d);
        xn.alloc(Mcap * d); att.alloc(Mcap * d); qkv.alloc(Mcap * 3 * d); hid.alloc(Mcap * 4 * d);
    }
    if (kv == WB_KV_F16) { kc16.alloc((size_t)L * Rmax * t_max * d); vc16.alloc((size_t)L * Rmax * t_max * d); }
    else { kc.alloc((size_t)L * Rmax * t_max * d); vc.alloc((size_t)L * Rmax * t_max * d); }
    dx.alloc((size_t)Rmax * d);
    att_pl.alloc(4 * dec5_plane_uint4(d)); hid_pl.alloc(8 * dec5_plane_uint4(d));   // attention + LayerNorm output planes (hi, lo each), MLP hidden planes
    WB_CUDA(cudaMemsetAsync(att_pl.p, 0, 4 * dec5_plane_uint4(d) * sizeof(uint4), st));
    WB_CUDA(cudaMemsetAsync(hid_pl.p, 0, 8 * dec5_plane_uint4(d) * sizeof(uint4), st));
    dq.alloc((size_t)Rmax * d); dhid.alloc((size_t)Rmax * 4 * d);
    logits.alloc((size_t)Rmax * V);
    tokens.alloc((size_t)Rmax * t_max); token_lp.alloc((size_t)Rmax * t_max); lengths.alloc((size_t)2 * Rmax); cur_tok.alloc(Rmax); finished.alloc(Rmax);
    row_window.alloc(Rmax); anc0.alloc((size_t)Rmax * t_max); anc1.alloc((size_t)Rmax * t_max); parent.alloc(Rmax);
    pos.alloc(1); n_unfinished.alloc(128);
    topk_id.alloc((size_t)Rmax * DEC_KC); topk_lp.alloc((size_t)Rmax * DEC_KC);
    eot_logit.alloc(Rmax);
    is_special.alloc(V);
    {
        ckv_tmp.alloc(Mcap * 2 * d);
        cudaDeviceProp prop;
        WB_CUDA(cudaGetDeviceProperties(&prop, m->device));
        n_sm = prop.multiProcessorCount;
        const int n_logit_ctas = 2 * prop.multiProcessorCount;
        // persistent decoder: per-layer pointer table, barrier words, larger split-KV partial buffers
        part_o.alloc((size_t)Rmax * H * 16 * 64); part_m.alloc((size_t)Rmax * H * 16); part_l.alloc((size_t)Rmax * H * 16);
        datt.alloc((size_t)Rmax * d); steps_done.alloc(128); dec_bar.alloc(4);
        WB_CUDA(cudaMemsetAsync(dec_bar.p, 0, 4 * sizeof(unsigned int), st));
        {
            const bool h16 = m->fp16_exact;
            auto wp = [&](const LinearW& w) -> const void* { return h16 ? (const void*)w.w16 : (const void*)w.w32; };
            std::vector<DecLayer> lay((size_t)L);
            for (int l = 0; l < L; ++l) {
                const DecBlockW& B = m->dec[(size_t)l];
                DecLayer& y = lay[(size_t)l];
                y.ln1_g = B.attn_ln.g; y.ln1_b = B.attn_ln.b; y.ln1_eps = B.attn_ln.eps;
                y.ln2_g = B.cross_ln.g; y.ln2_b = B.cross_ln.b; y.ln2_eps = B.cross_ln.eps;
                y.ln3_g = B.mlp_ln.g; y.ln3_b = B.mlp_ln.b; y.ln3_eps = B.mlp_ln.eps;
                y.Wqkv = wp(B.qkv); y.Wo = wp(B.out); y.Wcq = wp(B.cq); y.Wco = wp(B.cout); y.W1 = wp(B.mlp1); y.W2 = wp(B.mlp2);
                y.bqkv = B.qkv.b; y.bo = B.out.b; y.bcq = B.cq.b; y.bco = B.cout.b; y.b1 = B.mlp1.b; y.b2 = B.mlp2.b;
            }
            dec_layers.alloc((size_t)L);
            WB_CUDA(cudaMemcpy(dec_layers.p, lay.data(), lay.size() * sizeof(DecLayer), cudaMemcpyHostToDevice));
        }
        dec5_build_tables(*m, n_sm, d5);
        ypart.alloc((size_t)4 * Rmax * d);   // decoder5.cu: MLP2 K-slab partial sums
        lg_m.alloc((size_t)n_logit_ctas * Rmax); lg_s.alloc((size_t)n_logit_ctas * Rmax);
        lg_v.alloc((size_t)n_logit_ctas * Rmax * DEC_KC); lg_i.alloc((size_t)n_logit_ctas * Rmax * DEC_KC);
    }
    h_parent = pinned<int>(Rmax); h_window = pinned<int>(Rmax); h_token = pinned<int>(Rmax);
    h_topk_id = pinned<int>((size_t)Rmax * DEC_KC);
    WB_CUDA(cudaMemsetAsync(is_special.p, 0, V, st));

    DecArgs& a = dec_base;
    a.Rmax = Rmax; a.d = D.n_text_state; a.H = H; a.L = L; a.V = V; a.t_max = t_max; a.Mcap = Mcap;
    a.eps_outside = m->ln_eps_outside; a.qk_scale = (float)std::pow((double)D.n_text_state / (double)H, -0.25);
    a.layers = dec_layers.p; a.tok_emb = m->tok_emb32; a.pos_emb = m->dec_pos;
    a.E = m->fp16_exact ? (const void*)m->tok_emb16 : (const void*)m->tok_emb32;
    a.E_tiled = m->tok_emb16_tiled;
    a.lnf_g = m->dec_ln.g; a.lnf_b = m->dec_ln.b; a.lnf_eps = m->dec_ln.eps;
    a.x = dx.p; a.q = dq.p; a.att = datt.p; a.hid = dhid.p;
    a.ypart = ypart.p; a.lgbuf = logits.p; a.att_pl = att_pl.p; a.hid_pl = hid_pl.p;
    a.kv_half = kv == WB_KV_F16 ? 1 : 0;
    if (a.kv_half) { a.kc = kc16.p; a.vc = vc16.p; a.ckv = ckv16.p; } else { a.kc = kc.p; a.vc = vc.p; a.ckv = ckv.p; }
    a.row_window = row_window.p; a.win_row_off = d_win_row_off.p; a.win_T = d_win_T.p;
    a.part_o = part_o.p; a.part_m = part_m.p; a.part_l = part_l.p;
    a.tokens = tokens.p; a.token_lp = token_lp.p; a.cur_tok = cur_tok.p; a.lengths = lengths.p; a.finished = finished.p;
    a.eot_logit = eot_logit.p; a.topk_id = topk_id.p; a.topk_lp = topk_lp.p;
    a.lg_m = lg_m.p; a.lg_s = lg_s.p; a.lg_v = lg_v.p; a.lg_i = lg_i.p;
    a.pos = pos.p; a.n_unfinished = n_unfinished.p; a.steps_done = steps_done.p; a.bar = dec_bar.p;
    WB_CUDA(cudaStreamSynchronize(st));
}

Session::~Session() {
    if (st) cudaStreamSynchronize(st);
    for (auto& e : ev)
        if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
}

// ---- geometry helpers -------------------------------------------------------------------------
static void set_geometry(Session& s, const std::vector<int>& Tm, const std::vector<int>& F) {
    s.n_windows = (int)Tm.size();
    s.win_Tm = Tm;
    s.win_F = F;
    s.win_T.resize(Tm.size());
    s.win_row_off.resize(Tm.size());
    s.M_tot = 0;
    s.max_T = 0;
    s.max_Tm = 0;
    for (size_t w = 0; w < Tm.size(); ++w) {
        s.win_T[w] = (Tm[w] - 1) / 2 + 1;       // Conv1d k3 p1 s2 (mod.rs:179-182)
        s.win_row_off[w] = s.M_tot;
        s.M_tot += s.win_T[w];
        s.max_T = std::max(s.max_T, s.win_T[w]);
        s.max_Tm = std::max(s.max_Tm, Tm[w]);
    }
    const int d = s.m->dims.n_audio_state;
    std::vector<GemmGroup> g1(Tm.size()), g2(Tm.size());
    std::vector<AttnWindow> aw(Tm.size());
    for (size_t w = 0; w < Tm.size(); ++w) {
        // conv1: output frame t reads mel buffer rows t, t+1, t+2 (frames t-1, t, t+1), writes h1 row t+1
        g1[w] = GemmGroup{(int64_t)w * s.TmS * N_MELS, ((int64_t)w * s.TmS + 1) * d, Tm[w]};
        // conv2 (stride 2): output t reads h1 buffer rows 2t, 2t+1, 2t+2 (frames 2t-1, 2t, 2t+1)
        g2[w] = GemmGroup{(int64_t)w * s.TmS * d, s.win_row_off[w] * d, s.win_T[w]};
        aw[w] = AttnWindow{s.win_row_off[w], s.win_T[w]};
    }
    WB_CUDA(cudaMemcpyAsync(s.d_g1.p, g1.data(), g1.size() * sizeof(GemmGroup), cudaMemcpyHostToDevice, s.st));
    WB_CUDA(cudaMemcpyAsync(s.d_g2.p, g2.data(), g2.size() * sizeof(GemmGroup), cudaMemcpyHostToDevice, s.st));
    WB_CUDA(cudaMemcpyAsync(s.d_awin.p, aw.data(), aw.size() * sizeof(AttnWindow), cudaMemcpyHostToDevice, s.st));
    WB_CUDA(cudaMemcpyAsync(s.d_win_row_off.p, s.win_row_off.data(), Tm.size() * sizeof(int64_t),
                            cudaMemcpyHostToDevice, s.st));
    WB_CUDA(cudaMemcpyAsync(s.d_win_T.p, s.win_T.data(), Tm.size() * sizeof(int), cudaMemcpyHostToDevice, s.st));
    WB_CUDA(cudaStreamSynchronize(s.st));   // the host vectors above are temporaries
}

void Session::encode_from_device_wave(const float* wave_dev, const int64_t* offsets, const int64_t* lens, int64_t n) {
    WB_REQUIRE(n >= 1 && n <= max_windows, "encode: n_windows out of range for this session");
    std::vector<LogMelWindow> lw((size_t)n);
    std::vector<int> Tm((size_t)n), kept((size_t)n);
    int max_frames = 0;
    for (int64_t w = 0; w < n; ++w) {
        WB_REQUIRE(lens[w] >= N_FFT, "prep_audio: waveform shorter than n_fft (audio.rs:292)");
        WB_REQUIRE(lens[w] < (int64_t)1 << 30, "prep_audio: waveform too long");
        const int F = (int)(lens[w] / HOP);                        // frames after dropping the last one
        const int keep = std::min(F, mel_limit - MEL_PADDING);      // transcribe.rs:173
        Tm[(size_t)w] = keep + MEL_PADDING;
        kept[(size_t)w] = keep;
        lw[(size_t)w] = LogMelWindow{offsets[w], (int)lens[w], F, keep, (int)w, ((int64_t)w * TmS + 1) * N_MELS};
        max_frames = std::max(max_frames, F);
    }
    WB_CUDA(cudaMemcpyAsync(d_lmwin.p, lw.data(), lw.size() * sizeof(LogMelWindow), cudaMemcpyHostToDevice, st));
    set_geometry(*this, Tm, kept);   // syncs, so `lw` may go out of scope
    WB_CUDA(cudaEventRecord(ev[0], st));
    WB_CUDA(cudaMemsetAsync(mel_rows.p, 0, (size_t)n * TmS * N_MELS * sizeof(float), st));   // halo + 10 zero frames
    launch_logmel(*m, wave_dev, d_lmwin.p, (int)n, max_frames, mel_rows.p, max_slots.p, (int)n, st);
    WB_CUDA(cudaEventRecord(ev[1], st));
    run_encoder();
    WB_CUDA(cudaEventRecord(ev[2], st));
}

void Session::encode_waveforms_host(const float* const* waves, const int64_t* lens, int64_t n) {
    WB_REQUIRE(n >= 1 && n <= max_windows, "encode: n_windows out of range for this session");
    std::vector<int64_t> offs((size_t)n);
    int64_t total = 0;
    for (int64_t w = 0; w < n; ++w) {
        WB_REQUIRE(waves[w] != nullptr && lens[w] >= 0, "encode: null waveform");
        offs[(size_t)w] = total;
        total += (lens[w] + 3) / 4 * 4;   // keep windows 16-byte aligned
    }
    wave.ensure((size_t)total);
    for (int64_t w = 0; w < n; ++w)
        WB_CUDA(cudaMemcpyAsync(wave.p + offs[(size_t)w], waves[w], (size_t)lens[w] * sizeof(float),
                                cudaMemcpyHostToDevice, st));
    encode_from_device_wave(wave.p, offs.data(), lens, n);
}

void Session::encode_mels_host(const float* mel, int64_t n, int64_t n_mels, int64_t n_ctx) {
    const wb_dims& D = m->dims;
    WB_REQUIRE(n_mels == D.n_mels, "Audio mel spectrum size must be n_mels (mod.rs:231-235)");
    WB_REQUIRE(n_ctx >= 1 && n_ctx <= mel_limit, "Audio length cannot exceed the session's mel frame limit: n_audio_ctx, "
                                                 "2 * n_audio_ctx in native windowing (mod.rs:236-241)");
    WB_REQUIRE(n >= 1 && n <= max_windows, "encode: n_windows out of range for this session");
    std::vector<int> Tm((size_t)n, (int)n_ctx);
    set_geometry(*this, Tm, Tm);
    DevBuf<float> tmp;
    tmp.alloc((size_t)n * n_mels * n_ctx);
    WB_CUDA(cudaMemcpyAsync(tmp.p, mel, tmp.n * sizeof(float), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemsetAsync(mel_rows.p, 0, (size_t)n * TmS * N_MELS * sizeof(float), st));
    for (int64_t w = 0; w < n; ++w)
        launch_chan_to_rows(tmp.p + w * n_mels * n_ctx, mel_rows.p + ((int64_t)w * TmS + 1) * N_MELS, (int)n_ctx, n_ctx, st);
    run_encoder();
    WB_CUDA(cudaStreamSynchronize(st));
}

void Session::load_encoder_output_host(const float* xa_host, int64_t n, int64_t T) {
    WB_REQUIRE(n >= 1 && n <= max_windows && T >= 1 && T <= Tcap, "forward_decoder: encoder output shape out of range");
    std::vector<int> Tm((size_t)n, (int)(2 * T - 1));   // any Tm with (Tm-1)/2+1 == T
    set_geometry(*this, Tm, std::vector<int>((size_t)n, (int)(2 * T)));   // every encoder position holds audio
    const int d = m->dims.n_audio_state;
    WB_CUDA(cudaMemcpyAsync(xa.p, xa_host, (size_t)n * T * d * sizeof(float), cudaMemcpyHostToDevice, st));
    if (use_tc) launch_split_f16(xa.p, xa_h.p, xa_l.p, (int64_t)n * T * d, st);
    run_cross_kv();
    encoded = true;
}

// ---- encoder ------------------------------------------------------------------------------------
void Session::run_encoder() {
    if (use_tc) run_encoder_f16();
    else run_encoder_f32();
    run_cross_kv();
    encoded = true;
}

// Tensor-core encoder (fp16-exact weights): conv stems, attention and MLP GEMMs are wgmma GEMMs over fp16 hi/lo planes
// (gemm_f16.cu), attention is enc_attn_tc.cu; only the residual stream x and the encoder output stay fp32 rows.
void Session::run_encoder_f16() {
    const wb_dims& D = m->dims;
    const int d = D.n_audio_state;
    const int M = (int)M_tot;
    const float qk_scale = (float)std::pow((double)d / (double)D.n_audio_head, -0.25);   // mod.rs:503
    auto run = [&](size_t site, const GemmF16Params& p, int64_t gstride, int rows_per_group) {
        GemmF16Plan& pl = *enc_plans[site];
        if (!pl.matches(p.max_rows, p.groups ? p.n_groups : 1)) pl.build(p, gstride, rows_per_group);   // tensor maps once per geometry
        pl.launch(st);
    };
    // halo rows of the conv1 output must read as zero padding
    WB_CUDA(cudaMemsetAsync(h1_h.p, 0, (size_t)n_windows * TmS * d * sizeof(__half), st));
    WB_CUDA(cudaMemsetAsync(h1_l.p, 0, (size_t)n_windows * TmS * d * sizeof(__half), st));
    launch_split_f16(mel_rows.p, mel_h.p, mel_l.p, (int64_t)n_windows * TmS * N_MELS, st);
    GemmF16Params p;
    // conv1 + GELU (mod.rs:243): K = 3*80 over three consecutive token-major mel rows; a conv output row is a dot product with
    // ONE contiguous 240-vector, so the conv is a GEMM whose A rows overlap (lda = 80 < K)
    p.A_hi = mel_h.p; p.A_lo = mel_l.p; p.lda = N_MELS; p.B = m->conv1.w16; p.P_hi = h1_h.p; p.P_lo = h1_l.p; p.ldc = d; p.N = d; p.K = 3 * N_MELS;
    p.bias = m->conv1.b; p.act = ACT_GELU; p.groups = d_g1.p; p.n_groups = n_windows; p.max_rows = max_Tm;
    run(0, p, (int64_t)TmS * N_MELS, TmS - 2);
    // conv2 (stride 2) + GELU + transpose + positional embedding (mod.rs:244-252)
    p = GemmF16Params{};
    p.A_hi = h1_h.p; p.A_lo = h1_l.p; p.lda = 2 * d; p.B = m->conv2.w16; p.C = x.p; p.ldc = d; p.N = d; p.K = 3 * d;
    p.bias = m->conv2.b; p.act = ACT_GELU; p.pos = m->enc_pos; p.groups = d_g2.p; p.n_groups = n_windows; p.max_rows = max_T;
    run(1, p, (int64_t)TmS * d, Tcap);
    for (int l = 0; l < D.n_audio_layer; ++l) {
        const EncBlockW& B = m->enc[(size_t)l];
        const size_t site = (size_t)2 + 4 * l;
        // x = x + attn(attn_ln(x))   (mod.rs:300)
        launch_layernorm(x.p, nullptr, xn_h.p, xn_l.p, B.attn_ln, M, d, m->ln_eps_outside, st);
        p = GemmF16Params{};
        p.A_hi = xn_h.p; p.A_lo = xn_l.p; p.lda = d; p.B = B.qkv.w16; p.P_hi = qkv_h.p; p.P_lo = qkv_l.p; p.ldc = 3 * d; p.N = 3 * d; p.K = d;
        p.bias = B.qkv.b; p.scale = qk_scale; p.scale_cols = 2 * d; p.max_rows = M;
        run(site, p, 0, M);
        launch_encoder_attention_tc(qkv_h.p, qkv_l.p, att_h.p, att_l.p, d_awin.p, n_windows, max_T, d, D.n_audio_head, st);
        p = GemmF16Params{};
        p.A_hi = att_h.p; p.A_lo = att_l.p; p.lda = d; p.B = B.out.w16; p.C = x.p; p.ldc = d; p.N = d; p.K = d;
        p.bias = B.out.b; p.residual = x.p; p.max_rows = M;
        run(site + 1, p, 0, M);
        // x = x + mlp(mlp_ln(x))     (mod.rs:301); the MLP1 epilogue (bias + GELU) emits the hidden layer as planes
        launch_layernorm(x.p, nullptr, xn_h.p, xn_l.p, B.mlp_ln, M, d, m->ln_eps_outside, st);
        p = GemmF16Params{};
        p.A_hi = xn_h.p; p.A_lo = xn_l.p; p.lda = d; p.B = B.mlp1.w16; p.P_hi = hid_h.p; p.P_lo = hid_l.p; p.ldc = 4 * d; p.N = 4 * d; p.K = d;
        p.bias = B.mlp1.b; p.act = ACT_GELU; p.max_rows = M;
        run(site + 2, p, 0, M);
        p = GemmF16Params{};
        p.A_hi = hid_h.p; p.A_lo = hid_l.p; p.lda = 4 * d; p.B = B.mlp2.w16; p.C = x.p; p.ldc = d; p.N = d; p.K = 4 * d;
        p.bias = B.mlp2.b; p.residual = x.p; p.max_rows = M;
        run(site + 3, p, 0, M);
    }
    launch_layernorm(x.p, xa.p, xa_h.p, xa_l.p, m->ln_post, M, d, m->ln_eps_outside, st);   // mod.rs:259
}

// fp32 CUDA-core encoder: weights that are not exactly representable in fp16
void Session::run_encoder_f32() {
    const wb_dims& D = m->dims;
    const int d = D.n_audio_state;
    const int M = (int)M_tot;
    const float qk_scale = (float)std::pow((double)d / (double)D.n_audio_head, -0.25);   // mod.rs:503
    WB_CUDA(cudaMemsetAsync(h1.p, 0, (size_t)n_windows * TmS * d * sizeof(float), st));
    GemmParams p;
    p.A = mel_rows.p; p.lda = N_MELS; p.B = m->conv1.w32; p.C = h1.p; p.ldc = d; p.N = d; p.K = 3 * N_MELS;
    p.bias = m->conv1.b; p.act = ACT_GELU; p.groups = d_g1.p; p.n_groups = n_windows; p.max_rows = max_Tm;
    launch_gemm(p, st);
    p = GemmParams{};
    p.A = h1.p; p.lda = 2 * d; p.B = m->conv2.w32; p.C = x.p; p.ldc = d; p.N = d; p.K = 3 * d;
    p.bias = m->conv2.b; p.act = ACT_GELU; p.pos = m->enc_pos; p.groups = d_g2.p; p.n_groups = n_windows;
    p.max_rows = max_T;
    launch_gemm(p, st);
    for (int l = 0; l < D.n_audio_layer; ++l) {
        const EncBlockW& B = m->enc[(size_t)l];
        launch_layernorm(x.p, xn.p, nullptr, nullptr, B.attn_ln, M, d, m->ln_eps_outside, st);
        p = GemmParams{};
        p.A = xn.p; p.lda = d; p.B = B.qkv.w32; p.C = qkv.p; p.ldc = 3 * d; p.N = 3 * d; p.K = d;
        p.bias = B.qkv.b; p.scale = qk_scale; p.scale_cols = 2 * d; p.max_rows = M;
        launch_gemm(p, st);
        launch_encoder_attention(qkv.p, att.p, d_awin.p, n_windows, max_T, d, D.n_audio_head, st);
        p = GemmParams{};
        p.A = att.p; p.lda = d; p.B = B.out.w32; p.C = x.p; p.ldc = d; p.N = d; p.K = d;
        p.bias = B.out.b; p.residual = x.p; p.max_rows = M;
        launch_gemm(p, st);
        launch_layernorm(x.p, xn.p, nullptr, nullptr, B.mlp_ln, M, d, m->ln_eps_outside, st);
        p = GemmParams{};
        p.A = xn.p; p.lda = d; p.B = B.mlp1.w32; p.C = hid.p; p.ldc = 4 * d; p.N = 4 * d; p.K = d;
        p.bias = B.mlp1.b; p.act = ACT_GELU; p.max_rows = M;
        launch_gemm(p, st);
        p = GemmParams{};
        p.A = hid.p; p.lda = 4 * d; p.B = B.mlp2.w32; p.C = x.p; p.ldc = d; p.N = d; p.K = 4 * d;
        p.bias = B.mlp2.b; p.residual = x.p; p.max_rows = M;
        launch_gemm(p, st);
    }
    launch_layernorm(x.p, xa.p, nullptr, nullptr, m->ln_post, M, d, m->ln_eps_outside, st);   // mod.rs:259
}

// cross keys (pre-scaled) | values of every decoder layer, projected once per window (mod.rs:484-485 hoisted out of the step loop)
// into ckv_tmp, then re-laid out head-major per window (encoder.cu ckv_relayout_kernel): what the persistent decoders stream
void Session::run_cross_kv() {
    const wb_dims& D = m->dims;
    const int d = D.n_text_state;
    const float qk_scale = (float)std::pow((double)d / (double)D.n_text_head, -0.25);
    for (int l = 0; l < D.n_text_layer; ++l) {
        const DecBlockW& B = m->dec[(size_t)l];
        if (use_tc) {
            GemmF16Params p;
            p.A_hi = xa_h.p; p.A_lo = xa_l.p; p.lda = d; p.B = B.ckv.w16; p.C = ckv_tmp.p; p.ldc = 2 * d;
            p.N = 2 * d; p.K = d; p.bias = B.ckv.b; p.scale = qk_scale; p.scale_cols = d; p.max_rows = (int)M_tot;
            GemmF16Plan& pl = *enc_plans[(size_t)2 + 4 * D.n_audio_layer + l];
            if (!pl.matches(p.max_rows, 1)) pl.build(p, 0, (int)M_tot);
            pl.launch(st);
        } else {
            GemmParams p;
            p.A = xa.p; p.lda = d; p.B = B.ckv.w32; p.C = ckv_tmp.p; p.ldc = 2 * d;
            p.N = 2 * d; p.K = d; p.bias = B.ckv.b; p.scale = qk_scale; p.scale_cols = d; p.max_rows = (int)M_tot;
            launch_gemm(p, st);
        }
        void* dst = kv_dtype == WB_KV_F16 ? (void*)(ckv16.p + (size_t)l * Mcap * 2 * d) : (void*)(ckv.p + (size_t)l * Mcap * 2 * d);
        launch_ckv_relayout(ckv_tmp.p, dst, kv_dtype == WB_KV_F16, d_win_row_off.p, d_win_T.p, n_windows, M_tot, d, st);   // head-major
    }
}

// ---- decoder --------------------------------------------------------------------------------------
void Session::set_special(const uint8_t* sp) {
    if (sp) {
        WB_CUDA(cudaMemcpyAsync(is_special.p, sp, (size_t)m->dims.n_vocab, cudaMemcpyHostToDevice, st));
        WB_CUDA(cudaStreamSynchronize(st));
        have_special = true;
    }
}

void Session::seat_rows(int rows, int per_window, const std::vector<std::vector<int64_t>>& prompts, int max_depth) {
    if (!encoded) fail(WB_ERR_STATE, "session: decode before encode");
    WB_REQUIRE(rows <= Rmax && (int64_t)prompts.size() * per_window >= rows, "decode: rows out of range");
    const int V = m->dims.n_vocab;
    std::vector<int> tk((size_t)rows * t_max, 0), rw((size_t)rows), len((size_t)rows), lim((size_t)rows);
    for (int r = 0; r < rows; ++r) {
        const std::vector<int64_t>& pr = prompts[(size_t)(r / per_window)];
        WB_REQUIRE(!pr.empty() && (int64_t)pr.size() <= t_max, "decode: prompt length out of range");
        rw[(size_t)r] = r / per_window;
        len[(size_t)r] = (int)pr.size();
        lim[(size_t)r] = (int)pr.size() + max_depth;
        for (size_t i = 0; i < pr.size(); ++i) {
            WB_REQUIRE(pr[i] >= 0 && pr[i] < V, "decode: prompt token out of range");
            tk[(size_t)r * t_max + i] = (int)pr[i];
        }
    }
    WB_CUDA(cudaMemcpyAsync(tokens.p, tk.data(), tk.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(row_window.p, rw.data(), rw.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemsetAsync(finished.p, 0, sizeof(int) * Rmax, st));
    WB_CUDA(cudaMemsetAsync(pos.p, 0, sizeof(int), st));
    WB_CUDA(cudaMemcpyAsync(lengths.p, len.data(), len.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(lengths.p + Rmax, lim.data(), lim.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    R = rows;
    anc_identity = true;
    anc_cur = 0;
    host_pos = 0;
}

void Session::feed_positions(int n, float* logits_out) {
    const size_t V = (size_t)m->dims.n_vocab;
    const StepLogits out = logits_out ? StepLogits::topk_and_raw : StepLogits::none;
    for (int p = 0; p < n; ++p, ++host_pos) {
        // every row's token at p: column p of the token buffer
        WB_CUDA(cudaMemcpy2DAsync(cur_tok.p, sizeof(int), tokens.p + p, t_max * sizeof(int), sizeof(int), R, cudaMemcpyDeviceToDevice, st));
        launch_decoder(DecodeLaunch::cached_step(R, host_pos, out, MASK_NONE, 1));
        if (logits_out)
            WB_CUDA(cudaMemcpy2DAsync(logits_out + p * V, n * V * sizeof(float), logits.p, V * sizeof(float), V * sizeof(float), R,
                                      cudaMemcpyDeviceToHost, st));
    }
}

// the shortest and longest of n prompts
static std::pair<int, int> prompt_range(const std::vector<std::vector<int64_t>>& prompts) {
    int lo = INT_MAX, hi = 0;
    for (const auto& pr : prompts) { lo = std::min(lo, (int)pr.size()); hi = std::max(hi, (int)pr.size()); }
    return {lo, hi};
}

void Session::begin(const std::vector<std::vector<int64_t>>& prompts, bool prefill, int max_depth) {
    WB_REQUIRE((int64_t)prompts.size() == n_windows, "begin: one prompt per encoded window");
    for (const auto& pr : prompts) WB_REQUIRE(!pr.empty() && (int64_t)pr.size() < t_max, "begin: prompt length out of range");
    seat_rows(n_windows, 1, prompts, max_depth);
    if (prefill) feed_positions(prompt_range(prompts).first - 1, nullptr);   // before every prompt's last token: no logits needed
    WB_CUDA(cudaStreamSynchronize(st));
}

void Session::teacher_forced_logits(const int64_t* toks, int64_t n_rows, int64_t seq_len, float* logits_out) {
    WB_REQUIRE(n_rows >= 1 && seq_len >= 1, "forward_decoder: empty input");
    std::vector<std::vector<int64_t>> rows((size_t)n_rows);
    for (int64_t r = 0; r < n_rows; ++r) rows[(size_t)r].assign(toks + r * seq_len, toks + (r + 1) * seq_len);
    seat_rows((int)n_rows, 1, rows);
    feed_positions((int)seq_len, logits_out);
    WB_CUDA(cudaStreamSynchronize(st));
}

// The first of decoder4 -> decoder6 -> decoder5 -> decoder3 that covers the launch (each launch_decN decides that itself),
// or only the one WB200_DECODER names.
bool Session::launch_decoder(const DecodeLaunch& l) {
    DecArgs a = dec_base;
    a.R = l.rows;
    a.lg_slices = std::max(1, std::min(16, n_sm / std::max(1, l.rows)));
    a.n_splits = std::max(1, std::min(16, n_sm / std::max(1, l.rows * a.H)));
    a.anc = anc_identity ? nullptr : (anc_cur == 0 ? anc0.p : anc1.p);
    a.use_cur_tok = l.use_cur_tok; a.pos0 = l.pos0; a.n_steps = l.n_steps; a.logits_from = l.logits_from;
    a.is_special = have_special ? is_special.p : nullptr; a.mask_mode = l.mask_mode;
    a.k = l.k; a.greedy = l.greedy; a.eot = l.eot; a.loop_rules = l.loop_rules; a.max_depth = l.max_depth;
    a.logits_out = l.raw_logits ? logits.p : nullptr;
    if (getenv("WB200_TRACE")) {
        dec_trace.ensure(1 << 16);
        WB_CUDA(cudaMemsetAsync(dec_trace.p, 0, sizeof(unsigned long long) * (1 << 16), st));
        a.trace = dec_trace.p;
        a.trace_cap = 1 << 16;
    }
    WB_CUDA(cudaMemsetAsync(dec_bar.p, 0, 4 * sizeof(unsigned int), st));   // monotonic barrier counters start at 0
    const bool h16 = m->fp16_exact;
    auto allowed = [&](int n) { return only_decoder == 0 || only_decoder == n; };
    int groups = 0;
    last_groups = 1;
    if (l.beam > 1) {   // the whole search: only decoder6 has a beam mode
        a.beam = l.beam; a.n_win = l.rows / l.beam;
        a.anc = anc0.p; a.anc_alt = anc1.p; a.slot_live = slot_live.p;
        a.bm_head = bm_head.p; a.bm_seq = bm_seq.p; a.bm_cnt = bm_cnt.p; a.bm_win = bm_win.p; a.bm_out = bm_out.p; a.bm_out_len = bm_out_len.p;
        a.bm_seq_lp = bm_seq_lp.p; a.bm_out_lp = bm_out_lp.p;
        if (!allowed(6) || !launch_dec6(a, *m, d6, st)) return false;
        last_decoder = 6;
    } else if (allowed(4) && launch_dec4(a, h16, st)) last_decoder = 4;
    else if (allowed(6) && launch_dec6(a, *m, d6, st)) last_decoder = 6;
    else if (allowed(5) && (groups = launch_dec5(a, d5, n_sm, h16, st)) > 0) { last_decoder = 5; last_groups = groups; }
    else if (allowed(3)) { launch_dec3(a, n_sm, h16, st); last_decoder = 3; }
    else fail(WB_ERR_UNSUPPORTED, "WB200_DECODER=" + std::to_string(only_decoder) + ": decoder" + std::to_string(only_decoder) + " does not cover this launch");
    last_rows = l.rows;
    last_k = l.k;
    if (a.trace) {
        std::vector<unsigned long long> h(1 << 16);
        WB_CUDA(cudaStreamSynchronize(st));
        WB_CUDA(cudaMemcpy(h.data(), dec_trace.p, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        FILE* f = fopen(getenv("WB200_TRACE"), "w");   // debugging aid: WB200_TRACE=<file> receives the stage time stamps of CTA 0
        if (f) {
            for (size_t i = 0; i < h.size(); ++i)
                if (h[i]) fprintf(f, "%llu\n", h[i]);   // stage stamps of CTA 0
            fclose(f);
        }
    }
    return true;
}

void Session::profile_decode(const int64_t* prompt, int64_t prompt_len, int n_steps, float* logits_ms, float* step_ms) {
    WB_REQUIRE(n_steps >= 1 && prompt_len + n_steps <= t_max, "profile: n_steps out of range");
    // the whole decode is ONE kernel: time the launch (prefill + n_steps greedy steps) and report per position
    begin(std::vector<std::vector<int64_t>>((size_t)n_windows, std::vector<int64_t>(prompt, prompt + prompt_len)), false, n_steps);
    const int total = (int)prompt_len - 1 + n_steps;
    WB_CUDA(cudaEventRecord(ev[4], st));
    launch_decoder(DecodeLaunch::greedy_search(R, (int)prompt_len, (int)prompt_len, n_steps, /*eot=*/-1, /*loop_rules=*/false));
    WB_CUDA(cudaEventRecord(ev[5], st));
    WB_CUDA(cudaStreamSynchronize(st));
    float t = 0.f;
    WB_CUDA(cudaEventElapsedTime(&t, ev[4], ev[5]));
    *logits_ms = t / (float)total;
    *step_ms = t / (float)total;
}

void Session::step_beams(int64_t n_rows, const int32_t* window_of_row, const int32_t* parent_row, const int64_t* token,
                         int apply_mask, int k, int64_t* topk_ids_out, float* topk_lp_out) {
    if (!encoded) fail(WB_ERR_STATE, "session: step before encode/begin");
    WB_REQUIRE(n_rows >= 1 && n_rows <= Rmax, "step: n_rows out of range");
    WB_REQUIRE(k >= 1 && k <= DEC_KC - 1, "step: k must be in [1, 7]");
    WB_REQUIRE(host_pos + 1 < t_max, "step: session max_text_len exceeded");
    const int V = m->dims.n_vocab;
    for (int64_t r = 0; r < n_rows; ++r) {
        WB_REQUIRE(parent_row[r] >= 0 && parent_row[r] < R, "step: parent_row out of range");
        WB_REQUIRE(window_of_row[r] >= 0 && window_of_row[r] < n_windows, "step: window_of_row out of range");
        WB_REQUIRE(token[r] >= 0 && token[r] < V, "step: token out of range");
        h_parent[r] = parent_row[r];
        h_window[r] = window_of_row[r];
        h_token[r] = (int)token[r];
    }
    WB_CUDA(cudaMemcpyAsync(parent.p, h_parent.get(), sizeof(int) * n_rows, cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(row_window.p, h_window.get(), sizeof(int) * n_rows, cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(cur_tok.p, h_token.get(), sizeof(int) * n_rows, cudaMemcpyHostToDevice, st));
    if (anc_identity) {   // rows so far (prompt) live in their own cache rows
        launch_dec_anc_identity(anc0.p, Rmax, t_max, st);
        anc_cur = 0;
        anc_identity = false;
    }
    {
        int* cur = anc_cur == 0 ? anc0.p : anc1.p;
        int* nxt = anc_cur == 0 ? anc1.p : anc0.p;
        R = (int)n_rows;
        launch_dec_reorder(cur, nxt, parent.p, pos.p, R, t_max, st);
        anc_cur ^= 1;
    }
    launch_decoder(DecodeLaunch::cached_step(R, host_pos, StepLogits::topk, apply_mask ? MASK_ALWAYS : MASK_NONE, k));
    ++host_pos;
    WB_CUDA(cudaMemcpyAsync(h_topk_id.get(), topk_id.p, sizeof(int) * n_rows * k, cudaMemcpyDeviceToHost, st));
    WB_CUDA(cudaMemcpyAsync(topk_lp_out, topk_lp.p, sizeof(float) * n_rows * k, cudaMemcpyDeviceToHost, st));
    WB_CUDA(cudaStreamSynchronize(st));
    for (int64_t i = 0; i < n_rows * k; ++i) topk_ids_out[i] = h_topk_id[i];
}

void Session::last_topk(int64_t n_rows, int64_t k, int64_t* ids_out, float* lp_out) {
    if (last_decoder == 0) fail(WB_ERR_STATE, "last_topk: no decoder launch yet");
    WB_REQUIRE(k == last_k, "last_topk: k differs from the last launch's k");
    WB_REQUIRE(n_rows >= 1 && n_rows <= last_rows, "last_topk: n_rows exceeds the last launch's rows");
    std::vector<int> ids((size_t)(n_rows * k));
    WB_CUDA(cudaStreamSynchronize(st));
    WB_CUDA(cudaMemcpy(ids.data(), topk_id.p, ids.size() * sizeof(int), cudaMemcpyDeviceToHost));
    WB_CUDA(cudaMemcpy(lp_out, topk_lp.p, ids.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < ids.size(); ++i) ids_out[i] = ids[i];
}

void Session::greedy_decode(const std::vector<std::vector<int64_t>>& prompts, int max_depth, int64_t eot,
                            std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp, bool loop_rules) {
    const auto [min_lp, max_lp] = prompt_range(prompts);
    WB_REQUIRE(max_lp + max_depth <= t_max, "greedy: prompt + max_depth exceeds the session's max_text_len");
    // one launch: prompt prefill + every greedy step, early exit inside the kernel.  A row stops at EOT or at its own
    // prompt_len + max_depth ids; the greedy loop's context stop (prompt_len + max_depth <= t_max <= n_text_ctx) is the latter.
    begin(prompts, /*prefill=*/false, max_depth);
    if (max_depth > 0) launch_decoder(DecodeLaunch::greedy_search(R, min_lp, max_lp, max_depth, (int)eot, loop_rules));
    std::vector<int> tk((size_t)R * t_max), len((size_t)R);
    std::vector<float> lp((size_t)R * t_max);
    int sdv[128] = {0};
    WB_CUDA(cudaMemcpyAsync(tk.data(), tokens.p, tk.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    WB_CUDA(cudaMemcpyAsync(lp.data(), token_lp.p, lp.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    WB_CUDA(cudaMemcpyAsync(len.data(), lengths.p, len.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (max_depth > 0) WB_CUDA(cudaMemcpyAsync(sdv, steps_done.p, sizeof(int) * std::min(last_groups, 128), cudaMemcpyDeviceToHost, st));
    WB_CUDA(cudaStreamSynchronize(st));
    int sd = 0;
    for (int g = 0; g < std::min(last_groups, 128); ++g) sd = std::max(sd, sdv[g]);   // row groups stop on their own
    last_steps = max_depth > 0 ? sd - (min_lp - 1) : 0;
    host_pos = min_lp - 1 + (int)last_steps;
    out.assign((size_t)R, {});
    out_lp.assign((size_t)R, {});
    for (int r = 0; r < R; ++r) {
        const int64_t prompt_len = (int64_t)prompts[(size_t)r].size();
        for (int i = 0; i < len[(size_t)r]; ++i) {
            out[(size_t)r].push_back(tk[(size_t)r * t_max + i]);
            out_lp[(size_t)r].push_back(i < prompt_len ? 0.0f : lp[(size_t)r * t_max + i]);   // transcribe.rs:205-208
        }
        // a repetition cut that ends inside the prompt (the loop masks nothing) leaves its EOT in a prompt position
        if (loop_rules && max_depth > 0 && len[(size_t)r] <= prompt_len) out_lp[(size_t)r].back() = std::nanf("");
        // the greedy loop always ends in EOT: the EOT test's EOT and the context stop's are appended here (the latter may
        // not fit the token buffer); no step chose them, so their log-prob is NaN
        if (loop_rules && out[(size_t)r].back() != eot) {
            out[(size_t)r].push_back(eot);
            out_lp[(size_t)r].push_back(std::nanf(""));
        }
    }
}

bool Session::beam_decode(const std::vector<std::vector<int64_t>>& prompts, int beam_size, int max_depth, int64_t eot,
                          std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp,
                          std::vector<NBest>& nbest) {
    namespace fx = beamfx;
    const auto [min_lp, max_lp] = prompt_range(prompts);
    WB_REQUIRE(min_lp >= 1 && max_lp + max_depth <= t_max, "beam: prompt + max_depth exceeds the session's max_text_len");
    const int B = beam_size, W = n_windows, Rb = W * B;
    if (B < 2 || B > fx::MAX_BEAM || max_depth < 1 || Rb > Rmax) return false;
    // slot i of window w = row w * B + i; until the window's first search step only slot 0 holds a beam: the prompt, in its
    // own cache row
    seat_rows(Rb, B, prompts, max_depth);
    constexpr int MN = fx::MAX_NODES;
    slot_live.ensure((size_t)Rmax);
    bm_head.ensure((size_t)2 * W * MN); bm_seq.ensure((size_t)2 * W * MN * t_max); bm_seq_lp.ensure((size_t)2 * W * MN * t_max);
    bm_cnt.ensure((size_t)2 * W); bm_win.ensure((size_t)2 * W);
    bm_out.ensure((size_t)W * t_max); bm_out_lp.ensure((size_t)W * t_max); bm_out_len.ensure((size_t)W);
    std::vector<int> live((size_t)Rb);
    for (int r = 0; r < Rb; ++r) live[(size_t)r] = r % B == 0 ? 1 : 0;
    std::vector<fx::Head> heads((size_t)W * MN, fx::Head{0.0, 0, 0, 0, 0});
    std::vector<int> seq((size_t)W * MN * t_max, 0), cnt((size_t)2 * W, 0), win((size_t)2 * W, 0);   // depth-0 buffer; window: {buffer, done}
    for (int w = 0; w < W; ++w) {
        const std::vector<int64_t>& pr = prompts[(size_t)w];
        heads[(size_t)w * MN] = fx::Head{0.0, pr.back() == eot ? 1 : 0, w * B, (int)pr.size(), 0};
        for (size_t i = 0; i < pr.size(); ++i) seq[(size_t)w * MN * t_max + i] = (int)pr[i];
        cnt[(size_t)w] = 1;
    }
    WB_CUDA(cudaMemcpyAsync(slot_live.p, live.data(), live.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(bm_head.p, heads.data(), heads.size() * sizeof(fx::Head), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(bm_seq.p, seq.data(), seq.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemsetAsync(bm_seq_lp.p, 0, seq.size() * sizeof(float), st));   // the prompt's log-probs (transcribe.rs:205-208)
    WB_CUDA(cudaMemcpyAsync(bm_cnt.p, cnt.data(), cnt.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(bm_win.p, win.data(), win.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    launch_dec_anc_identity(anc0.p, Rb, t_max, st);
    const bool ran = launch_decoder(DecodeLaunch::beam_search(Rb, B, min_lp, max_lp, max_depth, (int)eot));
    std::vector<int> res((size_t)W * t_max), res_len((size_t)W);
    std::vector<float> res_lp((size_t)W * t_max);
    // the final carried lists: a window that finished early keeps its buffer (stage (b) skips done windows), so bm_win
    // picks each window's list out of both buffers.  Only the first max_lp + max_depth ids of a sequence can be set.
    const int used = max_lp + max_depth;
    std::vector<fx::Head> fin_head((size_t)2 * W * MN);
    std::vector<int> fin_cnt((size_t)2 * W), fin_win((size_t)2 * W), fin_seq((size_t)2 * W * MN * used);
    std::vector<float> fin_lp(fin_seq.size());
    int sd = 0;
    if (ran) {
        WB_CUDA(cudaMemcpyAsync(res.data(), bm_out.p, res.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(res_lp.data(), bm_out_lp.p, res_lp.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(res_len.data(), bm_out_len.p, res_len.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(&sd, steps_done.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(fin_head.data(), bm_head.p, fin_head.size() * sizeof(fx::Head), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(fin_cnt.data(), bm_cnt.p, fin_cnt.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpyAsync(fin_win.data(), bm_win.p, fin_win.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpy2DAsync(fin_seq.data(), used * sizeof(int), bm_seq.p, t_max * sizeof(int), used * sizeof(int),
                                  (size_t)2 * W * MN, cudaMemcpyDeviceToHost, st));
        WB_CUDA(cudaMemcpy2DAsync(fin_lp.data(), used * sizeof(float), bm_seq_lp.p, t_max * sizeof(float), used * sizeof(float),
                                  (size_t)2 * W * MN, cudaMemcpyDeviceToHost, st));
    }
    WB_CUDA(cudaStreamSynchronize(st));   // the host vectors above are in flight until here
    if (!ran) return false;
    // session state as the host search leaves it: position, ancestry of the last position
    last_steps = sd;
    host_pos = min_lp - 1 + sd;
    anc_identity = false;
    anc_cur = (sd - 1) & 1;
    out.assign((size_t)W, {});
    out_lp.assign((size_t)W, {});
    for (int w = 0; w < W; ++w)
        for (int i = 0; i < res_len[(size_t)w]; ++i) {
            out[(size_t)w].push_back(res[(size_t)w * t_max + i]);
            out_lp[(size_t)w].push_back(res_lp[(size_t)w * t_max + i]);
        }
    nbest.assign((size_t)W, {});
    for (int w = 0; w < W; ++w) {
        const size_t node0 = ((size_t)fin_win[(size_t)2 * w] * W + w) * MN;   // the window's current buffer
        const int n = fin_cnt[(size_t)fin_win[(size_t)2 * w] * W + w];
        Carried c;
        for (size_t i = node0; i < node0 + n; ++i) {
            c.heads.push_back(fin_head[i]);
            c.ids.emplace_back(fin_seq.begin() + i * used, fin_seq.begin() + i * used + fin_head[i].len);
            c.lps.emplace_back(fin_lp.begin() + i * used, fin_lp.begin() + i * used + fin_head[i].len);
        }
        nbest[(size_t)w] = ranked_nbest(c);
    }
    return true;
}

}  // namespace wb
