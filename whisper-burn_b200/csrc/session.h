// Decoding session: all device state between prep_audio and the emitted token ids.  Internal.
#pragma once
#include <climits>
#include <functional>
#include <memory>
#include <vector>

#include "decoder.h"
#include "wb_internal.h"

namespace wb {

constexpr int MEL_PADDING = 10;   // transcribe.rs:33

// The most mel frames one window gives the encoder (whisper_b200.h WB_WINDOWS_*): n_audio_ctx in the reference's windowing
// (transcribe.rs:32-34, 161-177), 2 * n_audio_ctx in native windowing (conv2 has stride 2, so T <= n_audio_ctx encoder
// positions).  Every other limit of a window follows from it: the waveform window is max_waveform_samples(limit - MEL_PADDING),
// a window keeps at most limit - MEL_PADDING frames.  Throws WB_ERR_INVALID_ARG on an unknown mode.
int window_mel_frames(int n_audio_ctx, int window_mode);
int64_t window_samples(int n_audio_ctx, int window_mode);

// what a cached step computes besides K/V: nothing (prefill), each row's k best candidates, or those and its raw logits
enum class StepLogits { none, topk, topk_and_raw };

// One persistent-decoder launch (Session::launch_decoder).  The named constructors are its three kinds; each field sets
// the DecArgs field of the same name (raw_logits: logits_out).
struct DecodeLaunch {
    int rows = 0, pos0 = 0, n_steps = 1, logits_from = INT_MAX;   // logits of the positions from logits_from on
    bool use_cur_tok = false, raw_logits = false;                  // tokens from cur_tok, else from the token buffer
    int mask_mode = MASK_NONE, k = 1, eot = -1;                    // k candidates per row; eot -1: no early finish
    bool greedy = false, loop_rules = false;
    int beam = 0, max_depth = 0;

    // position pos of every row, tokens from cur_tok
    static DecodeLaunch cached_step(int rows, int pos, StepLogits out, int mask_mode, int k) {
        DecodeLaunch l;
        l.rows = rows; l.pos0 = pos; l.use_cur_tok = true; l.mask_mode = mask_mode; l.k = k;
        l.logits_from = out == StepLogits::none ? INT_MAX : 0; l.raw_logits = out == StepLogits::topk_and_raw;
        return l;
    }
    // the prompt prefill (no logits), then max_depth positions of beam_size 1 of the beam search (special ids masked while
    // a sequence has <= 5 tokens) or, with loop_rules, of the reference's greedy loop (no mask); tokens from the token buffer.
    // Rows' prompts hold min_lp .. max_lp tokens (DecArgs::lengths): logits from the shortest prompt's last position on,
    // until the longest prompt's row has had max_depth steps
    static DecodeLaunch greedy_search(int rows, int min_lp, int max_lp, int max_depth, int eot, bool loop_rules) {
        DecodeLaunch l;
        l.rows = rows; l.n_steps = max_lp - 1 + max_depth; l.logits_from = min_lp - 1; l.eot = eot; l.max_depth = max_depth;
        l.greedy = true; l.loop_rules = loop_rules; l.mask_mode = loop_rules ? MASK_NONE : MASK_SHORT;
        return l;
    }
    // the same positions for the whole width-`beam` search of rows / beam windows (decoder6 beam mode)
    static DecodeLaunch beam_search(int rows, int beam, int min_lp, int max_lp, int max_depth, int eot) {
        DecodeLaunch l = greedy_search(rows, min_lp, max_lp, max_depth, eot, false);
        l.greedy = false; l.k = l.beam = beam;
        return l;
    }
};

// rows per pass of the teacher-forced decoder (token scoring, token alignment): sequences run in groups of whole sequences holding
// at most this many rows, so the workspace stays bounded (~56 KB per row at d = 1280)
constexpr int SCORE_GROUP_ROWS = 4096;

// workspace of token scoring (score.cu) and of the decoder pass token alignment shares with it, grown on demand
struct ScoreWs {
    DevBuf<int> tok, pos, target, seq_win, tile_i, am;   // per row: input token, position, target id; per sequence: window
    DevBuf<uint8_t> row_mask, special;
    DevBuf<AttnWindow> seqs;                              // rows of each sequence
    DevBuf<float> x, tile_m, tile_s, tgt_logit, lp;
    DevBuf<__half> xn_h, xn_l, qkv_h, qkv_l, att_h, att_l, hid_h, hid_l;
    std::vector<std::unique_ptr<GemmF16Plan>> plans;      // per decoder layer: qkv, out, cross query, cross out, mlp1, mlp2
};

// workspace of token alignment (align.cu), grown on demand
struct AlignSeq {        // one sequence of a group
    int64_t row_off;     // its first row in the group's packed rows
    int64_t mat_off;     // its first element in the group's packed matrices [N][C]
    int L, first, C, win;
};
struct AlignWs {
    DevBuf<AlignSeq> seqs;
    DevBuf<int64_t> out_off;         // per sequence its first aligned id in start / end
    DevBuf<int> heads, start, end;   // heads: the selected heads by layer, ascending; start / end: per aligned id
    DevBuf<float> w, mat;            // w: [heads of a layer][rows][Cmax] weights; mat: the group's packed matrices
    DevBuf<double> stats;            // [heads of a layer][sequences][Cmax]: column mean, biased std
};

// pinned host array
struct PinnedFree { void operator()(void* p) const { cudaFreeHost(p); } };
template <typename T> using Pinned = std::unique_ptr<T[], PinnedFree>;
template <typename T> Pinned<T> pinned(size_t n) { void* p = nullptr; WB_CUDA(cudaMallocHost(&p, n * sizeof(T))); return Pinned<T>((T*)p); }

struct Session {
    Model* m = nullptr;
    cudaStream_t st = nullptr;
    int max_windows = 0, max_beams = 0, t_max = 0, kv_dtype = WB_KV_F32;
    int window_mode = WB_WINDOWS_REFERENCE;
    int search = WB_SEARCH_BEAM;   // set_search: the rule transcribe_windows decodes by
    int64_t startofprev = -1;      // set_prev_prompt: >= 0 prompts each waveform window with the text before it
    int mel_limit = 0;   // window_mel_frames(n_audio_ctx, window_mode)
    int Rmax = 0;        // max_windows * max_beams decode rows
    int TmS = 0;         // rows per window in the token-major mel / conv1 buffers (mel_limit + 2 halo rows)
    int Tcap = 0;        // max encoder positions per window: (mel_limit - 1) / 2 + 1
    int64_t Mcap = 0;    // max packed encoder rows

    // ---- geometry of the windows currently encoded (host mirrors)
    int n_windows = 0;
    std::vector<int> win_Tm, win_T;
    std::vector<int> win_F;   // mel frames of each window that hold audio (kept frames; n_ctx of encode_mels): the alignment's columns
    std::vector<int64_t> win_row_off;
    int64_t M_tot = 0;
    int max_T = 0, max_Tm = 0;
    bool encoded = false;

    // ---- device: descriptors
    DevBuf<LogMelWindow> d_lmwin;
    DevBuf<GemmGroup> d_g1, d_g2;
    DevBuf<AttnWindow> d_awin;
    DevBuf<int64_t> d_win_row_off;
    DevBuf<int> d_win_T;
    // ---- device: frontend + encoder activations
    DevBuf<float> wave;
    ResampleBufs rs;   // waveforms_to_tokens_resampled: the interleaved inputs and their 16 kHz conversions
    DevBuf<int> max_slots;
    DevBuf<float> mel_rows, x, xa;           // token-major log-mel rows, residual stream, encoder output
    DevBuf<float> h1, xn, att, qkv, hid;     // fp32 activations of the CUDA-core encoder (weights that are not fp16-exact)
    // tensor-core path (fp16-exact weights): every GEMM input travels as a pair of fp16 planes (gemm_f16.cu)
    DevBuf<__half> mel_h, mel_l, h1_h, h1_l, xn_h, xn_l, qkv_h, qkv_l, att_h, att_l, hid_h, hid_l, xa_h, xa_l;
    std::vector<std::unique_ptr<GemmF16Plan>> enc_plans;   // conv1, conv2, per encoder layer qkv / out / mlp1 / mlp2, per decoder layer cross K|V
    bool use_tc = true;                // fp16-exact weights: tensor-core encoder; else the fp32 CUDA-core GEMM
    void run_encoder_f16();            // tensor-core encoder
    void run_encoder_f32();            // fp32 CUDA-core encoder (weights that are not fp16-exact)
    DevBuf<float> ckv;     // [L][Mcap][2d]  cross keys (scaled) | values, projected once per window
    DevBuf<float> ckv_tmp; // [Mcap][2d] one layer's projection in GEMM (row-major) order, before the head-major re-layout
    // ---- device: decode state
    DevBuf<float> kc, vc;  // [L][Rmax][t_max][d] self keys (scaled) / values
    DevBuf<__half> kc16, vc16, ckv16;   // fp16 caches (WB_KV_F16)
    DevBuf<float> dx, dq, dhid, logits;
    Dec5Tables d5;                  // decoder5.cu stage descriptors
    DevBuf<uint4> att_pl, hid_pl;   // decoder5.cu activation planes
    DevBuf<float> part_o, part_m, part_l;
    // lengths: [2][Rmax] each row's id count, then each seated row's id limit (DecArgs::lengths)
    DevBuf<int> tokens, lengths, cur_tok, finished, row_window, anc0, anc1, parent, pos, n_unfinished, topk_id;
    DevBuf<float> topk_lp;
    DevBuf<float> token_lp;    // [Rmax][t_max] log-prob of each token the greedy decoders commit (DecArgs::token_lp)
    DevBuf<float> eot_logit;   // [Rmax] raw EOT logit of each row at the current position (greedy loop)
    DevBuf<uint8_t> is_special;
    bool have_special = false;
    int anc_cur = 0;       // which ancestry table is current
    bool anc_identity = true;
    int R = 0;             // live rows
    int host_pos = 0;      // host mirror of *pos
    // pinned host staging of step_beams: [Rmax] rows in, [Rmax][DEC_KC] candidate ids out
    Pinned<int> h_parent, h_window, h_token, h_topk_id;
    // ev[0..3]: timings of the last transcribe call; ev[4], ev[5]: the launch profile_decode times
    cudaEvent_t ev[6] = {};
    // results of the last transcribe / waveform(s)_to_tokens call: timings, search steps, per output row the log-prob of each
    // id (have_logprobs: that call succeeded).  A call rejected before it encodes leaves them as they were.
    float last_ms[4] = {0, 0, 0, 0};
    int64_t last_steps = 0;
    std::vector<std::vector<float>> last_logprobs;
    bool have_logprobs = false;
    // per window of that call (waveform calls: waveform-major) its n-best list; have_nbest: that call succeeded under
    // WB_SEARCH_BEAM (the greedy loop carries no list)
    std::vector<NBest> last_nbest;
    bool have_nbest = false;
    int last_groups = 1;         // row groups (launches) of the last decode
    int last_decoder = 0;        // which persistent decoder the last launch used (6, 5, 4 or 3); 0 = none yet
    int last_rows = 0, last_k = 0;   // rows and candidates per row of the last launch (its topk_id / topk_lp)
    int only_decoder = 0;        // WB200_DECODER=3|4|5|6: every launch uses that decoder or fails; 0 = the first that covers it
    int n_sm = 0;
    DevBuf<DecLayer> dec_layers;
    Dec6Pack d6;                    // decoder6.cu packed weights
    DevBuf<unsigned int> dec_bar;
    DevBuf<int> steps_done;
    DevBuf<float> datt;
    DevBuf<unsigned long long> dec_trace;   // debug: WB200_TRACE=1
    DecArgs dec_base;   // the DecArgs fields that are fixed once the session exists; launch_decoder sets the rest
    // the first persistent decoder that covers the launch; false when a beam search launch is not covered (only decoder6
    // has a beam mode)
    bool launch_decoder(const DecodeLaunch& l);
    // device beam search state (decoder6.cu beam mode), allocated on first use
    DevBuf<int> slot_live, bm_seq, bm_cnt, bm_win, bm_out, bm_out_len;
    DevBuf<float> bm_seq_lp, bm_out_lp;
    DevBuf<beamfx::Head> bm_head;
    DevBuf<float> ypart, lg_m, lg_s, lg_v;
    DevBuf<int> lg_i;
    // the greedy search launch of n_steps positions after the prompt, with no early stop, timed by events
    void profile_decode(const int64_t* prompt, int64_t prompt_len, int n_steps, float* logits_ms, float* step_ms);

    Session(Model* model, int64_t max_windows, int64_t max_beams, int64_t max_text_len, int kv_dtype,
            int window_mode = WB_WINDOWS_REFERENCE);
    ~Session();
    Session(const Session&) = delete;
    Session& operator=(const Session&) = delete;

    // waveforms already in `wave` (device) at offsets[i], lens[i] samples each
    void encode_from_device_wave(const float* wave_dev, const int64_t* offsets, const int64_t* lens, int64_t n);
    void encode_waveforms_host(const float* const* waves, const int64_t* lens, int64_t n);
    void encode_mels_host(const float* mel, int64_t n, int64_t n_mels, int64_t n_ctx);
    // xa rows provided directly (stateless forward_decoder): n windows of T rows each
    void load_encoder_output_host(const float* xa_host, int64_t n, int64_t T);
    void run_encoder();      // conv stems .. ln_post .. cross K/V, from mel_rows
    void run_cross_kv();

    void set_search(int rule) {
        WB_REQUIRE(rule == WB_SEARCH_BEAM || rule == WB_SEARCH_GREEDY_LOOP, "set_search: unknown search rule");
        search = rule;
    }
    void set_prev_prompt(int64_t id) {
        WB_REQUIRE(id == -1 || (id >= 0 && id < m->dims.n_vocab), "set_prev_prompt: startofprev must be -1 or an id in [0, n_vocab)");
        startofprev = id;
    }
    void set_special(const uint8_t* is_special_host);
    // Seats `rows` rows for a new decode from position 0: row r decodes window r / per_window from the tokens of
    // prompts[r / per_window] (token buffer, lengths, id limits prompt length + max_depth); no row is finished and every row
    // reads only its own cache rows
    void seat_rows(int rows, int per_window, const std::vector<std::vector<int64_t>>& prompts, int max_depth = 0);
    // teacher forcing right after seat_rows: positions [0, n) of every row from its token buffer, one cached step each;
    // with logits_out (host), each position's raw logits go to logits_out [R][n][V]
    void feed_positions(int n, float* logits_out);
    // seats window w with prompts[w] (max_depth: the greedy search's steps after each prompt); the prefill feeds the
    // positions before the shortest prompt's last token
    void begin(const std::vector<std::vector<int64_t>>& prompts, bool prefill = true, int max_depth = 0);
    // the stateless forward_decoder: every position's logits [n_rows][seq_len][V] of tokens [n_rows][seq_len]
    void teacher_forced_logits(const int64_t* tokens, int64_t n_rows, int64_t seq_len, float* logits_out);
    void step_beams(int64_t n_rows, const int32_t* window_of_row, const int32_t* parent_row, const int64_t* token,
                    int apply_mask, int k, int64_t* topk_ids_out, float* topk_lp_out);
    // the [n_rows][k] candidates the last launch wrote at its last position
    void last_topk(int64_t n_rows, int64_t k, int64_t* ids_out, float* lp_out);
    // greedy search of window w from prompts[w] on the device in one launch; returns per-window token lists and the log-prob
    // of each token (0 for the prompt, NaN for an EOT a rule appended).  loop_rules: the reference's greedy loop
    // (WB_SEARCH_GREEDY_LOOP) instead of beam_size 1
    void greedy_decode(const std::vector<std::vector<int64_t>>& prompts, int max_depth, int64_t eot,
                       std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp, bool loop_rules = false);
    // the whole beam search (prefill + up to max_depth steps after each window's prompt) of every encoded window in ONE
    // decoder launch; false (nothing decoded) when no decoder covers it, and the caller runs the host search.  nbest: each
    // window's final carried list, ranked
    bool beam_decode(const std::vector<std::vector<int64_t>>& prompts, int beam_size, int max_depth, int64_t eot,
                     std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp, std::vector<NBest>& nbest);
    // teacher-forced scoring of n_seqs packed token sequences (wb_session_score_tokens): per position j >= 1 the log-prob of
    // token j given tokens 0 .. j-1 and the arg-max id; reads the cross K/V of the encoded windows, writes no decode state
    void score_tokens(int64_t n_seqs, const int32_t* window_of_seq, const int64_t* tokens, const int64_t* lens, bool apply_mask,
                      const uint8_t* is_special_host, float* lp_out, int64_t* argmax_out);
    ScoreWs score_ws;
    // the teacher-forced decoder over the M packed rows whose token ids and positions are in score_ws.tok / score_ws.pos (n
    // sequences, rows and windows in score_ws.seqs / score_ws.seq_win, at most max_T rows each): the embedding, then layers
    // 0 .. n_layers - 1.  after_cross_query(l), when set, runs once layer l's scaled cross queries are in score_ws.qkv_h /
    // score_ws.qkv_l; with full = false the last layer stops there
    void decoder_pass(int M, int n, int max_T, int n_layers, bool full, const std::function<void(int)>& after_cross_query);
    // token alignment (align.cu, wb_session_align_tokens): per aligned id its start and end encoder position on the DTW path
    // through the cross-attention matrix of the selected heads; writes no decode state
    void align_tokens(int64_t n_seqs, const int32_t* window_of_seq, const int64_t* tokens, const int64_t* lens, const int64_t* first,
                      int64_t n_heads, const int32_t* heads, int32_t* start_out, int32_t* end_out, float* matrix_out,
                      int64_t matrix_capacity);
    AlignWs align_ws;
};

// host pipeline (transcribe.cu).  window_prompts checks every argument of a decode call and builds each window's prompt
// (transcribe.rs:195-203 without the shadowing at :201): [startofprev] + prev[w] + [sot, lang, transcribe, notimestamps],
// or the four ids where prev[w] (mels_to_text's prev_nonspecial_tokens) is empty or prev is.
std::vector<std::vector<int64_t>> window_prompts(const Session& s, int64_t n_windows, int beam_size, int max_depth,
                                                 const wb_special_ids& ids, const uint8_t* is_special,
                                                 const std::vector<std::vector<int64_t>>& prev = {}, int64_t startofprev = -1);
// transcribe_windows runs `encode` (prompts.size() windows), then decodes each window from its prompt.  Both it and
// waveforms_to_tokens return at most capacity ids per row and leave the ids' log-probs and the timings in s.
std::vector<std::vector<int64_t>> transcribe_windows(Session& s, const std::vector<std::vector<int64_t>>& prompts, int beam_size,
                                                     int max_depth, int64_t eot, const uint8_t* is_special, int64_t capacity,
                                                     const std::function<void()>& encode);
std::vector<std::vector<int64_t>> waveforms_to_tokens(Session& s, const float* const* waveforms, const int64_t* n_samples,
                                                      int64_t n_waveforms, int64_t sample_rate, int beam_size, int max_depth,
                                                      const wb_special_ids& ids, const uint8_t* is_special, int64_t capacity);
// waveforms_to_tokens over waveforms of any supported rate and channel count: every argument checked, the interleaved inputs
// uploaded and resampled to 16 kHz mono into s.rs in one launch, then the same window loop with windows cut on the device
std::vector<std::vector<int64_t>> waveforms_to_tokens_resampled(Session& s, const float* const* waveforms, const int64_t* n_frames,
                                                                const int64_t* channels, const int64_t* sample_rates,
                                                                int64_t n_waveforms, int beam_size, int max_depth,
                                                                const wb_special_ids& ids, const uint8_t* is_special,
                                                                int64_t capacity);
std::vector<std::pair<int64_t, int64_t>> window_bounds(int64_t n_samples, int64_t sample_rate, int64_t window_len);
bool find_chunk_overlap(const int64_t* prev, int64_t n_prev, const int64_t* curr, int64_t n_curr, int64_t max_n_offsets,
                        int64_t min_n_overlaps, int64_t* prev_index, int64_t* curr_index);

// align.cu: whether the DTW kernel takes an [N][C] matrix (N <= 448 and its 2-bit trace fits one CTA's shared memory); the DTW
// of one host matrix on the current device (wb_align_dtw) -> start / end per row
bool dtw_fits(int64_t N, int64_t C);
void align_dtw(const float* matrix, int64_t N, int64_t C, int32_t* start_out, int32_t* end_out);

// wav.cu: load_audio_waveform (src/bin/transcribe/main.rs:31-55)
void load_wav(const std::string& path, bool strict, std::vector<float>& out, int64_t& sample_rate, int& channels);

// npytree.cu: the reference's model-file format (src/model/load.rs, python/dump.py)
void npy_tree_probe(const std::string& dir, wb_dims& dims);
void npy_tree_load(Model& m, const std::string& dir);

// model.cu
void model_set_tensor(Model& m, const char* path, const float* data, const int64_t* shape, int ndim);
void model_finalize(Model& m);
const std::string& last_error_string();

}  // namespace wb
