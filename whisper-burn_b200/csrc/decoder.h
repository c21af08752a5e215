// Argument blocks of the persistent decoder kernels.  Internal.
#pragma once
#include <stdint.h>

#include "../host/beam.hpp"
#include "wb_internal.h"

namespace wb {

constexpr int DEC_KC = 8;   // top candidates a persistent decoder keeps per record (k <= 7)
// DecArgs::mask_mode: when the vocabulary stage masks the special ids (is_special): never, at every position, or while the
// sequence has at most 5 tokens (transcribe.rs:271-275; dec_common.cuh SPECIAL_MASKED)
constexpr int MASK_NONE = 0, MASK_ALWAYS = 1, MASK_SHORT = 2;

// ---- persistent decoders (decoder3.cu .. decoder6.cu) -------------------------------------------------
struct DecLayer {
    const float *ln1_g, *ln1_b, *ln2_g, *ln2_b, *ln3_g, *ln3_b;
    float ln1_eps, ln2_eps, ln3_eps;
    const void *Wqkv, *Wo, *Wcq, *Wco, *W1, *W2;     // [N][K] fp16 or fp32
    const float *bqkv, *bo, *bcq, *bco, *b1, *b2;
};
// decoder5.cu stage descriptors, built on the host: entry [l * 16 + slot] for the stage slots of layer l (LN1, QKV, SELF, OUT, LN2,
// CQ, CROSS, COUT, LN3, MLP1, MLP2 = 0..10), entries [L * 16 + 11] / [L * 16 + 12] for the final LayerNorm and the logits.
enum { D5_KIND_LN = 0, D5_KIND_ATTN, D5_KIND_GEMM };
enum { D5_ST_LN_EMB = 0, D5_ST_LN_FOLD, D5_ST_LN_FOLD_NOPUB, D5_ST_LN_X, D5_ST_PLANES, D5_ST_CROSS };
enum { D5_EM_QKV = 0, D5_EM_RESID, D5_EM_CQ, D5_EM_HID, D5_EM_PART, D5_EM_LOGITS };
struct Dec5Desc {
    int kind = D5_KIND_ATTN;
    const void* W = nullptr;       // [N][n_slabs * d] fp16
    const float* bias = nullptr;
    int N = 0, n_slabs = 1, stage = 0, emit = 0;
    const float *g = nullptr, *b = nullptr;   // LayerNorm parameters (D5_KIND_LN)
    float eps = 0.0f;
    int src = 0;                   // input planes of a linear stage: 1 = attention output, 2 = MLP hidden, 3 = LayerNorm output
    int ks = 0;                    // K slab width of a linear stage (= columns staged per item); d except MLP2 when 4d splits into 3
    int n_fold = 0;                // LayerNorm stage: K-slab partial sums (ypart) folded into x first (the producing stage's n_slabs)
    int pad_[2] = {0, 0};          // sizeof % 16 == 0: the table is copied to shared memory in 16-byte words
};
static_assert(sizeof(Dec5Desc) % 16 == 0, "Dec5Desc must be a whole number of 16-byte words");
struct DecArgs {
    int R = 0, Rmax = 0, d = 0, H = 0, L = 0, V = 0, t_max = 0;
    int64_t Mcap = 0;
    int eps_outside = 1;
    float qk_scale = 1.0f;
    const DecLayer* layers = nullptr;    // device array [L]
    const float* tok_emb = nullptr;       // fp32 [V][d] (embedding lookup)
    const float* pos_emb = nullptr;
    const void* E = nullptr;              // logits matrix [V][d] fp16 or fp32
    const void* E_tiled = nullptr;        // decoder4.cu: the same matrix as contiguous half-tiles [ceil(V/16)][2][16][d/2] fp16
    const float *lnf_g = nullptr, *lnf_b = nullptr;
    float lnf_eps = 1e-5f;
    // state
    float *x = nullptr, *q = nullptr, *att = nullptr, *hid = nullptr;
    float* ypart = nullptr;                 // decoder5.cu: MLP2 partial sums [n_slabs][R][d], folded by the next LayerNorm stage
    const Dec5Desc* d5 = nullptr;           // decoder5.cu: device array [L * 8 + 1]
    void *att_pl = nullptr, *hid_pl = nullptr;   // decoder5.cu: fragment-order fp16 hi/lo planes of the attention output / MLP hidden layer
    float* lgbuf = nullptr;                 // decoder5.cu: [R][V] logits scratch (== logits_out when that is requested)
    int lg_slices = 1;                      // decoder5.cu: vocabulary slices per row in the softmax / candidate stage
    void *kc = nullptr, *vc = nullptr;    // [L][Rmax][t_max][d]  fp32 or fp16 (kv_half)
    const void* ckv = nullptr;            // [L][Mcap][2d] cross K/V, head-major per window (encoder.cu ckv_relayout_kernel)
    int kv_half = 0;
    int kv_row0 = 0;                      // decoder5.cu row groups: local row r of this launch is cache row r + kv_row0 (ancestry entries are absolute)
    const int* row_window = nullptr;
    const int64_t* win_row_off = nullptr;
    const int* win_T = nullptr;
    const int* anc = nullptr;
    int n_splits = 1;
    float *part_o = nullptr, *part_m = nullptr, *part_l = nullptr;   // [R][H][S][64], [R][H][S]
    // tokens / control
    int* tokens = nullptr;                // [Rmax][t_max]
    float* token_lp = nullptr;            // [Rmax][t_max] log-prob of each committed token (greedy_commit), NaN where a rule put EOT
    const int* cur_tok = nullptr;
    int use_cur_tok = 0;
    int pos0 = 0, n_steps = 1, logits_from = 0;
    const uint8_t* is_special = nullptr;
    int mask_mode = 0;
    int k = 1, greedy = 0, eot = -1;
    // lengths [R] ids of each row (the prompt length until its first commit); behind them, lengths[Rmax + r], the most ids
    // the row may hold, its prompt length + max_depth (Session::seat_rows, dec_common.cuh id_limit): kept in the same buffer
    // so that DecArgs, which decoder6's register allocation is sensitive to, does not grow, and decoder5's row groups offset
    // both with one pointer
    int *lengths = nullptr, *finished = nullptr;
    // greedy loop (WB_SEARCH_GREEDY_LOOP, host/loop_rules.hpp): the row finish also applies the EOT test and the repetition
    // cut (dec_common.cuh loop_finish); the vocabulary stage stores each row's raw EOT logit in eot_logit [R].  The context
    // stop is the launch's n_steps.
    int loop_rules = 0;
    float* eot_logit = nullptr;
    int *topk_id = nullptr;
    float* topk_lp = nullptr;
    float* logits_out = nullptr;
    float *lg_m = nullptr, *lg_s = nullptr, *lg_v = nullptr;
    int* lg_i = nullptr;
    int *pos = nullptr, *n_unfinished = nullptr, *steps_done = nullptr;
    unsigned int* bar = nullptr;          // [4] arrival count, generation / ticket, finish flag (decoder6.cu)
    const void* d6_pack = nullptr;        // decoder6.cu: packed weight slices [L][CS][PACK] bytes
    const float* d6_params = nullptr;     // decoder6.cu: parameter blocks [L][CS][PARAMS] floats
    unsigned long long* trace = nullptr;  // optional: stage / barrier timestamps of CTA 0 (ns)
    int trace_cap = 0;
    // decoder6.cu beam mode (beam > 1): prefill + the whole width-B search of n_win windows in one launch.  Row w * B + i is
    // slot i of window w; anc (read at even depths) / anc_alt (odd depths) are the double-buffered ancestry tables.
    // max_depth: search steps after each row's own prompt (greedy and beam mode).
    int beam = 0, n_win = 0, max_depth = 0;
    int* anc_alt = nullptr;
    int* slot_live = nullptr;             // [R] the slot holds a live beam at the current position
    beamfx::Head* bm_head = nullptr;      // [2][n_win][MAX_NODES] carried nodes, double-buffered by depth
    int* bm_seq = nullptr;                // [2][n_win][MAX_NODES][t_max] their token sequences
    float* bm_seq_lp = nullptr;           // [2][n_win][MAX_NODES][t_max] the log-prob each token was scored with (0 for the prompt)
    int* bm_cnt = nullptr;                // [2][n_win] carried nodes per window
    int* bm_win = nullptr;                // [n_win][2] current buffer, done
    int* bm_out = nullptr;                // [n_win][t_max] best sequence of each window when the search ends
    float* bm_out_lp = nullptr;           // [n_win][t_max] its log-probs
    int* bm_out_len = nullptr;            // [n_win]
};
// Each launch_decN launches decoder N when it covers the configuration and reports whether it did.
// grid-barrier FMA decoder (decoder3.cu): covers every configuration
void launch_dec3(const DecArgs& a, int n_ctas, bool w_half, cudaStream_t st);
// cluster / DSMEM decoder (decoder4.cu): greedy, d in {128, 384}, as many rows (<= 8) as co-resident 16-CTA clusters
bool launch_dec4(const DecArgs& a, bool w_half, cudaStream_t st);
// head-fused tensor-core cluster decoder (decoder6.cu): fp16-exact weights, d in {128, 384}, <= 24 rows, t_max <= 128; greedy,
// or (a.beam > 1) the whole beam search
struct Dec6Pack {   // this model's weights as per-CTA slices (built on the first launch)
    DevBuf<uint8_t> pack;   // [L][CS][PACK] bytes
    DevBuf<float> params;   // [L][CS][PARAMS] floats
};
bool launch_dec6(DecArgs a, const Model& m, Dec6Pack& pack, cudaStream_t st);
// batched tensor-core decoder (decoder5.cu): fp16-exact weights, d % 256 == 0; more than 32 rows run as row groups of 32.
// Returns the number of launches, 0 when the configuration is not covered.
struct Dec5Tables {   // stage descriptors (Dec5Desc)
    DevBuf<Dec5Desc> unsplit;   // the d x d projections unsplit
    DevBuf<Dec5Desc> split;     // the same as K slabs (launches whose cross attention is not split over keys); may be empty
};
void dec5_build_tables(const Model& m, int n_sm, Dec5Tables& t);   // nothing unless the weights are fp16-exact
int launch_dec5(const DecArgs& a, const Dec5Tables& t, int n_ctas, bool w_half, cudaStream_t st);
size_t dec5_plane_uint4(int d);   // uint4 elements of one global activation plane

void launch_dec_anc_identity(int* anc, int R, int t_max, cudaStream_t st);
void launch_dec_reorder(const int* anc_old, int* anc_new, const int* parent, const int* pos_ptr, int R, int t_max,
                        cudaStream_t st);

}  // namespace wb
