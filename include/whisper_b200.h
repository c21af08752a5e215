/* whisper_b200.h -- C ABI of the H100-native Whisper hot path (libwhisper_b200.so).
 *
 * The reference (Gadersd/whisper-burn) has no FFI: its hot path is Rust generic over
 * burn::tensor::backend::Backend.  This header is the boundary a thin Rust shim (rust/ in
 * this repo, INTEGRATION.md) binds with `extern "C"` so that whisper-burn's own public
 * functions keep their signatures while every tensor op runs in hand-written sm_90a CUDA:
 *
 *   audio::max_waveform_samples        src/audio.rs:12-17          -> wb_max_waveform_samples
 *   audio::prep_audio                  src/audio.rs:34-56          -> wb_prep_audio
 *   `sox audio.wav -r 16000 -c 1` step README.md:69-73 (no reference code) -> wb_resample, wb_waveforms_to_tokens_resampled
 *   WhisperConfig / Whisper            src/model/mod.rs:16-71      -> wb_model_*
 *   model::load::load_whisper          src/model/load.rs:295-310   -> wb_model_set_tensor (same npy-tree paths)
 *   Whisper::forward_encoder           src/model/mod.rs:52-54      -> wb_forward_encoder
 *   Whisper::forward_decoder           src/model/mod.rs:56-62      -> wb_forward_decoder
 *   Whisper::{encoder,decoder}_ctx_size src/model/mod.rs:64-70     -> wb_model_get_dims
 *   beamsearch_next closure            src/transcribe.rs:253-307   -> wb_session_step (KV-cached, top-k only)
 *   forward_decoder + log_softmax      mod.rs:131-157, transcribe.rs:276 -> wb_session_score_tokens (every position)
 *   beam::beam_search(_step)           src/beam.rs:9-79            -> wb_beam_* (host C++, same tie-breaks)
 *   beam_search's final carried list   src/beam.rs:33-36           -> wb_session_last_nbest (the n-best the search drops)
 *   mels_to_text (token part)          src/transcribe.rs:148-383   -> wb_transcribe_windows
 *   waveform_to_text (token part)      src/transcribe.rs:23-74     -> wb_waveform_to_tokens
 *   find_chunk_overlap                 src/transcribe.rs:76-110    -> wb_find_chunk_overlap
 *   first_repetition_end / repetition_period / find_repeated_tokens_index
 *                                      src/transcribe.rs:385-447   -> wb_first_repetition_end, wb_repetition_period,
 *                                                                     wb_find_repeated_tokens_index (compiled but unused there)
 *
 * Conventions (SURVEY.md 8b):
 *   - plain pointers and sizes only; host buffers are caller-owned and only read/written
 *     during the call; every call is synchronous from the caller's point of view.
 *   - every function returns an int status (WB_OK == 0).  WB_ERR_INVALID_ARG marks what the
 *     reference treats as a contract violation (assert!/panic: shapes, n < 400 samples, ...);
 *     the Rust shim turns it into panic!, everything else into Err.  wb_last_error() returns a
 *     thread-local message.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     WB_ERR_CUDA.
 *   - a wb_model is immutable after wb_model_finalize and may be shared by threads; a
 *     wb_session (KV caches, workspaces, one CUDA stream) is used by one thread at a time.
 *   - `*_dev` variants take device pointers on the model's device (inputs resident in HBM).
 */
#ifndef WHISPER_B200_H
#define WHISPER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WB_OK 0
#define WB_ERR_INVALID_ARG 1   /* reference would assert!/panic */
#define WB_ERR_CUDA 2          /* no device / CUDA runtime failure */
#define WB_ERR_OOM 3
#define WB_ERR_STATE 4         /* call order violated (e.g. model not finalized) */
#define WB_ERR_UNSUPPORTED 5

#define WB_KV_F32 0            /* reference numerics */
#define WB_KV_F16 1            /* fp16 K/V cache (north_star); rounding restated by the oracle's kv_dtype="f16" */

/* Window modes of a session: the most mel frames one window gives the encoder.  Everything else of the reference's
 * windowing (10 zero frames appended, 3 s overlap, overlap merge, prompt, beam rules) is the same in both.
 *   REFERENCE: n_audio_ctx mel frames, as the reference (transcribe.rs:32-34, 161-177): a window keeps at most
 *              n_audio_ctx - 10 frames, so T <= n_audio_ctx / 2 encoder positions (750 for Whisper: a 30 s chunk is
 *              3 windows).  The default, and the mode the reference's outputs are compared in.
 *   NATIVE:    2 * n_audio_ctx mel frames: a window keeps at most 2 * n_audio_ctx - 10 frames, T <= n_audio_ctx
 *              (1500 for Whisper: the 30 s context the models were trained on; 480 000 samples give one window of
 *              T = 1500, the last 0.1 s clipped as in the reference).  Buffers sized per window double. */
#define WB_WINDOWS_REFERENCE 0
#define WB_WINDOWS_NATIVE 1

/* Search rules of a session (wb_session_set_search): how wb_transcribe_windows[_dev] and wb_waveform(s)_to_tokens pick tokens.
 *   BEAM:        the reference's beam::beam_search (transcribe.rs:232-309) with beam_size / max_depth; greedy is beam_size 1.
 *                The special ids are masked while a sequence has at most 5 tokens.  The default.
 *   GREEDY_LOOP: the greedy loop the reference leaves commented out (transcribe.rs:314-380).  At each step the arg-max of
 *                the raw logits (no special-token mask; is_special is ignored and may be NULL) is appended, then
 *                - EOT test: when exp(eot_logit - token_logit) > 0.5 (f64 on the two f32 logits) the window ends, with EOT
 *                  appended unless the arg-max was EOT;
 *                - repetition cut: when find_repeated_tokens_index(tokens, 5, 4) (the whole sequence, prompt included)
 *                  finds (first, end), the sequence is cut to `end` tokens and EOT appended;
 *                - context stop: a sequence of min(n_text_ctx, 4 + max_depth) tokens gets EOT appended.
 *                beam_size must be 1 (WB_ERR_INVALID_ARG otherwise), and every window ends in EOT, so an output row holds
 *                up to 4 + max_depth + 1 ids.  max_depth = n_text_ctx - 4 on a session with max_text_len = n_text_ctx is
 *                the reference's loop exactly.  Windowing and the overlap merge are those of both window modes. */
#define WB_SEARCH_BEAM 0
#define WB_SEARCH_GREEDY_LOOP 1

typedef struct wb_model wb_model;
typedef struct wb_session wb_session;

/* WhisperConfig = AudioEncoderConfig + TextDecoderConfig (src/model/mod.rs:16-39,73-80,164-171) */
typedef struct wb_dims {
    int32_t n_mels, n_audio_ctx, n_audio_state, n_audio_head, n_audio_layer;
    int32_t n_vocab, n_text_ctx, n_text_state, n_text_head, n_text_layer;
} wb_dims;

/* the ids mels_to_text looks up in the tokenizer (src/transcribe.rs:179-185); the tokenizer
 * itself (src/token.rs) stays on the caller's side of the boundary */
typedef struct wb_special_ids {
    int64_t sot, lang, transcribe, notimestamps, eot;
} wb_special_ids;

const char* wb_version(void);
const char* wb_last_error(void);
int wb_device_count(int* n_out);

/* ---- audio.rs ---------------------------------------------------------------------- */
/* audio.rs:12-17 */
int64_t wb_max_waveform_samples(int64_t n_frame_max);
/* Samples of one window in a window mode (transcribe.rs:32-34 with that mode's frame limit): the window_len of
 * wb_window_bounds.  WB_WINDOWS_REFERENCE gives wb_max_waveform_samples(n_audio_ctx - 10) (238 559 for Whisper),
 * WB_WINDOWS_NATIVE wb_max_waveform_samples(2 * n_audio_ctx - 10) (478 559).  -1 for an unknown mode or n_audio_ctx <= 10. */
int64_t wb_window_samples(int64_t n_audio_ctx, int window_mode);
/* audio.rs:34-56: wave [n_batch, n_samples] -> mel_out [n_batch, 80, n_samples/160] (f32, row-major).
 * The max of audio.rs:50 is taken over the whole call (all batches), as in the reference.
 * WB_ERR_INVALID_ARG if n_samples < 400 (audio.rs:292). */
int wb_prep_audio(int device, const float* wave, int64_t n_batch, int64_t n_samples,
                  float* mel_out, int64_t* n_frames_out);
int wb_prep_audio_dev(int device, const float* wave_dev, int64_t n_batch, int64_t n_samples,
                      float* mel_out_dev, int64_t* n_frames_out);
/* Downmix and resampling to the 16 kHz mono every other entry point takes; the reference has none (its README converts
 * with sox first, its binary asserts 16 kHz mono).  An input of n_frames x channels interleaved f32 samples at an integer
 * sample_rate is downmixed, x[i] = (x[i,0] + .. + x[i,C-1]) / C (f64, channel order), and resampled as
 * scipy.signal.resample_poly(x, up, down) with its defaults: g = gcd(sample_rate, 16000), up = 16000 / g, down =
 * sample_rate / g, supported when sample_rate >= 1 and max(up, down) <= 1024 (8000, 11025, 22050, 44100, 48000, 96000,
 * 192000 Hz, ...); a Kaiser (beta 5) low-pass of 2 * 10 * max(up, down) + 1 taps designed in f64, products and sums in f64,
 * each output rounded once to f32.  16 kHz mono passes through bit-unchanged.
 * wb_resampled_length: the output length ceil(n_frames * up / down) (host only); -1 for an unsupported rate or n_frames < 0. */
int64_t wb_resampled_length(int64_t n_frames, int64_t sample_rate);
/* in [n_frames][channels] (host) -> out [*n_out] (host, 16 kHz mono), *n_out = wb_resampled_length(n_frames, sample_rate).
 * WB_ERR_UNSUPPORTED for an unsupported rate; WB_ERR_INVALID_ARG for a null pointer, n_frames < 1, channels < 1 or capacity
 * below the output length.  Both are reported before the device is touched. */
int wb_resample(int device, const float* in, int64_t n_frames, int64_t channels, int64_t sample_rate, float* out,
                int64_t capacity, int64_t* n_out);

/* ---- model (src/model/mod.rs, src/model/load.rs) ------------------------------------- */
int wb_model_create(const wb_dims* dims, int device, wb_model** out);
/* `path` is the reference's npy-tree path without ".npy" (load.rs:29-45, dump.py:130-213), e.g.
 * "encoder/block_0/attn/query/weight".  Linear weights are burn layout [d_in, d_out]
 * (dump.py:141-145), Conv1d weights [out, in, k], embeddings [rows, d], LayerNorm eps is a
 * 1-element tensor.  Data is copied. */
int wb_model_set_tensor(wb_model* m, const char* path, const float* data, const int64_t* shape, int ndim);
/* model::load::load_whisper (src/model/load.rs:295-310): builds a finalized model from the npy tree that
 * python/dump.py writes (one f32 .npy per tensor, payload = [dims..., values...], scalars as [1.0, value]);
 * the dimensions come from the tree itself.  wb_npy_tree_probe only reads the dimensions (host only). */
int wb_npy_tree_probe(const char* dir, wb_dims* dims_out);
int wb_model_load_npy_tree(const char* dir, int device, int ln_eps_outside, wb_model** out);
/* burn's nn::LayerNorm is third-party and un-vendored: burn 0.9 (the reference's pin, Cargo.lock:242-244)
 * normalises by (sqrt(var) + eps); later burn releases by sqrt(var + eps).  outside != 0 selects the
 * former (default).  Must be called before wb_model_finalize. */
int wb_model_set_layernorm_eps_mode(wb_model* m, int outside);
/* Validates that every tensor of the tree is present, uploads and re-lays the weights. */
int wb_model_finalize(wb_model* m);
void wb_model_destroy(wb_model* m);
int wb_model_get_dims(const wb_model* m, wb_dims* out);
/* 1 if every weight is exactly representable in fp16 (true for OpenAI checkpoints) and the
 * compact fp16 decoder weight storage is in use, 0 if weights are kept in fp32. */
int wb_model_weights_fp16_exact(const wb_model* m);

/* mod.rs:52-54 / 228-260: mel [n_batch, n_mels, n_ctx] -> out [n_batch, (n_ctx-1)/2+1, d].
 * WB_ERR_INVALID_ARG if n_mels != 80-config or n_ctx > n_audio_ctx (mod.rs:231-241). */
int wb_forward_encoder(wb_model* m, const float* mel, int64_t n_batch, int64_t n_mels, int64_t n_ctx,
                       float* out);
/* mod.rs:56-62 / 131-157, stateless: tokens [n_batch, seq_len] (i64), encoder_output
 * [n_batch, n_audio_ctx_used, d] -> logits_out [n_batch, seq_len, n_vocab].
 * WB_ERR_INVALID_ARG if seq_len > n_text_ctx (mod.rs:134-139). */
int wb_forward_decoder(wb_model* m, const int64_t* tokens, int64_t n_batch, int64_t seq_len,
                       const float* encoder_output, int64_t n_enc_ctx, float* logits_out);

/* ---- KV-cached decoding session -------------------------------------------------------- */
/* A session holds, for up to max_windows audio windows x max_beams live beams each: encoder
 * output, per-layer cross K/V (computed once per window), per-layer self K/V for
 * max_text_len positions, and all workspaces.  max_beams <= 7 and k <= 7 in wb_session_step (the decoders keep 8 candidates per
 * record; the reference searches with width 5, src/transcribe.rs:232); larger values are rejected with WB_ERR_INVALID_ARG.
 * wb_session_create makes a WB_WINDOWS_REFERENCE session; wb_session_create_windows takes the window mode (WB_WINDOWS_*),
 * which sets the frame limit of every call below: encode_waveforms clips windows at limit - 10 frames, encode_mels takes
 * n_ctx <= limit, get_mel / get_encoder_output return up to limit / (limit - 1) / 2 + 1 rows per window, and
 * waveform(s)_to_tokens cut windows of wb_window_samples(n_audio_ctx, mode) samples.  A native session holds twice the
 * per-window encoder and cross K/V memory of a reference one. */
int wb_session_create(wb_model* m, int64_t max_windows, int64_t max_beams, int64_t max_text_len,
                      int kv_dtype, wb_session** out);
int wb_session_create_windows(wb_model* m, int64_t max_windows, int64_t max_beams, int64_t max_text_len,
                              int kv_dtype, int window_mode, wb_session** out);
void wb_session_destroy(wb_session* s);
/* Sets the search rule (WB_SEARCH_*) of the session's decode calls; WB_ERR_INVALID_ARG on an unknown rule. */
int wb_session_set_search(wb_session* s, int rule);
/* The previous-text prompt of wb_waveform(s)_to_tokens (the prompt transcribe.rs:43-54, 195-199 builds and line 201
 * shadows).  startofprev = -1 (the default) keeps the 4-id prompt.  An id in [0, n_vocab), the tokenizer's
 * <|startofprev|>, prompts window i of a waveform with [startofprev] + prev + [sot, lang, transcribe, notimestamps], prev =
 * the last (at most) 5 ids of that waveform's merged ids so far with is_special 0, in order (window 0: the 4 ids alone).
 * A waveform's windows are then decoded in order: round i decodes window i of every waveform that has one, so the rule is
 * slower than the default.  is_special must be given, and the rule does not combine with WB_SEARCH_GREEDY_LOOP
 * (WB_ERR_INVALID_ARG from the waveform call); WB_ERR_INVALID_ARG here for any other id. */
int wb_session_set_prev_prompt(wb_session* s, int64_t startofprev);
/* prep_audio + mel padding of mels_to_text (transcribe.rs:161-177) + forward_encoder + cross
 * K/V for n_windows waveforms; waves[i] has lens[i] samples (ragged; each >= 400). */
int wb_session_encode_waveforms(wb_session* s, const float* const* waves, const int64_t* lens,
                                int64_t n_windows);
/* same, windows already on the device, concatenated: window i = wave_dev[offsets[i] .. +lens[i]) */
int wb_session_encode_waveforms_dev(wb_session* s, const float* wave_dev, const int64_t* offsets,
                                    const int64_t* lens, int64_t n_windows);
/* forward_encoder + cross K/V from caller-provided mels [n_windows, n_mels, n_ctx] (no padding added); n_ctx up to the
 * session's frame limit (n_audio_ctx, or 2 * n_audio_ctx in WB_WINDOWS_NATIVE), WB_ERR_INVALID_ARG above it */
int wb_session_encode_mels(wb_session* s, const float* mel, int64_t n_windows, int64_t n_mels, int64_t n_ctx);
/* copies the session's padded mel [n_windows, 80, n_ctx] / encoder output [n_ctx_enc, d] of one window */
int wb_session_get_mel(wb_session* s, int64_t window, float* mel_out, int64_t capacity, int64_t* n_ctx_out);
int wb_session_get_encoder_output(wb_session* s, int64_t window, float* out, int64_t capacity, int64_t* n_ctx_out);
/* Starts decoding: clears the self K/V and feeds prompt[0 .. prompt_len-1) to one beam per window. */
int wb_session_begin(wb_session* s, const int64_t* prompt, int64_t prompt_len);
/* One beamsearch_next evaluation (transcribe.rs:253-307) for n_rows live beams:
 *   row r continues cache row parent_row[r] of window window_of_row[r] with token[r];
 *   apply_special_mask != 0 adds -inf on ids with is_special[id] != 0 (transcribe.rs:271-275);
 *   returns, per row, the k best (token id, f32 log-prob) of log_softmax over the vocabulary,
 *   ordered best first, ties broken towards the lower id (what beam.rs:81-110 keeps).
 * Rows of one window must be contiguous and use slots 0..n-1 of that window in order. */
int wb_session_step(wb_session* s, int64_t n_rows, const int32_t* window_of_row, const int32_t* parent_row,
                    const int64_t* token, int apply_special_mask, const uint8_t* is_special,
                    int k, int64_t* topk_ids_out, float* topk_logprob_out);

/* ---- transcribe.rs (token side) ---------------------------------------------------------- */
/* mels_to_text for a batch of independent windows: encode, then beam::beam_search with
 * beam_size / max_depth (reference: 5 / 100; greedy = beam_size 1).  tokens_out is
 * [n_windows, capacity]; each row gets prompt + generated ids (incl. EOT if reached).
 * Beam search (beam_size > 1) runs entirely on the GPU in one decoder launch (prefill + every search step, selection
 * included) when the weights are fp16-exact, n_text_state is 128 or 384, n_windows * beam_size <= 24 and
 * max_text_len <= 128; otherwise the host drives the search one batched device step per depth.  Both give the same ids. */
int wb_transcribe_windows(wb_session* s, const float* const* waves, const int64_t* lens, int64_t n_windows,
                          int beam_size, int max_depth, const wb_special_ids* ids, const uint8_t* is_special,
                          int64_t* tokens_out, int64_t capacity, int64_t* lens_out);
int wb_transcribe_windows_dev(wb_session* s, const float* wave_dev, const int64_t* offsets, const int64_t* lens,
                              int64_t n_windows, int beam_size, int max_depth, const wb_special_ids* ids,
                              const uint8_t* is_special, int64_t* tokens_out, int64_t capacity, int64_t* lens_out);
/* wb_transcribe_windows with mels_to_text's prev_nonspecial_tokens given per window (transcribe.rs:195-203 without the
 * shadowing at :201).  Window w's previous ids are prev_tokens[off_w .. off_w + prev_lens[w]), off_w = prev_lens[0] + .. +
 * prev_lens[w-1] (packed as wb_session_score_tokens packs its sequences; prev_tokens may be NULL when every prev_lens is 0).
 * Its prompt is [startofprev] + those ids + [sot, lang, transcribe, notimestamps], or the 4 ids when prev_lens[w] = 0.
 * Windows with prompts of different lengths share one decoder launch.  The search rules apply per window at absolute
 * positions: the special ids are masked while a sequence has at most 5 tokens (never for a prompt of 6 or more), and
 * max_depth counts steps after the window's own prompt.  Rows are written as wb_transcribe_windows writes them, prompt
 * included, and wb_session_last_logprobs gives 0.0 for every prompt id.  WB_ERR_INVALID_ARG for startofprev or a previous
 * id outside [0, n_vocab), a negative prev_lens entry, Lp + max_depth > max_text_len or capacity < Lp + max_depth + 1 (Lp:
 * the longest prompt), and for any previous ids under WB_SEARCH_GREEDY_LOOP (the greedy loop builds its own prompt). */
int wb_transcribe_windows_prev(wb_session* s, const float* const* waves, const int64_t* lens, int64_t n_windows,
                               const int64_t* prev_tokens, const int64_t* prev_lens, int64_t startofprev, int beam_size,
                               int max_depth, const wb_special_ids* ids, const uint8_t* is_special, int64_t* tokens_out,
                               int64_t capacity, int64_t* lens_out);
/* waveform_to_text without detokenisation: windowing (transcribe.rs:114-138), per-window
 * decoding, overlap merge (transcribe.rs:56-63).  Writes the merged ids.
 * sample_rate must be 16000 (WB_ERR_INVALID_ARG otherwise): the log-mel tables are the 16 kHz ones the reference's binary
 * always uses (src/bin/transcribe/main.rs:38-41); wb_prep_audio likewise assumes 16 kHz input. */
int wb_waveform_to_tokens(wb_session* s, const float* waveform, int64_t n_samples, int64_t sample_rate,
                          int beam_size, int max_depth, const wb_special_ids* ids, const uint8_t* is_special,
                          int64_t* tokens_out, int64_t capacity, int64_t* n_tokens_out);
/* The same for n_waveforms independent waveforms at once (the unit BASELINE.json shards over GPUs: "8x30 s chunks
 * batched"): the windows of all waveforms are decoded in one batch, each waveform's windows are merged in order.
 * tokens_out is [n_waveforms][capacity], n_tokens_out [n_waveforms]. */
int wb_waveforms_to_tokens(wb_session* s, const float* const* waveforms, const int64_t* n_samples, int64_t n_waveforms,
                           int64_t sample_rate, int beam_size, int max_depth, const wb_special_ids* ids,
                           const uint8_t* is_special, int64_t* tokens_out, int64_t capacity, int64_t* n_tokens_out);
/* wb_waveforms_to_tokens for waveforms of any supported rate and channel count: waveform w is n_frames[w] x channels[w]
 * interleaved f32 samples at sample_rates[w] (rates and channel counts may differ within a call).  All inputs are uploaded
 * once and converted to 16 kHz mono in one launch (wb_resample's definition, same values); then the windows of the converted
 * waveforms (wb_window_bounds at 16 kHz) are cut on the device and decoded exactly as wb_waveforms_to_tokens decodes the
 * converted audio: search rule, previous-text prompt, max_windows batching, overlap merge.  wb_session_last_logprobs /
 * last_nbest / last_timings / last_steps mean what they mean after wb_waveforms_to_tokens.  Every argument that does not
 * depend on decoded ids is checked before the upload: null pointers, n_waveforms >= 1, n_frames >= 1, channels >= 1, a
 * supported rate (WB_ERR_UNSUPPORTED), a last window of at least 400 converted samples (WB_ERR_INVALID_ARG, audio.rs:292) and
 * the decode arguments; a call rejected there leaves the encoded windows and every wb_session_last_* result as they were.
 * The session keeps the inputs and their conversions in device buffers grown to the largest call: 4 * (n_frames * channels +
 * n_out) bytes summed over the call's waveforms (n_out = wb_resampled_length), plus the filters (at most 160 KB per rate). */
int wb_waveforms_to_tokens_resampled(wb_session* s, const float* const* waveforms, const int64_t* n_frames, const int64_t* channels,
                                     const int64_t* sample_rates, int64_t n_waveforms, int beam_size, int max_depth,
                                     const wb_special_ids* ids, const uint8_t* is_special, int64_t* tokens_out, int64_t capacity,
                                     int64_t* n_tokens_out);
/* Per-token log-probs of the last wb_transcribe_windows[_dev/_prev] (index = window) or wb_waveform(s)_to_tokens[_resampled] (index =
 * waveform) call on this session, aligned with the ids that call wrote: n_out = that row's id count.  WB_ERR_STATE before the
 * first such call, WB_ERR_INVALID_ARG for an index out of range or capacity < n_out.  out == NULL only sets n_out.
 * Those calls check every argument that does not depend on decoded ids before they encode (the waveform calls: each batch's
 * before that batch's encode); a call rejected there leaves the encoded windows, these log-probs, wb_session_last_timings
 * and wb_session_last_steps as they were.  A call that fails later (a row beyond capacity, say) leaves no log-probs.
 * The values (float32; the reference's BeamSearchToken.log_prob, transcribe.rs:142-146, holds the same f32 widened to f64):
 *   - the prompt ids (4, or those of a previous-text prompt): 0.0 (transcribe.rs:205-208);
 *   - WB_SEARCH_BEAM, beam_size >= 2: the f32 log_softmax value the search scored the id with, special-id mask included
 *     while sequences have <= 5 tokens (transcribe.rs:291-299).  The left-to-right f64 sum of a row is the cumulative
 *     log-prob the search chose the row by;
 *   - WB_SEARCH_BEAM, beam_size 1: the same, the value wb_session_last_topk reports for that position;
 *   - WB_SEARCH_GREEDY_LOOP: log_softmax of the unmasked logits at the arg-max id; NaN for an EOT a rule appended (EOT test,
 *     repetition cut, context stop);
 *   - wb_waveform(s)_to_tokens: each log-prob travels with its id through the overlap merge (transcribe.rs:56-63). */
int wb_session_last_logprobs(wb_session* s, int64_t index, float* out, int64_t capacity, int64_t* n_out);
/* The n-best list of one window of the last wb_transcribe_windows[_dev/_prev] call (index = window) or wb_waveform(s)_to_tokens
 * call (index = window in waveform-major order: waveform 0's windows as wb_window_bounds lists them, then waveform 1's, ...).
 * ids_out / lp_out are [max_hyps][capacity], lens_out / scores_out / finished_out [max_hyps]; hypotheses best first.
 * ids_out == NULL only sets *n_hyps_out (and lens_out when given).  lp_out / finished_out may be NULL.
 * Under WB_SEARCH_BEAM the list is the search's carried list when beam::beam_search returns (`beams` at beam.rs:33): the
 * search stopped because its best node was finished (beam.rs:22-27), or it ran max_depth steps past the window's own prompt.
 * It holds at most 2 * beam_size hypotheses (up to beam_size live ones, then up to beam_size finished ones, beam.rs:71-78),
 * ranked by applying max_by_last repeatedly to what remains: descending score, exact ties with the LATER carried node first.
 * Rank 0 is therefore always the row the decode call wrote.  Each hypothesis has
 *   - ids:      the window's prompt (any previous-text prompt included) + the generated ids, laid out as a transcribe row;
 *   - lp:       0 for each prompt id, else the f32 log-prob the search scored the id with (as wb_session_last_logprobs);
 *   - score:    the node's cumulative f64 log-prob as the search carried it, bit-equal to the left-to-right f64 sum of lp;
 *   - finished: 1 when the last id is EOT.
 * beam_size 1 gives one hypothesis, the row itself; max_depth 0 one hypothesis, the prompt, with score 0.
 * WB_ERR_STATE before the first decode call and after a WB_SEARCH_GREEDY_LOOP call (the greedy loop carries no list);
 * WB_ERR_INVALID_ARG for an index out of range, max_hyps below the list's size or capacity below its longest hypothesis.
 * A decode call rejected before it encodes leaves the previous n-best as it was, a call that fails later leaves none, and
 * wb_session_score_tokens / wb_session_step leave it as it was. */
int wb_session_last_nbest(wb_session* s, int64_t index, int64_t max_hyps, int64_t capacity, int64_t* ids_out,
                          float* lp_out, int64_t* lens_out, double* scores_out, int32_t* finished_out, int64_t* n_hyps_out);
/* Teacher-forced scoring of n_seqs token sequences against windows this session has encoded:
 * forward_decoder (mod.rs:131-157) + log_softmax (transcribe.rs:276) at every position, in one pass on the GPU.
 * Sequence i is tokens[off_i .. off_i + lens[i]) with off_i = lens[0] + .. + lens[i-1], on window window_of_seq[i].
 * For j >= 1:  lp_out[off_i + j]     = log_softmax(logits of position j-1)[tokens[off_i + j]]   (f32)
 *              argmax_out[off_i + j] = arg-max id of that row, ties to the lower id               (argmax_out may be NULL)
 * and lp_out[off_i] = 0, argmax_out[off_i] = -1.
 * apply_special_mask != 0 adds -inf on is_special ids to the rows whose prefix has <= 5 tokens (j <= 5; the beam rule of
 * transcribe.rs:271-275), so a masked target scores -inf.  Several sequences may share a window.
 * WB_ERR_STATE before an encode call; WB_ERR_INVALID_ARG for lens[i] outside [1, n_text_ctx], a token outside [0, n_vocab),
 * a window outside the encoded ones, or apply_special_mask without is_special; WB_ERR_UNSUPPORTED when the weights are not
 * fp16-exact.  Leaves the session's decode state and every wb_session_last_* result as they were. */
int wb_session_score_tokens(wb_session* s, int64_t n_seqs, const int32_t* window_of_seq, const int64_t* tokens,
                            const int64_t* lens, int apply_special_mask, const uint8_t* is_special,
                            float* lp_out, int64_t* argmax_out);
/* Token alignment: when in the audio each token was spoken, by openai-whisper's find_alignment (whisper/timing.py), not by
 * timestamp tokens: a teacher-forced pass over given ids on windows this session has encoded, the cross-attention weights of
 * chosen heads, and dynamic time warping, all on the GPU.  The ids decoded are not touched.
 * Sequences are packed as in wb_session_score_tokens: sequence i is tokens[off_i .. off_i + lens[i]) on window
 * window_of_seq[i].  first[i] is the index of its first aligned id (4 for a default transcribe row, the prompt length for a
 * previous-text row).  heads holds n_heads (layer, head) int32 pairs in any order; n_heads = 0 selects openai's fallback,
 * every head of decoder layers n_text_layer / 2 .. n_text_layer - 1 (heads may then be NULL).
 * For sequence ids[0 .. L) on window w, with first in [1, L - 1]:
 *   1. columns C = max(1, F_w / 2), F_w the window's mel frames that hold audio (the kept frames of a waveform window without
 *      the 10 zero frames; n_ctx for wb_session_encode_mels);
 *   2. for every position p in 0 .. L - 1 and selected head: the scaled cross query of p against the window's scaled keys
 *      0 .. C - 1 (the decoders' q and k; fp16-rounded keys under WB_KV_F16), then softmax over those C columns;
 *   3. per head and column: minus the mean over the L positions, divided by the biased std (0 where the std is 0);
 *   4. median filter of width 7 along the columns with reflect padding (torch's; scipy's "mirror"), skipped when C <= 3;
 *   5. sum over the heads in ascending (layer, head) order divided by their count; rows first - 1 .. L - 2 are the matrix,
 *      N = L - first rows (row k is the query that predicts ids[first + k]);
 *   6. DTW on -matrix with openai's dtw_cpu rules: f32 cost; diagonal if c0 < c1 && c0 < c2, else up if c1 < c0 && c1 < c2,
 *      else left; backtrace with row 0 read as left and column 0 as up;
 *   7. start[k] = the column where the path first enters row k, end[k] = start[k + 1], end[N - 1] = C.
 * start_out / end_out: per aligned id (sequence i's N_i ids after those of sequences 0 .. i-1) its int32 encoder positions;
 * one position is 20 ms from the window's start in both window modes.  matrix_out (may be NULL): each sequence's matrix, f32
 * [N_i][C_i], packed in sequence order, matrix_capacity floats.  Word grouping is text work and stays with the caller.
 * Sequences run in groups of at most 4096 positions; the workspace holds one layer's selected heads of one group:
 * heads x positions x C x 4 bytes.
 * WB_ERR_STATE before an encode call; WB_ERR_INVALID_ARG for lens[i] outside [2, n_text_ctx], first[i] outside [1, lens[i] - 1],
 * a token outside [0, n_vocab), a window outside the encoded ones, a head outside the model or listed twice, or matrix_capacity
 * below sum N_i C_i; WB_ERR_UNSUPPORTED when the weights are not fp16-exact, or when a sequence's DTW does not fit one CTA
 * (N_i > 448, or its 2-bit trace N_i x ceil(C_i / 16) x 4 bytes beyond ~221 KB of shared memory: only a model with
 * n_audio_ctx above 2016 gets there; 447 x 1500 fits).  Leaves the session's decode state and every
 * wb_session_last_* result as they were. */
int wb_session_align_tokens(wb_session* s, int64_t n_seqs, const int32_t* window_of_seq, const int64_t* tokens,
                            const int64_t* lens, const int64_t* first, int64_t n_heads, const int32_t* heads,
                            int32_t* start_out, int32_t* end_out, float* matrix_out, int64_t matrix_capacity);
/* Step 6 and 7 of wb_session_align_tokens alone, on a caller's f32 matrix [n_rows][n_cols] (host), on the GPU: start_out /
 * end_out [n_rows].  n_rows in [1, 448], n_cols >= 1 with the 2-bit trace, n_rows x ceil(n_cols / 16) x 4 bytes, within one
 * CTA's shared memory (~221 KB; 447 x 1500 fits).  WB_ERR_INVALID_ARG otherwise, WB_ERR_CUDA without a device. */
int wb_align_dtw(int device, const float* matrix, int64_t n_rows, int64_t n_cols, int32_t* start_out, int32_t* end_out);
/* transcribe.rs:114-138: number of windows and their [start, end) bounds */
int64_t wb_window_count(int64_t n_samples, int64_t sample_rate, int64_t window_len);
int wb_window_bounds(int64_t n_samples, int64_t sample_rate, int64_t window_len, int64_t* starts, int64_t* ends);
/* transcribe.rs:76-110; returns 1 and fills the indices if an overlap was found, else 0 */
int wb_find_chunk_overlap(const int64_t* prev, int64_t n_prev, const int64_t* curr, int64_t n_curr,
                          int64_t max_n_offsets, int64_t min_n_overlaps, int64_t* prev_index, int64_t* curr_index);
/* Repetition heuristics the reference compiles but calls only from its commented-out greedy loop (transcribe.rs:314-380).
 * transcribe.rs:385-393: position after the last mismatch between a block of `period` tokens and the block before it, walking
 * back from the end; `period` when none; -1 where the reference's usize arithmetic underflows (period > n). */
int64_t wb_first_repetition_end(const int64_t* tokens, int64_t n, int64_t period);
/* transcribe.rs:395-419: the period of a suffix repeated at least min_repetitions times before itself, 0 for None. */
int64_t wb_repetition_period(const int64_t* tokens, int64_t n, int64_t min_repetitions);
/* transcribe.rs:421-447: 1 and (first_repeat_index, end) when at least min_repeat_count earlier windows equal the last window of
 * window_size tokens, 0 for None, -1 where the reference unwraps a second repeat that does not exist. */
int wb_find_repeated_tokens_index(const int64_t* tokens, int64_t n, int64_t window_size, int64_t min_repeat_count,
                                  int64_t* first_repeat_index, int64_t* end);

/* ---- beam.rs (host) ------------------------------------------------------------------------ */
/* get_top_elements (beam.rs:81-110) on f64 scores, num 0 .. 7: writes the indices of the kept elements in
 * the reference's output order (ascending score); returns how many were kept, or -1 on bad arguments. */
int64_t wb_beam_get_top_elements(const double* scores, int64_t n, int64_t num, int64_t* idx_out);

/* beam::beam_search (beam.rs:9-37) with a table-driven `next` (see csrc/api.cu): the library's beam search (host/beam.hpp) on
 * the CPU, for tests.  Each live beam contributes its beam_size best table entries, as the device contributes its top-k
 * candidates.  beam_size 1 .. 7.  Returns the length of the best sequence written to seq_out, or -1 on bad arguments. */
int64_t wb_beam_search_table(const double* table, int64_t n_ctx, int64_t n_vocab, int64_t first_token, int64_t eot,
                             int64_t beam_size, int64_t max_depth, int64_t* seq_out, int64_t capacity);
/* The ranked final carried list (the n-best of wb_session_last_nbest) of the same table-driven search.  ids_out is
 * [max_hyps][capacity], lens_out / scores_out / finished_out [max_hyps] (finished_out may be NULL); hypotheses best first.
 * Returns the hypothesis count, or -1 on bad arguments, a list longer than max_hyps or a sequence longer than capacity. */
int64_t wb_beam_nbest_table(const double* table, int64_t n_ctx, int64_t n_vocab, int64_t first_token, int64_t eot, int64_t beam_size,
                            int64_t max_depth, int64_t max_hyps, int64_t capacity, int64_t* ids_out, int64_t* lens_out,
                            double* scores_out, int32_t* finished_out);

/* ---- transcribe binary helpers (host) ---------------------------------------------------------- */
/* load_audio_waveform (src/bin/transcribe/main.rs:31-55): PCM int samples / (2^(bits-1) - 1), float samples as they
 * are, interleaved.  strict_16k_mono != 0 enforces the reference's asserts (16 kHz, one channel) as WB_ERR_INVALID_ARG.
 * out may be NULL to query the sample count. */
int wb_load_wav(const char* path, int strict_16k_mono, float* out, int64_t capacity, int64_t* n_samples_out,
                int64_t* sample_rate_out, int* channels_out);

/* ---- measurement ----------------------------------------------------------------------------- */
/* Diagnostics: which persistent decoder kernel the last decode launch used: 6 = head-fused cluster decoder (decoder6.cu),
 * 5 = batched tensor-core (decoder5.cu), 4 = cluster/DSMEM (decoder4.cu), 3 = grid-barrier FMA fallback (decoder3.cu), 0 = none yet. */
int wb_session_last_decoder(const wb_session* s);
/* Diagnostics: the candidates the last decoder launch selected at its last position, [n_rows][k] ids and log-probs, for rows
 * 0 .. n_rows-1 of that launch.  Every decoder writes them, in greedy decoding too (k = 1: the chosen id and its log-prob), so
 * a greedy run can be checked step by step.  WB_ERR_INVALID_ARG when k differs from that launch's k or n_rows exceeds its rows,
 * WB_ERR_STATE before the first launch. */
int wb_session_last_topk(wb_session* s, int64_t n_rows, int64_t k, int64_t* ids_out, float* lp_out);
/* kernels launched by this library on this thread's sessions since the last reset */
int64_t wb_kernel_launch_count(void);
void wb_kernel_launch_count_reset(void);
/* device-side duration (CUDA events on the session stream) of the phases of the last
 * wb_transcribe_windows* call, in milliseconds: [0]=log-mel, [1]=encoder+cross-KV, [2]=decode, [3]=total; a call rejected
 * before it encodes leaves them as they were (wb_session_last_logprobs) */
int wb_session_last_timings(wb_session* s, float* ms_out4);
int wb_session_last_steps(wb_session* s, int64_t* n_steps_out);
/* roofline aid: re-runs n_steps greedy decoder steps on the currently encoded windows with CUDA
 * events (session stream) around the dominant kernel of the step -- the logits GEMV -- and around
 * each whole step; returns the average durations in milliseconds. */
int wb_session_profile_decode(wb_session* s, const wb_special_ids* ids, int n_steps, float* logits_kernel_ms,
                              float* step_ms);

#ifdef __cplusplus
}
#endif
#endif /* WHISPER_B200_H */
