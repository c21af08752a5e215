// extern "C" boundary (include/whisper_b200.h).  No exceptions cross it: every entry point maps
// wb::Error / std::exception to a status code and a thread-local message.
#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>

#include "../host/beam.hpp"
#include "../host/repeat.hpp"
#include "session.h"

struct wb_model {
    wb::Model impl;
    // the stateless entry points (wb_forward_encoder / wb_forward_decoder) keep ONE session between calls instead of paying
    // dozens of cudaMalloc per call; it is rebuilt only when a call needs more windows or positions than it holds
    std::mutex fwd_mu;
    std::unique_ptr<wb::Session> fwd;
    wb::Session& forward_session(int64_t n_windows, int64_t text_len) {
        if (!fwd || fwd->max_windows < n_windows || fwd->t_max < text_len) {
            fwd.reset();
            fwd.reset(new wb::Session(&impl, std::max<int64_t>(n_windows, 1), 1, std::max<int64_t>(text_len, 2), WB_KV_F32));
        }
        return *fwd;
    }
    ~wb_model() { fwd.reset(); }   // sessions die before their model
};
struct wb_session {
    std::unique_ptr<wb::Session> impl;
};

namespace {

template <typename F>
int guarded(F&& f) {
    try {
        f();
        return WB_OK;
    } catch (const wb::Error& e) {
        wb::set_last_error(e.what());
        return e.code;
    } catch (const std::bad_alloc&) {
        wb::set_last_error("host out of memory");
        return WB_ERR_OOM;
    } catch (const std::exception& e) {
        wb::set_last_error(e.what());
        return WB_ERR_CUDA;
    }
}

void require_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        wb::fail(WB_ERR_CUDA, std::string("no CUDA device available (there is no CPU fallback): ") + cudaGetErrorString(e));
    }
    if (device < 0 || device >= n) wb::fail(WB_ERR_INVALID_ARG, "device index out of range");
    WB_CUDA(cudaSetDevice(device));
}

// row w of the ids to tokens_out[w * capacity ..], its length to lens_out[w] (the pipeline has checked that rows fit)
void copy_tokens_out(const std::vector<std::vector<int64_t>>& toks, int64_t* tokens_out, int64_t capacity, int64_t* lens_out) {
    for (size_t w = 0; w < toks.size(); ++w) {
        std::copy(toks[w].begin(), toks[w].end(), tokens_out + (int64_t)w * capacity);
        lens_out[w] = (int64_t)toks[w].size();
    }
}

// prep_audio on the device; `wave` and `mel_out` are device pointers
void prep_audio_device(wb::Model& model, const float* wave_dev, int64_t n_batch, int64_t n_samples, float* mel_out_dev,
                       int64_t* n_frames_out, cudaStream_t st) {
    using namespace wb;
    WB_REQUIRE(n_batch >= 1, "prep_audio: n_batch must be >= 1");
    WB_REQUIRE(n_samples >= N_FFT, "prep_audio: waveform shorter than n_fft (audio.rs:292)");
    WB_REQUIRE(n_samples < ((int64_t)1 << 30), "prep_audio: waveform too long");
    const int F = (int)(n_samples / HOP);
    std::vector<LogMelWindow> lw((size_t)n_batch);
    for (int64_t b = 0; b < n_batch; ++b)
        lw[(size_t)b] = LogMelWindow{b * n_samples, (int)n_samples, F, F, 0, b * (int64_t)F * N_MELS};   // one global max (audio.rs:50)
    DevBuf<LogMelWindow> dwin;
    DevBuf<int> slot;
    DevBuf<float> rows;
    dwin.alloc((size_t)n_batch);
    slot.alloc(1);
    rows.alloc((size_t)n_batch * F * N_MELS + 4);
    WB_CUDA(cudaMemcpyAsync(dwin.p, lw.data(), lw.size() * sizeof(LogMelWindow), cudaMemcpyHostToDevice, st));
    if (F > 0) {
        launch_logmel(model, wave_dev, dwin.p, (int)n_batch, F, rows.p, slot.p, 1, st);
        for (int64_t b = 0; b < n_batch; ++b)
            launch_rows_to_chan(rows.p + b * (int64_t)F * N_MELS, mel_out_dev + b * (int64_t)N_MELS * F, F, st);
    }
    WB_CUDA(cudaStreamSynchronize(st));
    if (n_frames_out) *n_frames_out = F;
}

// a model holding only the frontend tables (prep_audio needs no weights); one per device, uploaded on first use
struct FrontendOnly {
    wb::Model m;
    explicit FrontendOnly(int device) {
        using namespace wb;
        m.device = device;
        const FrontendTables& ft = frontend_tables();
        auto up = [&](const void* src, size_t bytes) {
            void* p = nullptr;
            WB_CUDA(cudaMalloc(&p, bytes));
            m.allocs.push_back(p);
            WB_CUDA(cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice));
            return p;
        };
        m.basis_t = (float*)up(ft.basis_t.data(), ft.basis_t.size() * sizeof(float));
        m.mel_filt = (float*)up(ft.mel_filt.data(), ft.mel_filt.size() * sizeof(float));
        std::vector<int> rng(2 * N_MELS);
        for (int i = 0; i < N_MELS; ++i) { rng[2 * i] = ft.mel_lo[i]; rng[2 * i + 1] = ft.mel_hi[i]; }
        m.mel_range = (int*)up(rng.data(), rng.size() * sizeof(int));
    }
};

FrontendOnly& frontend_for(int device) {
    static std::mutex mu;
    static std::map<int, std::unique_ptr<FrontendOnly>> cache;
    std::lock_guard<std::mutex> lock(mu);
    auto& slot = cache[device];
    if (!slot) slot.reset(new FrontendOnly(device));
    return *slot;
}

// The ranked final carried list of the search of wb_beam_search_table / wb_beam_nbest_table: beam_search_windows over one
// window with prompt {first_token} from position 0, stepped by a table.  The candidates of a row fed token t at position p (a
// sequence of p + 1 ids) are the beam_size best entries of table row (t * 131 + p + 1) % n_ctx, as the device contributes
// its top-k per-token log-probs; a beam is finished when its last token is eot.  Host only: lets the CPU tests drive the
// library's search against the oracle without a GPU.
wb::NBest table_nbest(const double* table, int64_t n_ctx, int64_t n_vocab, int64_t first_token, int64_t eot, int beam_size,
                      int max_depth) {
    namespace fx = wb::beamfx;
    auto step = [&](int p, int64_t n_rows, const int32_t*, const int32_t*, const int64_t* token, int, int k, int64_t* ids_out,
                    double* lps_out) {
        for (int64_t r = 0; r < n_rows; ++r) {
            const double* row = table + ((token[r] * 131 + p + 1) % n_ctx) * n_vocab;
            int top[fx::MAX_BEAM + 1];
            const int nt = fx::top_elements(row, (int)n_vocab, k, top);
            for (int i = 0; i < k; ++i) {
                ids_out[r * k + i] = i < nt ? top[i] : -1;
                lps_out[r * k + i] = i < nt ? row[top[i]] : 0.0;
            }
        }
    };
    const std::vector<std::vector<int64_t>> prompt{{first_token}};
    int64_t steps = 0;
    return wb::ranked_nbest(wb::beam_search_windows(prompt, 0, beam_size, max_depth, eot, step, &steps)[0]);
}

// the table entry points' arguments: beam_size 1 .. beamfx::MAX_BEAM
bool table_args_ok(const double* table, int64_t n_ctx, int64_t n_vocab, int64_t beam_size, int64_t max_depth) {
    return table && n_ctx >= 1 && n_vocab >= 1 && n_vocab <= INT32_MAX && beam_size >= 1 && beam_size <= wb::beamfx::MAX_BEAM &&
           max_depth >= 0 && max_depth <= INT32_MAX;
}

}  // namespace

extern "C" {

const char* wb_version(void) { return "whisper_b200 0.1.0 (sm_90a)"; }
const char* wb_last_error(void) { return wb::last_error_string().c_str(); }

int wb_device_count(int* n_out) {
    return guarded([&] {
        WB_REQUIRE(n_out != nullptr, "null output");
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
        *n_out = n;
    });
}

int64_t wb_max_waveform_samples(int64_t n_frame_max) {
    // audio.rs:12-17: HOP * (n_frame_max + 1) + is_odd(N_FFT) - 1
    return (int64_t)wb::HOP * (n_frame_max + 1) + (wb::N_FFT % 2) - 1;
}

int wb_prep_audio(int device, const float* wave, int64_t n_batch, int64_t n_samples, float* mel_out,
                  int64_t* n_frames_out) {
    return guarded([&] {
        WB_REQUIRE(wave && mel_out, "prep_audio: null pointer");
        WB_REQUIRE(n_batch >= 1, "prep_audio: n_batch must be >= 1");
        WB_REQUIRE(n_samples >= wb::N_FFT, "prep_audio: waveform shorter than n_fft (audio.rs:292)");
        require_device(device);
        FrontendOnly& fe = frontend_for(device);
        const int64_t F = n_samples / wb::HOP;
        wb::DevBuf<float> dw, dm;
        dw.alloc((size_t)(n_batch * n_samples));
        dm.alloc((size_t)(n_batch * wb::N_MELS * F) + 4);
        WB_CUDA(cudaMemcpy(dw.p, wave, (size_t)(n_batch * n_samples) * sizeof(float), cudaMemcpyHostToDevice));
        prep_audio_device(fe.m, dw.p, n_batch, n_samples, dm.p, n_frames_out, nullptr);
        WB_CUDA(cudaMemcpy(mel_out, dm.p, (size_t)(n_batch * wb::N_MELS * F) * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

int wb_prep_audio_dev(int device, const float* wave_dev, int64_t n_batch, int64_t n_samples, float* mel_out_dev,
                      int64_t* n_frames_out) {
    return guarded([&] {
        WB_REQUIRE(wave_dev && mel_out_dev, "prep_audio: null pointer");
        require_device(device);
        FrontendOnly& fe = frontend_for(device);
        prep_audio_device(fe.m, wave_dev, n_batch, n_samples, mel_out_dev, n_frames_out, nullptr);
    });
}

int64_t wb_resampled_length(int64_t n_frames, int64_t sample_rate) { return wb::resampled_length(n_frames, sample_rate); }

int wb_resample(int device, const float* in, int64_t n_frames, int64_t channels, int64_t sample_rate, float* out, int64_t capacity,
                int64_t* n_out) {
    return guarded([&] {
        WB_REQUIRE(in && out && n_out, "resample: null pointer");
        WB_REQUIRE(n_frames >= 1, "resample: n_frames must be >= 1");
        WB_REQUIRE(channels >= 1 && channels <= INT32_MAX, "resample: channels must be >= 1");
        const int64_t len = wb::resampled_length(n_frames, sample_rate);
        if (len < 0) wb::fail(WB_ERR_UNSUPPORTED, "resample: unsupported sample rate (gcd with 16000 must leave up and down <= 1024)");
        WB_REQUIRE(n_frames <= INT64_MAX / channels, "resample: waveform too long");
        WB_REQUIRE(capacity >= len, "resample: capacity below wb_resampled_length");
        require_device(device);
        wb::ResampleBufs b;
        std::vector<int64_t> off, n;
        wb::resample_waveforms(b, &in, &n_frames, &channels, &sample_rate, 1, off, n, nullptr);
        WB_CUDA(cudaMemcpy(out, b.out.p, (size_t)len * sizeof(float), cudaMemcpyDeviceToHost));
        *n_out = len;
    });
}

int wb_model_create(const wb_dims* dims, int device, wb_model** out) {
    return guarded([&] {
        WB_REQUIRE(dims && out, "model_create: null pointer");
        WB_REQUIRE(dims->n_mels > 0 && dims->n_audio_ctx > 0 && dims->n_audio_state > 0 && dims->n_audio_head > 0 &&
                       dims->n_audio_layer > 0 && dims->n_vocab > 0 && dims->n_text_ctx > 0 && dims->n_text_state > 0 &&
                       dims->n_text_head > 0 && dims->n_text_layer > 0,
                   "model_create: non-positive dimension");
        require_device(device);
        wb_model* m = new wb_model();
        m->impl.dims = *dims;
        m->impl.device = device;
        *out = m;
    });
}

int wb_model_set_tensor(wb_model* m, const char* path, const float* data, const int64_t* shape, int ndim) {
    return guarded([&] {
        WB_REQUIRE(m != nullptr, "null model");
        wb::model_set_tensor(m->impl, path, data, shape, ndim);
    });
}

int wb_npy_tree_probe(const char* dir, wb_dims* dims_out) {
    return guarded([&] {
        WB_REQUIRE(dir && dims_out, "npy_tree_probe: null pointer");
        wb::npy_tree_probe(dir, *dims_out);
    });
}

int wb_model_load_npy_tree(const char* dir, int device, int ln_eps_outside, wb_model** out) {
    return guarded([&] {
        WB_REQUIRE(dir && out, "model_load_npy_tree: null pointer");
        wb_dims dims{};
        wb::npy_tree_probe(dir, dims);
        require_device(device);
        std::unique_ptr<wb_model> m(new wb_model());
        m->impl.dims = dims;
        m->impl.device = device;
        m->impl.ln_eps_outside = ln_eps_outside ? 1 : 0;
        wb::npy_tree_load(m->impl, dir);
        wb::model_finalize(m->impl);
        *out = m.release();
    });
}

int wb_model_set_layernorm_eps_mode(wb_model* m, int outside) {
    return guarded([&] {
        WB_REQUIRE(m != nullptr, "null model");
        if (m->impl.finalized) wb::fail(WB_ERR_STATE, "model already finalized");
        m->impl.ln_eps_outside = outside ? 1 : 0;
    });
}

int wb_model_finalize(wb_model* m) {
    return guarded([&] {
        WB_REQUIRE(m != nullptr, "null model");
        wb::model_finalize(m->impl);
    });
}

void wb_model_destroy(wb_model* m) { delete m; }

int wb_model_get_dims(const wb_model* m, wb_dims* out) {
    return guarded([&] {
        WB_REQUIRE(m && out, "null pointer");
        *out = m->impl.dims;
    });
}

int wb_model_weights_fp16_exact(const wb_model* m) { return (m && m->impl.fp16_exact) ? 1 : 0; }

int wb_forward_encoder(wb_model* m, const float* mel, int64_t n_batch, int64_t n_mels, int64_t n_ctx, float* out) {
    return guarded([&] {
        WB_REQUIRE(m && mel && out, "forward_encoder: null pointer");
        WB_REQUIRE(n_batch >= 1, "forward_encoder: n_batch must be >= 1");
        std::lock_guard<std::mutex> lock(m->fwd_mu);
        wb::Session& s = m->forward_session(n_batch, 2);
        s.encode_mels_host(mel, n_batch, n_mels, n_ctx);
        const int d = m->impl.dims.n_audio_state;
        WB_CUDA(cudaMemcpy(out, s.xa.p, (size_t)s.M_tot * d * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

int wb_forward_decoder(wb_model* m, const int64_t* tokens, int64_t n_batch, int64_t seq_len, const float* encoder_output,
                       int64_t n_enc_ctx, float* logits_out) {
    return guarded([&] {
        WB_REQUIRE(m && tokens && encoder_output && logits_out, "forward_decoder: null pointer");
        const wb_dims& D = m->impl.dims;
        WB_REQUIRE(n_batch >= 1 && seq_len >= 1, "forward_decoder: empty input");
        WB_REQUIRE(seq_len <= D.n_text_ctx, "Token sequence length must not exceed n_text_ctx (mod.rs:134-139)");
        std::lock_guard<std::mutex> lock(m->fwd_mu);
        wb::Session& s = m->forward_session(n_batch, std::min<int64_t>(D.n_text_ctx, std::max<int64_t>(seq_len, 2)));
        s.load_encoder_output_host(encoder_output, n_batch, n_enc_ctx);
        s.teacher_forced_logits(tokens, n_batch, seq_len, logits_out);
    });
}

int64_t wb_window_samples(int64_t n_audio_ctx, int window_mode) {
    if (n_audio_ctx <= wb::MEL_PADDING || n_audio_ctx > INT32_MAX / 2 || (window_mode != WB_WINDOWS_REFERENCE && window_mode != WB_WINDOWS_NATIVE)) return -1;
    return wb::window_samples((int)n_audio_ctx, window_mode);
}

int wb_session_create_windows(wb_model* m, int64_t max_windows, int64_t max_beams, int64_t max_text_len, int kv_dtype,
                              int window_mode, wb_session** out) {
    return guarded([&] {
        WB_REQUIRE(m && out, "session_create: null pointer");
        std::unique_ptr<wb_session> s(new wb_session());
        s->impl.reset(new wb::Session(&m->impl, max_windows, max_beams, max_text_len, kv_dtype, window_mode));
        *out = s.release();
    });
}

int wb_session_create(wb_model* m, int64_t max_windows, int64_t max_beams, int64_t max_text_len, int kv_dtype,
                      wb_session** out) {
    return wb_session_create_windows(m, max_windows, max_beams, max_text_len, kv_dtype, WB_WINDOWS_REFERENCE, out);
}

void wb_session_destroy(wb_session* s) { delete s; }

int wb_session_set_search(wb_session* s, int rule) {
    return guarded([&] {
        WB_REQUIRE(s, "set_search: null pointer");
        s->impl->set_search(rule);
    });
}

int wb_session_set_prev_prompt(wb_session* s, int64_t startofprev) {
    return guarded([&] {
        WB_REQUIRE(s, "set_prev_prompt: null pointer");
        s->impl->set_prev_prompt(startofprev);
    });
}

int wb_session_encode_waveforms(wb_session* s, const float* const* waves, const int64_t* lens, int64_t n_windows) {
    return guarded([&] {
        WB_REQUIRE(s && waves && lens, "encode: null pointer");
        s->impl->encode_waveforms_host(waves, lens, n_windows);
        WB_CUDA(cudaStreamSynchronize(s->impl->st));
    });
}

int wb_session_encode_waveforms_dev(wb_session* s, const float* wave_dev, const int64_t* offsets, const int64_t* lens,
                                    int64_t n_windows) {
    return guarded([&] {
        WB_REQUIRE(s && wave_dev && offsets && lens, "encode: null pointer");
        s->impl->encode_from_device_wave(wave_dev, offsets, lens, n_windows);
        WB_CUDA(cudaStreamSynchronize(s->impl->st));
    });
}

int wb_session_encode_mels(wb_session* s, const float* mel, int64_t n_windows, int64_t n_mels, int64_t n_ctx) {
    return guarded([&] {
        WB_REQUIRE(s && mel, "encode: null pointer");
        s->impl->encode_mels_host(mel, n_windows, n_mels, n_ctx);
    });
}

int wb_session_get_mel(wb_session* s, int64_t window, float* mel_out, int64_t capacity, int64_t* n_ctx_out) {
    return guarded([&] {
        WB_REQUIRE(s && mel_out && n_ctx_out, "get_mel: null pointer");
        wb::Session& S = *s->impl;
        if (!S.encoded) wb::fail(WB_ERR_STATE, "get_mel: nothing encoded");
        WB_REQUIRE(window >= 0 && window < S.n_windows, "get_mel: window out of range");
        const int Tm = S.win_Tm[(size_t)window];
        WB_REQUIRE(capacity >= (int64_t)Tm * wb::N_MELS, "get_mel: capacity too small");
        std::vector<float> rows((size_t)Tm * wb::N_MELS);
        WB_CUDA(cudaMemcpy(rows.data(), S.mel_rows.p + ((int64_t)window * S.TmS + 1) * wb::N_MELS,
                           rows.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (int t = 0; t < Tm; ++t)
            for (int c = 0; c < wb::N_MELS; ++c) mel_out[(int64_t)c * Tm + t] = rows[(size_t)t * wb::N_MELS + c];
        *n_ctx_out = Tm;
    });
}

int wb_session_get_encoder_output(wb_session* s, int64_t window, float* out, int64_t capacity, int64_t* n_ctx_out) {
    return guarded([&] {
        WB_REQUIRE(s && out && n_ctx_out, "get_encoder_output: null pointer");
        wb::Session& S = *s->impl;
        if (!S.encoded) wb::fail(WB_ERR_STATE, "get_encoder_output: nothing encoded");
        WB_REQUIRE(window >= 0 && window < S.n_windows, "get_encoder_output: window out of range");
        const int d = S.m->dims.n_audio_state;
        const int T = S.win_T[(size_t)window];
        WB_REQUIRE(capacity >= (int64_t)T * d, "get_encoder_output: capacity too small");
        WB_CUDA(cudaMemcpy(out, S.xa.p + S.win_row_off[(size_t)window] * d, (size_t)T * d * sizeof(float),
                           cudaMemcpyDeviceToHost));
        *n_ctx_out = T;
    });
}

int wb_session_begin(wb_session* s, const int64_t* prompt, int64_t prompt_len) {
    return guarded([&] {
        WB_REQUIRE(s && prompt, "begin: null pointer");
        WB_REQUIRE(prompt_len >= 1, "begin: prompt length out of range");
        s->impl->begin(std::vector<std::vector<int64_t>>((size_t)s->impl->n_windows, std::vector<int64_t>(prompt, prompt + prompt_len)));
    });
}

int wb_session_step(wb_session* s, int64_t n_rows, const int32_t* window_of_row, const int32_t* parent_row,
                    const int64_t* token, int apply_special_mask, const uint8_t* is_special, int k,
                    int64_t* topk_ids_out, float* topk_logprob_out) {
    return guarded([&] {
        WB_REQUIRE(s && window_of_row && parent_row && token && topk_ids_out && topk_logprob_out, "step: null pointer");
        if (is_special) s->impl->set_special(is_special);
        WB_REQUIRE(!apply_special_mask || s->impl->have_special, "step: special mask requested but no is_special bitmap given");
        s->impl->step_beams(n_rows, window_of_row, parent_row, token, apply_special_mask, k, topk_ids_out, topk_logprob_out);
    });
}

int wb_transcribe_windows(wb_session* s, const float* const* waves, const int64_t* lens, int64_t n_windows,
                          int beam_size, int max_depth, const wb_special_ids* ids, const uint8_t* is_special,
                          int64_t* tokens_out, int64_t capacity, int64_t* lens_out) {
    return guarded([&] {
        WB_REQUIRE(s && waves && lens && ids && tokens_out && lens_out, "transcribe: null pointer");
        wb::Session& S = *s->impl;
        const auto prompts = wb::window_prompts(S, n_windows, beam_size, max_depth, *ids, is_special);
        copy_tokens_out(wb::transcribe_windows(S, prompts, beam_size, max_depth, ids->eot, is_special, capacity,
                                               [&] { S.encode_waveforms_host(waves, lens, n_windows); }),
                        tokens_out, capacity, lens_out);
    });
}

int wb_transcribe_windows_prev(wb_session* s, const float* const* waves, const int64_t* lens, int64_t n_windows,
                               const int64_t* prev_tokens, const int64_t* prev_lens, int64_t startofprev, int beam_size,
                               int max_depth, const wb_special_ids* ids, const uint8_t* is_special, int64_t* tokens_out,
                               int64_t capacity, int64_t* lens_out) {
    return guarded([&] {
        WB_REQUIRE(s && waves && lens && prev_lens && ids && tokens_out && lens_out, "transcribe_windows_prev: null pointer");
        wb::Session& S = *s->impl;
        WB_REQUIRE(n_windows >= 1 && n_windows <= S.max_windows, "transcribe_windows_prev: n_windows out of range");
        std::vector<std::vector<int64_t>> prev((size_t)n_windows);
        int64_t off = 0;
        for (int64_t w = 0; w < n_windows; ++w) {
            WB_REQUIRE(prev_lens[w] >= 0, "transcribe_windows_prev: negative prev_lens entry");
            WB_REQUIRE(prev_lens[w] == 0 || prev_tokens, "transcribe_windows_prev: null prev_tokens");
            prev[(size_t)w].assign(prev_tokens + off, prev_tokens + off + prev_lens[w]);
            off += prev_lens[w];
        }
        const auto prompts = wb::window_prompts(S, n_windows, beam_size, max_depth, *ids, is_special, prev, startofprev);
        size_t max_lp = 0;
        for (const auto& pr : prompts) max_lp = std::max(max_lp, pr.size());
        WB_REQUIRE(capacity >= (int64_t)max_lp + max_depth + 1, "transcribe_windows_prev: capacity below prompt + max_depth + 1");
        copy_tokens_out(wb::transcribe_windows(S, prompts, beam_size, max_depth, ids->eot, is_special, capacity,
                                               [&] { S.encode_waveforms_host(waves, lens, n_windows); }),
                        tokens_out, capacity, lens_out);
    });
}

int wb_transcribe_windows_dev(wb_session* s, const float* wave_dev, const int64_t* offsets, const int64_t* lens,
                              int64_t n_windows, int beam_size, int max_depth, const wb_special_ids* ids,
                              const uint8_t* is_special, int64_t* tokens_out, int64_t capacity, int64_t* lens_out) {
    return guarded([&] {
        WB_REQUIRE(s && wave_dev && offsets && lens && ids && tokens_out && lens_out, "transcribe: null pointer");
        wb::Session& S = *s->impl;
        const auto prompts = wb::window_prompts(S, n_windows, beam_size, max_depth, *ids, is_special);
        copy_tokens_out(wb::transcribe_windows(S, prompts, beam_size, max_depth, ids->eot, is_special, capacity,
                                               [&] { S.encode_from_device_wave(wave_dev, offsets, lens, n_windows); }),
                        tokens_out, capacity, lens_out);
    });
}

int64_t wb_window_count(int64_t n_samples, int64_t sample_rate, int64_t window_len) {
    return (int64_t)wb::window_bounds(n_samples, sample_rate, window_len).size();
}

int wb_window_bounds(int64_t n_samples, int64_t sample_rate, int64_t window_len, int64_t* starts, int64_t* ends) {
    return guarded([&] {
        WB_REQUIRE(starts && ends, "window_bounds: null pointer");
        const auto b = wb::window_bounds(n_samples, sample_rate, window_len);
        for (size_t i = 0; i < b.size(); ++i) { starts[i] = b[i].first; ends[i] = b[i].second; }
    });
}

int wb_waveform_to_tokens(wb_session* s, const float* waveform, int64_t n_samples, int64_t sample_rate, int beam_size,
                          int max_depth, const wb_special_ids* ids, const uint8_t* is_special, int64_t* tokens_out,
                          int64_t capacity, int64_t* n_tokens_out) {
    if (!waveform) return guarded([] { wb::fail(WB_ERR_INVALID_ARG, "waveform_to_tokens: null pointer"); });
    return wb_waveforms_to_tokens(s, &waveform, &n_samples, 1, sample_rate, beam_size, max_depth, ids, is_special, tokens_out,
                                  capacity, n_tokens_out);
}

int wb_waveforms_to_tokens(wb_session* s, const float* const* waveforms, const int64_t* n_samples, int64_t n_waveforms,
                           int64_t sample_rate, int beam_size, int max_depth, const wb_special_ids* ids,
                           const uint8_t* is_special, int64_t* tokens_out, int64_t capacity, int64_t* n_tokens_out) {
    return guarded([&] {
        WB_REQUIRE(s && waveforms && n_samples && ids && tokens_out && n_tokens_out, "waveforms_to_tokens: null pointer");
        copy_tokens_out(wb::waveforms_to_tokens(*s->impl, waveforms, n_samples, n_waveforms, sample_rate, beam_size, max_depth,
                                                *ids, is_special, capacity),
                        tokens_out, capacity, n_tokens_out);
    });
}

int wb_waveforms_to_tokens_resampled(wb_session* s, const float* const* waveforms, const int64_t* n_frames, const int64_t* channels,
                                     const int64_t* sample_rates, int64_t n_waveforms, int beam_size, int max_depth,
                                     const wb_special_ids* ids, const uint8_t* is_special, int64_t* tokens_out, int64_t capacity,
                                     int64_t* n_tokens_out) {
    return guarded([&] {
        WB_REQUIRE(s && waveforms && n_frames && channels && sample_rates && ids && tokens_out && n_tokens_out,
                   "waveforms_to_tokens_resampled: null pointer");
        copy_tokens_out(wb::waveforms_to_tokens_resampled(*s->impl, waveforms, n_frames, channels, sample_rates, n_waveforms, beam_size,
                                                          max_depth, *ids, is_special, capacity),
                        tokens_out, capacity, n_tokens_out);
    });
}

int wb_session_last_logprobs(wb_session* s, int64_t index, float* out, int64_t capacity, int64_t* n_out) {
    return guarded([&] {
        WB_REQUIRE(s && n_out, "last_logprobs: null pointer");
        const wb::Session& S = *s->impl;
        if (!S.have_logprobs) wb::fail(WB_ERR_STATE, "last_logprobs: no transcribe or waveform(s)_to_tokens call yet");
        WB_REQUIRE(index >= 0 && index < (int64_t)S.last_logprobs.size(), "last_logprobs: index out of range");
        const std::vector<float>& v = S.last_logprobs[(size_t)index];
        *n_out = (int64_t)v.size();
        if (!out) return;   // size query
        WB_REQUIRE(capacity >= (int64_t)v.size(), "last_logprobs: capacity too small");
        std::memcpy(out, v.data(), v.size() * sizeof(float));
    });
}

int wb_session_last_nbest(wb_session* s, int64_t index, int64_t max_hyps, int64_t capacity, int64_t* ids_out, float* lp_out,
                          int64_t* lens_out, double* scores_out, int32_t* finished_out, int64_t* n_hyps_out) {
    return guarded([&] {
        WB_REQUIRE(s && n_hyps_out, "last_nbest: null pointer");
        const wb::Session& S = *s->impl;
        if (!S.have_nbest)
            wb::fail(WB_ERR_STATE, "last_nbest: no beam-search transcribe or waveform(s)_to_tokens call yet (the greedy loop keeps none)");
        WB_REQUIRE(index >= 0 && index < (int64_t)S.last_nbest.size(), "last_nbest: index out of range");
        const wb::NBest& nb = S.last_nbest[(size_t)index];
        *n_hyps_out = (int64_t)nb.size();
        if (!ids_out) {   // size query
            if (lens_out)
                for (size_t r = 0; r < nb.size() && (int64_t)r < max_hyps; ++r) lens_out[r] = (int64_t)nb[r].ids.size();
            return;
        }
        WB_REQUIRE(lens_out && scores_out, "last_nbest: null pointer");
        WB_REQUIRE(max_hyps >= (int64_t)nb.size(), "last_nbest: max_hyps below the list's hypothesis count");
        for (const wb::Hypothesis& h : nb) WB_REQUIRE(capacity >= (int64_t)h.ids.size(), "last_nbest: capacity below the longest hypothesis");
        for (size_t r = 0; r < nb.size(); ++r) {
            const wb::Hypothesis& h = nb[r];
            std::copy(h.ids.begin(), h.ids.end(), ids_out + (int64_t)r * capacity);
            if (lp_out) std::copy(h.lps.begin(), h.lps.end(), lp_out + (int64_t)r * capacity);
            lens_out[r] = (int64_t)h.ids.size();
            scores_out[r] = h.score;
            if (finished_out) finished_out[r] = h.finished ? 1 : 0;
        }
    });
}

int wb_session_score_tokens(wb_session* s, int64_t n_seqs, const int32_t* window_of_seq, const int64_t* tokens, const int64_t* lens,
                            int apply_special_mask, const uint8_t* is_special, float* lp_out, int64_t* argmax_out) {
    return guarded([&] {
        WB_REQUIRE(s && window_of_seq && tokens && lens && lp_out, "score_tokens: null pointer");
        s->impl->score_tokens(n_seqs, window_of_seq, tokens, lens, apply_special_mask != 0, is_special, lp_out, argmax_out);
    });
}

int wb_session_align_tokens(wb_session* s, int64_t n_seqs, const int32_t* window_of_seq, const int64_t* tokens, const int64_t* lens,
                            const int64_t* first, int64_t n_heads, const int32_t* heads, int32_t* start_out, int32_t* end_out,
                            float* matrix_out, int64_t matrix_capacity) {
    return guarded([&] {
        WB_REQUIRE(s && window_of_seq && tokens && lens && first && start_out && end_out, "align_tokens: null pointer");
        s->impl->align_tokens(n_seqs, window_of_seq, tokens, lens, first, n_heads, heads, start_out, end_out, matrix_out, matrix_capacity);
    });
}

int wb_align_dtw(int device, const float* matrix, int64_t n_rows, int64_t n_cols, int32_t* start_out, int32_t* end_out) {
    return guarded([&] {
        WB_REQUIRE(matrix && start_out && end_out, "align_dtw: null pointer");
        WB_REQUIRE(wb::dtw_fits(n_rows, n_cols), "align_dtw: n_rows must be in [1, 448] and n_cols >= 1, with the 2-bit trace in one CTA's shared memory");
        require_device(device);
        wb::align_dtw(matrix, n_rows, n_cols, start_out, end_out);
    });
}

int wb_find_chunk_overlap(const int64_t* prev, int64_t n_prev, const int64_t* curr, int64_t n_curr, int64_t max_n_offsets,
                          int64_t min_n_overlaps, int64_t* prev_index, int64_t* curr_index) {
    int64_t pi = 0, ci = 0;
    const bool found = wb::find_chunk_overlap(prev, n_prev, curr, n_curr, max_n_offsets, min_n_overlaps, &pi, &ci);
    if (found) {
        if (prev_index) *prev_index = pi;
        if (curr_index) *curr_index = ci;
    }
    return found ? 1 : 0;
}

int64_t wb_first_repetition_end(const int64_t* tokens, int64_t n, int64_t period) {
    if ((!tokens && n > 0) || n < 0) return -1;
    return wb::repeat::first_repetition_end(tokens, n, period);
}

int64_t wb_repetition_period(const int64_t* tokens, int64_t n, int64_t min_repetitions) {
    if ((!tokens && n > 0) || n < 0) return -1;
    return wb::repeat::repetition_period(tokens, n, min_repetitions);
}

int wb_find_repeated_tokens_index(const int64_t* tokens, int64_t n, int64_t window_size, int64_t min_repeat_count, int64_t* first_repeat_index,
                                  int64_t* end) {
    if ((!tokens && n > 0) || n < 0 || !first_repeat_index || !end) return -1;
    return wb::repeat::find_repeated_tokens_index(tokens, n, window_size, min_repeat_count, first_repeat_index, end);
}

int64_t wb_beam_get_top_elements(const double* scores, int64_t n, int64_t num, int64_t* idx_out) {
    if (!scores || !idx_out || n < 0 || n > INT32_MAX || num < 0 || num > wb::beamfx::MAX_BEAM) return -1;
    int top[wb::beamfx::MAX_BEAM + 1];
    const int nt = wb::beamfx::top_elements(scores, (int)n, (int)num, top);
    std::copy(top, top + nt, idx_out);
    return nt;
}

int wb_load_wav(const char* path, int strict_16k_mono, float* out, int64_t capacity, int64_t* n_samples_out, int64_t* sample_rate_out,
                int* channels_out) {
    return guarded([&] {
        WB_REQUIRE(path && n_samples_out, "load_wav: null pointer");
        std::vector<float> v;
        int64_t sr = 0;
        int ch = 0;
        wb::load_wav(path, strict_16k_mono != 0, v, sr, ch);
        *n_samples_out = (int64_t)v.size();
        if (sample_rate_out) *sample_rate_out = sr;
        if (channels_out) *channels_out = ch;
        if (out) {
            WB_REQUIRE(capacity >= (int64_t)v.size(), "load_wav: capacity too small");
            std::memcpy(out, v.data(), v.size() * sizeof(float));
        }
    });
}

int wb_session_last_decoder(const wb_session* s) { return s ? s->impl->last_decoder : -1; }

int wb_session_last_topk(wb_session* s, int64_t n_rows, int64_t k, int64_t* ids_out, float* lp_out) {
    return guarded([&] {
        WB_REQUIRE(s && ids_out && lp_out, "last_topk: null pointer");
        s->impl->last_topk(n_rows, k, ids_out, lp_out);
    });
}

int64_t wb_beam_search_table(const double* table, int64_t n_ctx, int64_t n_vocab, int64_t first_token, int64_t eot, int64_t beam_size,
                             int64_t max_depth, int64_t* seq_out, int64_t capacity) {
    if (!seq_out || !table_args_ok(table, n_ctx, n_vocab, beam_size, max_depth)) return -1;
    const std::vector<int64_t> best = table_nbest(table, n_ctx, n_vocab, first_token, eot, (int)beam_size, (int)max_depth)[0].ids;
    if ((int64_t)best.size() > capacity) return -1;
    std::copy(best.begin(), best.end(), seq_out);
    return (int64_t)best.size();
}

int64_t wb_beam_nbest_table(const double* table, int64_t n_ctx, int64_t n_vocab, int64_t first_token, int64_t eot, int64_t beam_size,
                            int64_t max_depth, int64_t max_hyps, int64_t capacity, int64_t* ids_out, int64_t* lens_out,
                            double* scores_out, int32_t* finished_out) {
    if (!ids_out || !lens_out || !scores_out || !table_args_ok(table, n_ctx, n_vocab, beam_size, max_depth) || max_hyps < 0 ||
        capacity < 0) return -1;
    const wb::NBest nb = table_nbest(table, n_ctx, n_vocab, first_token, eot, (int)beam_size, (int)max_depth);
    if ((int64_t)nb.size() > max_hyps) return -1;
    for (size_t r = 0; r < nb.size(); ++r) {
        const wb::Hypothesis& h = nb[r];
        if ((int64_t)h.ids.size() > capacity) return -1;
        std::copy(h.ids.begin(), h.ids.end(), ids_out + (int64_t)r * capacity);
        lens_out[r] = (int64_t)h.ids.size();
        scores_out[r] = h.score;
        if (finished_out) finished_out[r] = h.finished ? 1 : 0;
    }
    return (int64_t)nb.size();
}

int64_t wb_kernel_launch_count(void) { return wb::g_launch_count; }
void wb_kernel_launch_count_reset(void) { wb::g_launch_count = 0; }

int wb_session_last_timings(wb_session* s, float* ms_out4) {
    return guarded([&] {
        WB_REQUIRE(s && ms_out4, "null pointer");
        for (int i = 0; i < 4; ++i) ms_out4[i] = s->impl->last_ms[i];
    });
}

int wb_session_profile_decode(wb_session* s, const wb_special_ids* ids, int n_steps, float* logits_kernel_ms,
                              float* step_ms) {
    return guarded([&] {
        WB_REQUIRE(s && ids && logits_kernel_ms && step_ms, "null pointer");
        const int64_t prompt[4] = {ids->sot, ids->lang, ids->transcribe, ids->notimestamps};
        s->impl->profile_decode(prompt, 4, n_steps, logits_kernel_ms, step_ms);
    });
}

int wb_session_last_steps(wb_session* s, int64_t* n_steps_out) {
    return guarded([&] {
        WB_REQUIRE(s && n_steps_out, "null pointer");
        *n_steps_out = s->impl->last_steps;
    });
}

}  // extern "C"
