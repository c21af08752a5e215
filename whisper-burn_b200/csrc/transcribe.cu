// Host pipeline above the kernels: the token side of src/transcribe.rs, behind every decode entry point of the C ABI.
//   waveforms_to_tokens  waveform_to_text        transcribe.rs:23-74 (previous ids :43-54, merge :56-63)
//   window_bounds        waveform_to_mel_tensor  transcribe.rs:114-138
//   transcribe_windows   mels_to_text            transcribe.rs:148-383 (prompt: window_prompts :195-203, search :232-309)
//   find_chunk_overlap                           transcribe.rs:76-110
// All windows of a call advance in lock-step: one batched device step per search depth evaluates
// the live beams of every unfinished window (the reference evaluates one window at a time and
// re-runs the whole decoder per step; results per window are identical because windows are
// independent, SURVEY.md F9).
#include <algorithm>
#include <functional>

#include "../host/beam.hpp"
#include "session.h"

namespace wb {

std::vector<std::pair<int64_t, int64_t>> window_bounds(int64_t n_samples, int64_t sample_rate, int64_t window_len) {
    const int64_t chunk_overlap = sample_rate * 3;                                    // transcribe.rs:120
    const int64_t shift = std::max<int64_t>(std::max<int64_t>(window_len - chunk_overlap, 0), 1);   // saturating_sub.max(1)
    const int64_t iter_len = std::max<int64_t>(n_samples - 1, 0) / shift + 1;
    std::vector<std::pair<int64_t, int64_t>> out;
    for (int64_t i = 0; i < iter_len; ++i) {
        const int64_t start = i * shift;
        out.emplace_back(start, std::min(start + window_len, n_samples));
    }
    return out;
}

bool find_chunk_overlap(const int64_t* prev, int64_t n_prev, const int64_t* curr, int64_t n_curr, int64_t max_n_offsets,
                        int64_t min_n_overlaps, int64_t* prev_index, int64_t* curr_index) {
    int64_t max_overlap = 0, best_prev = 0, best_curr = 0;
    const int64_t n_offsets = std::min(std::min(n_prev, n_curr), max_n_offsets);
    for (int64_t offset = 0; offset < n_offsets; ++offset) {
        const int64_t prev_start = n_prev - 1 - offset;
        int64_t n_overlap = 0, first = -1;
        for (int64_t i = 0; prev_start + i < n_prev && i < n_curr; ++i) {
            if (prev[prev_start + i] == curr[i]) {
                if (first < 0) first = i;
                ++n_overlap;
            }
        }
        if (n_overlap > max_overlap) {
            max_overlap = n_overlap;
            best_prev = prev_start + first;
            best_curr = first;
        }
    }
    if (max_overlap >= min_n_overlaps) {
        *prev_index = best_prev;
        *curr_index = best_curr;
        return true;
    }
    return false;
}

namespace {

// the host beam search (beam_search_windows) of every encoded window, one decoder launch per position (Session::step_beams)
void host_beam_search(Session& s, const std::vector<std::vector<int64_t>>& prompts, int beam_size, int max_depth, int64_t eot,
                      std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp, std::vector<NBest>& nbest) {
    s.begin(prompts);
    std::vector<float> lp32;
    auto step = [&](int, int64_t n_rows, const int32_t* window_of_row, const int32_t* parent_row, const int64_t* token,
                    int apply_mask, int k, int64_t* ids_out, double* lps_out) {
        lp32.resize((size_t)n_rows * k);
        s.step_beams(n_rows, window_of_row, parent_row, token, apply_mask, k, ids_out, lp32.data());
        std::copy(lp32.begin(), lp32.end(), lps_out);
    };
    int64_t steps = 0;
    const std::vector<Carried> carried = beam_search_windows(prompts, s.host_pos, beam_size, max_depth, eot, step, &steps);
    s.last_steps = steps;
    // each window's final carried list, ranked; the best row is its rank 0 (max_by_last)
    out.assign(carried.size(), {});
    out_lp.assign(carried.size(), {});
    nbest.assign(carried.size(), {});
    for (size_t w = 0; w < carried.size(); ++w) {
        nbest[w] = ranked_nbest(carried[w]);
        if (nbest[w].empty()) continue;
        out[w] = nbest[w][0].ids;
        out_lp[w] = nbest[w][0].lps;
    }
}

// the one-hypothesis list of a beam_size 1 row: the carried list of a width-1 search holds one node, the row itself, whose
// cumulative log-prob is the left-to-right f64 sum of its ids' log-probs
NBest row_nbest(const std::vector<int64_t>& ids, const std::vector<float>& lps, int64_t eot) {
    Hypothesis h;
    h.ids = ids;
    h.lps = lps;
    for (float l : lps) h.score += (double)l;
    h.finished = !ids.empty() && ids.back() == eot;
    return NBest{std::move(h)};
}

// per window the ids and the log-prob each was chosen with (BeamSearchToken.log_prob), decoded from prompts[w] on the
// encoded windows, and the window's n-best list (none under the greedy loop)
void decode_windows(Session& s, const std::vector<std::vector<int64_t>>& prompts, int beam_size, int max_depth, int64_t eot,
                    const uint8_t* is_special, std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp,
                    std::vector<NBest>& nbest) {
    s.set_special(is_special);
    nbest.clear();
    if (beam_size == 1) {   // greedy: beam_size 1 of the search, or the greedy loop (transcribe.rs:314-380)
        const bool loop = s.search == WB_SEARCH_GREEDY_LOOP;
        s.greedy_decode(prompts, max_depth, eot, out, out_lp, loop);
        if (!loop)
            for (size_t w = 0; w < out.size(); ++w) nbest.push_back(row_nbest(out[w], out_lp[w], eot));
    }
    // beam search: on the device in one launch where decoder6 covers it (fp16-exact weights, d = 128 / 384,
    // n_windows * beam_size <= 24, t_max <= 128), same selection rules and ids as the host search
    else if (max_depth == 0 || !s.beam_decode(prompts, beam_size, max_depth, eot, out, out_lp, nbest))
        host_beam_search(s, prompts, beam_size, max_depth, eot, out, out_lp, nbest);
    WB_CUDA(cudaEventRecord(s.ev[3], s.st));
}

// the phases the encode and decode_windows recorded: log-mel, encoder + cross K/V, decode, total
void collect_timings(Session& s) {
    WB_CUDA(cudaStreamSynchronize(s.st));
    cudaEventElapsedTime(&s.last_ms[0], s.ev[0], s.ev[1]);
    cudaEventElapsedTime(&s.last_ms[1], s.ev[1], s.ev[2]);
    cudaEventElapsedTime(&s.last_ms[2], s.ev[2], s.ev[3]);
    cudaEventElapsedTime(&s.last_ms[3], s.ev[0], s.ev[3]);
}

// the overlap merge of one window's ids and log-probs into its waveform's (transcribe.rs:56-63)
void merge_window(std::vector<int64_t>& tokens, std::vector<float>& tlp, const std::vector<int64_t>& nt,
                  const std::vector<float>& nl) {
    int64_t pi = 0, ci = 0;
    if (find_chunk_overlap(tokens.data(), (int64_t)tokens.size(), nt.data(), (int64_t)nt.size(), 40, 3, &pi, &ci)) {
        tokens.resize((size_t)pi);                                    // transcribe.rs:59-60
        tokens.insert(tokens.end(), nt.begin() + ci, nt.end());
        tlp.resize((size_t)pi);
        tlp.insert(tlp.end(), nl.begin() + ci, nl.end());
    } else {
        tokens.insert(tokens.end(), nt.begin(), nt.end());
        tlp.insert(tlp.end(), nl.begin(), nl.end());
    }
}

// transcribe.rs:43-50: the last (at most) 5 ids of the merged tokens that are not special, in order
std::vector<int64_t> prev_nonspecial(const std::vector<int64_t>& tokens, const uint8_t* is_special) {
    std::vector<int64_t> prev;
    for (size_t i = tokens.size(); i-- > 0 && prev.size() < 5;)
        if (!is_special[tokens[i]]) prev.push_back(tokens[i]);
    std::reverse(prev.begin(), prev.end());
    return prev;
}

}  // namespace

std::vector<std::vector<int64_t>> window_prompts(const Session& s, int64_t n_windows, int beam_size, int max_depth,
                                                 const wb_special_ids& ids, const uint8_t* is_special,
                                                 const std::vector<std::vector<int64_t>>& prev, int64_t startofprev) {
    const bool loop = s.search == WB_SEARCH_GREEDY_LOOP;
    WB_REQUIRE(n_windows >= 1 && n_windows <= s.max_windows, "transcribe: n_windows out of range for this session");
    WB_REQUIRE(is_special || loop, "transcribe: is_special is needed outside the greedy loop");
    WB_REQUIRE(!loop || beam_size == 1, "transcribe: the greedy loop takes beam_size 1");
    WB_REQUIRE(beam_size >= 1 && beam_size <= s.max_beams, "transcribe: beam_size exceeds the session's max_beams");
    WB_REQUIRE(max_depth >= 0, "transcribe: negative max_depth");
    WB_REQUIRE(prev.empty() || (int64_t)prev.size() == n_windows, "transcribe: one previous-id list per window");
    const int V = s.m->dims.n_vocab;
    WB_REQUIRE(prev.empty() || (startofprev >= 0 && startofprev < V), "transcribe: startofprev id out of range");
    const int64_t head[4] = {ids.sot, ids.lang, ids.transcribe, ids.notimestamps};   // transcribe.rs:203
    for (int64_t t : head) WB_REQUIRE(t >= 0 && t < V, "transcribe: special id out of range");
    WB_REQUIRE(ids.eot >= 0 && ids.eot < V, "transcribe: eot id out of range");
    std::vector<std::vector<int64_t>> prompts((size_t)n_windows);
    for (size_t w = 0; w < prompts.size(); ++w) {
        std::vector<int64_t>& pr = prompts[w];
        if (!prev.empty() && !prev[w].empty()) {
            WB_REQUIRE(!loop, "transcribe: the greedy loop builds its own prompt; no previous ids with it");
            pr.push_back(startofprev);
            for (int64_t t : prev[w]) {
                WB_REQUIRE(t >= 0 && t < V, "transcribe: previous id out of range");
                pr.push_back(t);
            }
        }
        pr.insert(pr.end(), head, head + 4);
        WB_REQUIRE((int64_t)pr.size() + max_depth <= s.t_max, "transcribe: prompt + max_depth exceeds the session's max_text_len");
    }
    return prompts;
}

std::vector<std::vector<int64_t>> transcribe_windows(Session& s, const std::vector<std::vector<int64_t>>& prompts, int beam_size,
                                                     int max_depth, int64_t eot, const uint8_t* is_special, int64_t capacity,
                                                     const std::function<void()>& encode) {
    s.have_logprobs = false;
    s.have_nbest = false;
    encode();
    std::vector<std::vector<int64_t>> out;
    decode_windows(s, prompts, beam_size, max_depth, eot, is_special, out, s.last_logprobs, s.last_nbest);
    for (const auto& row : out) WB_REQUIRE((int64_t)row.size() <= capacity, "tokens_out capacity too small");
    collect_timings(s);
    s.have_logprobs = true;
    s.have_nbest = s.search == WB_SEARCH_BEAM;
    return out;
}

namespace {

// one window of a waveform call: samples [start, start + len) of waveform `owner`
struct WaveWindow {
    int owner;
    int64_t start, len;
};

// the checks of a waveform call that come before its windows are cut
void check_waveform_call(const Session& s, int64_t n_waveforms) {
    WB_REQUIRE(n_waveforms >= 1, "waveforms_to_tokens: n_waveforms must be >= 1");
    WB_REQUIRE(s.startofprev < 0 || s.search != WB_SEARCH_GREEDY_LOOP,
               "waveform_to_tokens: the previous-text prompt (set_prev_prompt) does not combine with the greedy loop");
}

// the windows of every waveform of n_samples[w] 16 kHz samples, waveform-major (transcribe.rs:32-34, 114-138)
std::vector<WaveWindow> waveform_windows(const Session& s, const int64_t* n_samples, int64_t n_waveforms) {
    const int64_t window_len = window_samples(s.m->dims.n_audio_ctx, s.window_mode);
    std::vector<WaveWindow> wins;
    for (int64_t w = 0; w < n_waveforms; ++w)
        for (const auto& b : window_bounds(n_samples[w], 16000, window_len)) wins.push_back(WaveWindow{(int)w, b.first, b.second - b.first});
    return wins;
}

// windows of ALL waveforms are decoded together in batches of the session's capacity (they are independent,
// SURVEY.md F9), then each waveform's windows are merged in order exactly like the reference's sequential
// loop (transcribe.rs:42-71); each id's log-prob travels with it through the merge.
// With the previous-text prompt (Session::startofprev >= 0) window i of a waveform needs the merged ids of windows
// 0 .. i-1: round i decodes window i of every waveform that has one, in batches of the session's capacity.
// encode_batch encodes one batch of windows, after that batch's arguments are checked.
std::vector<std::vector<int64_t>> window_loop(Session& s, const std::vector<WaveWindow>& wins, int64_t n_waveforms, int beam_size,
                                              int max_depth, const wb_special_ids& ids, const uint8_t* is_special, int64_t capacity,
                                              const std::function<void(const std::vector<WaveWindow>&)>& encode_batch) {
    const bool prev_prompt = s.startofprev >= 0;
    std::vector<std::vector<int64_t>> out((size_t)n_waveforms);
    std::vector<std::vector<float>> out_lp((size_t)n_waveforms);
    std::vector<NBest> nbest(wins.size());   // per window, waveform-major
    // batches: window-major order (all windows at once) or, with the previous-text prompt, rounds of window index i
    std::vector<std::vector<size_t>> rounds(1);
    std::vector<size_t> idx((size_t)n_waveforms, 0);   // per waveform, the index of its next window
    for (size_t j = 0; j < wins.size(); ++j) {
        const size_t i = prev_prompt ? idx[(size_t)wins[j].owner]++ : 0;
        if (rounds.size() <= i) rounds.resize(i + 1);
        rounds[i].push_back(j);
    }
    for (const std::vector<size_t>& round : rounds) {
        for (size_t b0 = 0; b0 < round.size(); b0 += (size_t)s.max_windows) {
            const size_t nb = std::min(round.size() - b0, (size_t)s.max_windows);
            std::vector<WaveWindow> batch(nb);
            std::vector<std::vector<int64_t>> prev(prev_prompt ? nb : 0);
            for (size_t i = 0; i < nb; ++i) {
                batch[i] = wins[round[b0 + i]];
                if (prev_prompt) prev[i] = prev_nonspecial(out[(size_t)batch[i].owner], is_special);
            }
            const auto prompts = window_prompts(s, (int64_t)nb, beam_size, max_depth, ids, is_special, prev, s.startofprev);
            s.have_logprobs = false;
            s.have_nbest = false;
            encode_batch(batch);
            std::vector<std::vector<int64_t>> toks;
            std::vector<std::vector<float>> lps;
            std::vector<NBest> nbs;
            decode_windows(s, prompts, beam_size, max_depth, ids.eot, is_special, toks, lps, nbs);
            for (size_t i = 0; i < nb; ++i) {
                merge_window(out[(size_t)batch[i].owner], out_lp[(size_t)batch[i].owner], toks[i], lps[i]);
                if (!nbs.empty()) nbest[round[b0 + i]] = std::move(nbs[i]);
            }
        }
    }
    collect_timings(s);
    for (const auto& row : out) WB_REQUIRE((int64_t)row.size() <= capacity, "tokens_out capacity (per waveform) too small");
    s.last_logprobs = std::move(out_lp);
    s.have_logprobs = true;
    s.last_nbest = std::move(nbest);
    s.have_nbest = s.search == WB_SEARCH_BEAM;
    return out;
}

}  // namespace

std::vector<std::vector<int64_t>> waveforms_to_tokens(Session& s, const float* const* waveforms, const int64_t* n_samples,
                                                      int64_t n_waveforms, int64_t sample_rate, int beam_size, int max_depth,
                                                      const wb_special_ids& ids, const uint8_t* is_special, int64_t capacity) {
    check_waveform_call(s, n_waveforms);
    // the frontend tables (mel filterbank, DFT bins) are the 16 kHz ones: the reference builds them from the caller's rate
    // (audio.rs:44, 67-143) but its binary only ever passes 16 kHz (src/bin/transcribe/main.rs:38-41 asserts it);
    // waveforms_to_tokens_resampled converts other rates first
    WB_REQUIRE(sample_rate == 16000, "waveform_to_tokens: only 16 kHz input is supported (frontend tables are built for 16 kHz)");
    return window_loop(s, waveform_windows(s, n_samples, n_waveforms), n_waveforms, beam_size, max_depth, ids, is_special, capacity,
                       [&](const std::vector<WaveWindow>& batch) {
                           std::vector<const float*> bp(batch.size());
                           std::vector<int64_t> bl(batch.size());
                           for (size_t i = 0; i < batch.size(); ++i) {
                               bp[i] = waveforms[batch[i].owner] + batch[i].start;
                               bl[i] = batch[i].len;
                           }
                           s.encode_waveforms_host(bp.data(), bl.data(), (int64_t)batch.size());
                       });
}

std::vector<std::vector<int64_t>> waveforms_to_tokens_resampled(Session& s, const float* const* waveforms, const int64_t* n_frames,
                                                                const int64_t* channels, const int64_t* sample_rates,
                                                                int64_t n_waveforms, int beam_size, int max_depth,
                                                                const wb_special_ids& ids, const uint8_t* is_special,
                                                                int64_t capacity) {
    // every argument check that does not depend on decoded ids, before the upload and the resample
    check_waveform_call(s, n_waveforms);
    std::vector<int64_t> n16((size_t)n_waveforms);
    for (int64_t w = 0; w < n_waveforms; ++w) {
        WB_REQUIRE(waveforms[w] != nullptr, "waveforms_to_tokens_resampled: null waveform");
        WB_REQUIRE(n_frames[w] >= 1, "waveforms_to_tokens_resampled: n_frames must be >= 1");
        WB_REQUIRE(channels[w] >= 1 && channels[w] <= INT32_MAX, "waveforms_to_tokens_resampled: channels must be >= 1");
        n16[(size_t)w] = resampled_length(n_frames[w], sample_rates[w]);
        if (n16[(size_t)w] < 0) fail(WB_ERR_UNSUPPORTED, "waveforms_to_tokens_resampled: unsupported sample rate (gcd with 16000 "
                                                         "must leave up and down <= 1024)");
        WB_REQUIRE(n_frames[w] <= INT64_MAX / channels[w], "waveforms_to_tokens_resampled: waveform too long");
    }
    const std::vector<WaveWindow> wins = waveform_windows(s, n16.data(), n_waveforms);
    for (const WaveWindow& win : wins) WB_REQUIRE(win.len >= N_FFT, "prep_audio: waveform shorter than n_fft (audio.rs:292)");
    const int64_t first_batch = std::min<int64_t>(s.startofprev >= 0 ? n_waveforms : (int64_t)wins.size(), s.max_windows);
    window_prompts(s, first_batch, beam_size, max_depth, ids, is_special);
    std::vector<int64_t> off, n_out;
    resample_waveforms(s.rs, waveforms, n_frames, channels, sample_rates, n_waveforms, off, n_out, s.st);
    return window_loop(s, wins, n_waveforms, beam_size, max_depth, ids, is_special, capacity,
                       [&](const std::vector<WaveWindow>& batch) {
                           std::vector<int64_t> bo(batch.size()), bl(batch.size());
                           for (size_t i = 0; i < batch.size(); ++i) {
                               bo[i] = off[(size_t)batch[i].owner] + batch[i].start;
                               bl[i] = batch[i].len;
                           }
                           s.encode_from_device_wave(s.rs.out.p, bo.data(), bl.data(), (int64_t)batch.size());
                       });
}

}  // namespace wb
