// Host pipeline above the kernels: the token side of src/transcribe.rs.
//   window_bounds        waveform_to_mel_tensor  transcribe.rs:114-138
//   transcribe_windows   mels_to_text            transcribe.rs:148-383 (prompt :195-203, search :232-309)
//   find_chunk_overlap                           transcribe.rs:76-110
// All windows of a call advance in lock-step: one batched device step per search depth evaluates
// the live beams of every unfinished window (the reference evaluates one window at a time and
// re-runs the whole decoder per step; results per window are identical because windows are
// independent, SURVEY.md F9).
#include <algorithm>

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

struct BeamSearchToken {   // transcribe.rs:142-146 (+ the cache row that produced it)
    int64_t token;
    double log_prob;
    int32_t row;           // device row whose K/V ancestry this token extends
};
using Node = beam::BeamNode<BeamSearchToken>;

// the beam search on the host, all windows in lock-step at one position p, one decoder launch per position
// (Session::step_beams).  Window w's search starts at p = prompts[w].size() - 1; until then its prompt node rides along in
// one row (its own row as parent, its next prompt token) and its candidates are discarded.
void host_beam_search(Session& s, const std::vector<std::vector<int64_t>>& prompts, int beam_size, int max_depth, int64_t eot,
                      std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp) {
    const int W = s.n_windows;
    auto is_finished = [eot](const std::vector<BeamSearchToken>& seq) { return !seq.empty() && seq.back().token == eot; };
    std::vector<std::vector<Node>> beams((size_t)W);
    std::vector<char> done((size_t)W, 0);
    for (int w = 0; w < W; ++w) {
        Node n;
        for (int64_t t : prompts[(size_t)w]) n.seq.push_back(BeamSearchToken{t, 0.0, w});
        n.log_prob = 0.0;
        beams[(size_t)w].push_back(std::move(n));
    }
    s.begin(prompts);
    std::vector<int32_t> win_of_row, parent;
    std::vector<int64_t> tok, top_id;
    std::vector<float> top_lp;
    int64_t steps = 0;
    for (;;) {
        const int p = s.host_pos;
        auto searching = [&](int w) { return p + 1 >= (int)prompts[(size_t)w].size(); };
        // beam.rs:22-27: stop a search when its best beam is finished, or after max_depth steps past its prompt
        bool any = false;
        for (int w = 0; w < W; ++w) {
            if (done[(size_t)w]) continue;
            const int best = beam::max_by_last(beams[(size_t)w]);
            if (searching(w) && ((best >= 0 && is_finished(beams[(size_t)w][(size_t)best].seq)) ||
                                 p + 1 - (int)prompts[(size_t)w].size() >= max_depth))
                done[(size_t)w] = 1;
            else any = true;
        }
        if (!any) break;
        // rows = live beams of unfinished windows, window-major
        win_of_row.clear(); parent.clear(); tok.clear();
        std::vector<std::vector<int>> row_of_beam((size_t)W);
        size_t max_seq_len = 0;   // over searching windows: every one's longest beam has p + 1 tokens
        for (int w = 0; w < W; ++w) {
            if (done[(size_t)w]) continue;
            if (!searching(w)) {   // the prompt node: the token at p, its row extended by one position
                BeamSearchToken& last = beams[(size_t)w][0].seq.back();
                parent.push_back(last.row);
                last.row = (int32_t)win_of_row.size();
                win_of_row.push_back(w);
                tok.push_back(prompts[(size_t)w][(size_t)p]);
                continue;
            }
            row_of_beam[(size_t)w].assign(beams[(size_t)w].size(), -1);
            for (size_t b = 0; b < beams[(size_t)w].size(); ++b) {
                const Node& n = beams[(size_t)w][b];
                max_seq_len = std::max(max_seq_len, n.seq.size());
                if (is_finished(n.seq)) continue;   // continuations of finished beams are discarded (beam.rs:56-57)
                row_of_beam[(size_t)w][b] = (int)win_of_row.size();
                win_of_row.push_back(w);
                parent.push_back(n.seq.back().row);
                tok.push_back(n.seq.back().token);
            }
        }
        const int64_t n_rows = (int64_t)win_of_row.size();
        if (n_rows == 0) break;
        const int k = beam_size;
        top_id.resize((size_t)n_rows * k);
        top_lp.resize((size_t)n_rows * k);
        const int apply_mask = max_seq_len > 5 ? 0 : 1;   // transcribe.rs:271-275
        s.step_beams(n_rows, win_of_row.data(), parent.data(), tok.data(), apply_mask, k, top_id.data(), top_lp.data());
        ++steps;
        for (int w = 0; w < W; ++w) {
            if (done[(size_t)w] || !searching(w)) continue;
            auto next = [&](const std::vector<Node>& bs) {
                std::vector<std::vector<std::pair<BeamSearchToken, double>>> conts(bs.size());
                for (size_t b = 0; b < bs.size(); ++b) {
                    const int row = row_of_beam[(size_t)w][b];
                    if (row < 0) continue;
                    // candidates in ascending token order, as the reference enumerates the vocabulary
                    std::vector<std::pair<int64_t, float>> c;
                    for (int i = 0; i < k; ++i)
                        if (top_id[(size_t)row * k + i] >= 0) c.emplace_back(top_id[(size_t)row * k + i], top_lp[(size_t)row * k + i]);
                    std::sort(c.begin(), c.end(), [](const auto& a, const auto& b2) { return a.first < b2.first; });
                    for (const auto& e : c)
                        conts[b].emplace_back(BeamSearchToken{e.first, (double)e.second, row},
                                              bs[b].log_prob + (double)e.second);   // transcribe.rs:291-299
                }
                return conts;
            };
            beams[(size_t)w] = beam::beam_search_step(beams[(size_t)w], next, is_finished, (size_t)beam_size);
        }
    }
    s.last_steps = steps;
    out.assign((size_t)W, {});
    out_lp.assign((size_t)W, {});
    for (int w = 0; w < W; ++w) {
        const int best = beam::max_by_last(beams[(size_t)w]);
        if (best >= 0)
            for (const auto& t : beams[(size_t)w][(size_t)best].seq) {
                out[(size_t)w].push_back(t.token);
                out_lp[(size_t)w].push_back((float)t.log_prob);   // exact: a widened f32 (transcribe.rs:291-299)
            }
    }
}

}  // namespace

void transcribe_windows(Session& s, int beam_size, int max_depth, const wb_special_ids& ids, const uint8_t* is_special,
                        std::vector<std::vector<int64_t>>& out, std::vector<std::vector<float>>& out_lp,
                        const std::vector<std::vector<int64_t>>& prev, int64_t startofprev) {
    const bool loop = s.search == WB_SEARCH_GREEDY_LOOP;
    WB_REQUIRE(!loop || beam_size == 1, "transcribe: the greedy loop takes beam_size 1");
    WB_REQUIRE(beam_size >= 1 && beam_size <= s.max_beams, "transcribe: beam_size exceeds the session's max_beams");
    WB_REQUIRE(max_depth >= 0, "transcribe: negative max_depth");
    WB_REQUIRE(prev.empty() || (int64_t)prev.size() == s.n_windows, "transcribe: one previous-id list per window");
    const int V = s.m->dims.n_vocab;
    const int64_t head[4] = {ids.sot, ids.lang, ids.transcribe, ids.notimestamps};   // transcribe.rs:203
    for (int64_t t : head) WB_REQUIRE(t >= 0 && t < V, "transcribe: special id out of range");
    WB_REQUIRE(ids.eot >= 0 && ids.eot < V, "transcribe: eot id out of range");
    // window w's prompt: [startofprev] + prev[w] + the four ids when prev[w] is not empty (transcribe.rs:195-203 without the
    // shadowing at :201), else the four ids
    std::vector<std::vector<int64_t>> prompts((size_t)s.n_windows);
    for (size_t w = 0; w < prompts.size(); ++w) {
        std::vector<int64_t>& pr = prompts[w];
        if (!prev.empty() && !prev[w].empty()) {
            WB_REQUIRE(!loop, "transcribe: the greedy loop builds its own prompt; no previous ids with it");
            WB_REQUIRE(startofprev >= 0 && startofprev < V, "transcribe: startofprev id out of range");
            pr.push_back(startofprev);
            for (int64_t t : prev[w]) {
                WB_REQUIRE(t >= 0 && t < V, "transcribe: previous id out of range");
                pr.push_back(t);
            }
        }
        pr.insert(pr.end(), head, head + 4);
        WB_REQUIRE((int64_t)pr.size() + max_depth <= s.t_max, "transcribe: prompt + max_depth exceeds the session's max_text_len");
    }
    s.set_special(is_special);
    if (beam_size == 1)   // greedy: beam_size 1 of the search, or the greedy loop (transcribe.rs:314-380)
        s.greedy_decode(prompts, max_depth, ids.eot, out, out_lp, loop);
    // beam search: on the device in one launch where decoder6 covers it (fp16-exact weights, d = 128 / 384,
    // n_windows * beam_size <= 24, t_max <= 128), same selection rules and ids as the host search
    else if (max_depth == 0 || !s.beam_decode(prompts, beam_size, max_depth, ids.eot, out, out_lp))
        host_beam_search(s, prompts, beam_size, max_depth, ids.eot, out, out_lp);
    WB_CUDA(cudaEventRecord(s.ev[3], s.st));
}

}  // namespace wb
