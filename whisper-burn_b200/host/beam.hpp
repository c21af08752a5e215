// The library's one beam search (src/beam.rs:9-110, src/transcribe.rs:232-309).  One step runs over fixed-capacity arrays,
// callable from host and device code: decoder6.cu's beam mode runs it on the GPU, one warp per window, and the host window loop
// below (beam_search_windows) runs it on the CPU for every other beam search and for the table-driven entry points the CPU
// tests drive.  The restatement the tests compare against is the Python oracle (oracle/beam.py).  The step's choices:
//   * the continuations of a live beam are its (at most beam_size) candidates in ascending token id, as the reference
//     enumerates the vocabulary; score = parent log-prob + (double) candidate log-prob;
//   * get_top_elements: on exact ties the EARLIER element wins, output in ascending score;
//   * carried list = top beam_size of the continuations, then top beam_size of the beams that were already finished;
//   * max_by_last: the LAST maximum.  A beam is finished when its last token is eot; its continuations are discarded.
// Token sequences are not touched here: a Pick says which input node a carried node extends and by which token, and the caller
// copies sequences (the device does it warp-parallel).
#pragma once

#include <stdint.h>

#include <algorithm>
#include <vector>

#if defined(__CUDACC__)
#define WB_HD __host__ __device__
#else
#define WB_HD
#endif

namespace wb {
namespace beamfx {

constexpr int MAX_BEAM = 7;                    // beam_size <= 7 (candidates kept per record by the persistent decoders: 8)
constexpr int MAX_NODES = 2 * MAX_BEAM;        // carried: <= beam_size live + <= beam_size finished
constexpr int MAX_CONT = MAX_BEAM * MAX_BEAM;  // continuations of one step

struct Head {          // a carried node without its token sequence
    double log_prob;   // cumulative
    int finished;      // last token is eot
    int row;           // decoder cache row that scored its last token (its parent's row at that step)
    int len;           // tokens in its sequence
    int pad;
};

struct Pick {          // one node of the next carried list
    Head head;
    int src;           // the input node it extends (token >= 0) or carries unchanged (token < 0)
    int token;
    double lp;         // the appended token's own log-prob (the candidate's cand_lp); 0 when token < 0
};

// get_top_elements (beam.rs:81-110) over scores s[0..n), num <= MAX_BEAM: writes the kept indices in output order to top
// (capacity num + 1), returns how many were kept
WB_HD inline int top_elements(const double* s, int n, int num, int* top) {
    double sc[MAX_BEAM + 1];
    int cnt = 0;
    for (int e = 0; e < n; ++e) {
        const double v = s[e];
        if (cnt == num && (num == 0 || v < sc[0])) continue;
        int idx = cnt;
        for (int i = 0; i < cnt; ++i)
            if (sc[i] >= v) { idx = i; break; }
        for (int i = cnt; i > idx; --i) { sc[i] = sc[i - 1]; top[i] = top[i - 1]; }
        sc[idx] = v;
        top[idx] = e;
        if (++cnt > num) {
            for (int i = 0; i + 1 < cnt; ++i) { sc[i] = sc[i + 1]; top[i] = top[i + 1]; }
            --cnt;
        }
    }
    return cnt;
}

// Iterator::max_by(partial_cmp): the last maximum; -1 if n == 0
WB_HD inline int max_by_last(const Head* h, int n) {
    int best = -1;
    for (int i = 0; i < n; ++i)
        if (best < 0 || !(h[i].log_prob < h[best].log_prob)) best = i;
    return best;
}

// The n-best ranking of a final carried list (beam.rs:33-36 applied again to what remains after each pick): max_by_last
// repeatedly, i.e. descending log-prob with exact ties ordered by LATER carried position first.  Writes the carried indices
// best first to order[0..n); order[0] is max_by_last.  Every n-best list (host search, device search, table helpers) is
// ranked here.  (An insertion that places node i before the first kept node it is not below gives the same order.)
WB_HD inline void rank_final(const double* log_prob, int n, int* order) {
    for (int i = 0; i < n; ++i) {
        int k = i;
        for (; k > 0 && !(log_prob[order[k - 1]] > log_prob[i]); --k) order[k] = order[k - 1];
        order[k] = i;
    }
}

// beam_search (beam.rs:22-27): the search stops when its best carried node is finished
WB_HD inline bool search_done(const Head* h, int n) {
    const int best = max_by_last(h, n);
    return best >= 0 && h[best].finished != 0;
}

// beam_search_step (beam.rs:39-79) for one window.  in[0..n_in) = the carried nodes.  A live node b has beam_size candidate
// slots cand_id / cand_lp [b * beam_size + i] in any order (ids < 0 are empty) and was scored by cache row step_row[b].
// Writes the next carried list (<= 2 * beam_size nodes, live results first) to out and returns its length.
WB_HD inline int beam_step(const Head* in, int n_in, const int* step_row, const int* cand_id, const double* cand_lp, int beam_size,
                           int eot, Pick* out) {
    double ns[MAX_CONT], fs[MAX_NODES];
    int nsrc[MAX_CONT], nslot[MAX_CONT], fsrc[MAX_NODES];   // a continuation: its node, its candidate slot, its score
    int n_new = 0, n_fin = 0;
    for (int b = 0; b < n_in; ++b) {
        if (in[b].finished) {
            fsrc[n_fin] = b;
            fs[n_fin++] = in[b].log_prob;
            continue;
        }
        // this beam's continuations in ascending token id (insertion sort of its <= 7 candidate slots)
        int slot[MAX_BEAM];
        int nc = 0;
        for (int i = 0; i < beam_size; ++i) {
            const int s = b * beam_size + i, t = cand_id[s];
            if (t < 0) continue;
            int k = nc++;
            for (; k > 0 && cand_id[slot[k - 1]] > t; --k) slot[k] = slot[k - 1];
            slot[k] = s;
        }
        double sc[MAX_BEAM];
        for (int i = 0; i < nc; ++i) sc[i] = in[b].log_prob + cand_lp[slot[i]];   // transcribe.rs:291-299
        int top[MAX_BEAM + 1];
        const int nt = top_elements(sc, nc, beam_size, top);
        for (int i = 0; i < nt; ++i) {
            nsrc[n_new] = b;
            nslot[n_new] = slot[top[i]];
            ns[n_new++] = sc[top[i]];
        }
    }
    int top[MAX_BEAM + 1];
    int n_out = 0;
    const int nl = top_elements(ns, n_new, beam_size, top);
    for (int i = 0; i < nl; ++i) {
        const int c = top[i], b = nsrc[c];
        Pick& o = out[n_out++];
        o.src = b;
        o.token = cand_id[nslot[c]];
        o.lp = cand_lp[nslot[c]];
        o.head.log_prob = ns[c];
        o.head.finished = o.token == eot ? 1 : 0;
        o.head.row = step_row[b];
        o.head.len = in[b].len + 1;
        o.head.pad = 0;
    }
    const int nf = top_elements(fs, n_fin, beam_size, top);
    for (int i = 0; i < nf; ++i) {
        const int b = fsrc[top[i]];
        Pick& o = out[n_out++];
        o.src = b;
        o.token = -1;
        o.lp = 0.0;
        o.head = in[b];
    }
    return n_out;
}

}  // namespace beamfx

// ---- host only ----------------------------------------------------------------------------------------------------------

// one hypothesis of a window's n-best list (wb_session_last_nbest): a node of the beam search's final carried list
struct Hypothesis {
    std::vector<int64_t> ids;   // prompt + generated ids
    std::vector<float> lps;     // 0 for each prompt id, else the log-prob the search scored the id with
    double score = 0.0;         // the node's cumulative log-prob as the search carried it
    bool finished = false;      // last id is eot
};
using NBest = std::vector<Hypothesis>;   // best first (beamfx::rank_final)

// one window's carried list: node i is heads[i], its ids ids[i] and their log-probs lps[i]
struct Carried {
    std::vector<beamfx::Head> heads;
    std::vector<std::vector<int64_t>> ids;
    std::vector<std::vector<float>> lps;
};

// the n-best list of a final carried list: its nodes ranked by beamfx::rank_final; rank 0 is the search's result (max_by_last)
inline NBest ranked_nbest(const Carried& c) {
    const int n = (int)c.heads.size();
    std::vector<double> lp((size_t)n);
    std::vector<int> order((size_t)n);
    for (int i = 0; i < n; ++i) lp[(size_t)i] = c.heads[(size_t)i].log_prob;
    beamfx::rank_final(lp.data(), n, order.data());
    NBest nb((size_t)n);
    for (int r = 0; r < n; ++r) {
        const size_t i = (size_t)order[(size_t)r];
        nb[(size_t)r] = Hypothesis{c.ids[i], c.lps[i], c.heads[i].log_prob, c.heads[i].finished != 0};
    }
    return nb;
}

// The beam search of every window on the host, all windows in lock-step at one position p = p0, p0 + 1, ..., one step call
// per position.  Window w's search starts at p = prompts[w].size() - 1; until then its prompt node rides along in one row (its
// own row as parent, its next prompt token) and its candidates are discarded.  A window is done when search_done holds
// (beam.rs:22-27) or after max_depth steps past its prompt.  A step's rows are the live nodes of the unfinished windows,
// window-major in carried order; apply_mask is 1 while the longest sequence of a searching window has at most 5 ids
// (transcribe.rs:271-275).
//   step(p, n_rows, window_of_row, parent_row, token, apply_mask, k, ids_out, lps_out) writes k = beam_size candidate slots
//   [n_rows][k] (int64_t ids, -1: empty; double log-probs) for the tokens at position p.
// Window w's prompt node starts in row w.  beam_size is 1 .. beamfx::MAX_BEAM.  Returns each window's final carried list;
// *steps = the number of step calls.
template <typename Step>
std::vector<Carried> beam_search_windows(const std::vector<std::vector<int64_t>>& prompts, int p0, int beam_size, int max_depth,
                                         int64_t eot, Step&& step, int64_t* steps) {
    namespace fx = beamfx;
    const int W = (int)prompts.size(), B = beam_size;
    std::vector<Carried> c((size_t)W);
    for (int w = 0; w < W; ++w) {
        const std::vector<int64_t>& pr = prompts[(size_t)w];
        c[(size_t)w].heads.push_back(fx::Head{0.0, pr.back() == eot ? 1 : 0, w, (int)pr.size(), 0});
        c[(size_t)w].ids.push_back(pr);
        c[(size_t)w].lps.emplace_back(pr.size(), 0.0f);   // transcribe.rs:205-208
    }
    std::vector<char> done((size_t)W, 0);
    std::vector<int32_t> win_of_row, parent;
    std::vector<int64_t> tok, cand_id;
    std::vector<double> cand_lp;
    int64_t n_steps = 0;
    for (int p = p0;; ++p) {
        auto searching = [&](int w) { return p + 1 >= (int)prompts[(size_t)w].size(); };
        bool any = false;
        for (int w = 0; w < W; ++w) {
            if (done[(size_t)w]) continue;
            const std::vector<fx::Head>& h = c[(size_t)w].heads;
            if (searching(w) && (fx::search_done(h.data(), (int)h.size()) || p + 1 - (int)prompts[(size_t)w].size() >= max_depth))
                done[(size_t)w] = 1;
            else any = true;
        }
        if (!any) break;
        win_of_row.clear(); parent.clear(); tok.clear();
        int max_len = 0;
        for (int w = 0; w < W; ++w) {
            if (done[(size_t)w]) continue;
            Carried& cw = c[(size_t)w];
            for (size_t b = 0; b < cw.heads.size(); ++b) {
                fx::Head& h = cw.heads[b];
                if (searching(w)) max_len = std::max(max_len, h.len);
                if (h.finished && searching(w)) continue;   // continuations of finished beams are discarded (beam.rs:56-57)
                parent.push_back(h.row);
                h.row = (int)win_of_row.size();
                win_of_row.push_back(w);
                tok.push_back(searching(w) ? cw.ids[b].back() : prompts[(size_t)w][(size_t)p]);
            }
        }
        const int64_t n_rows = (int64_t)win_of_row.size();
        if (n_rows == 0) break;
        cand_id.resize((size_t)n_rows * B);
        cand_lp.resize((size_t)n_rows * B);
        step(p, n_rows, win_of_row.data(), parent.data(), tok.data(), max_len > 5 ? 0 : 1, B, cand_id.data(), cand_lp.data());
        ++n_steps;
        for (int w = 0; w < W; ++w) {
            if (done[(size_t)w] || !searching(w)) continue;
            Carried& cw = c[(size_t)w];
            const int n = (int)cw.heads.size();
            int step_row[fx::MAX_NODES], id[fx::MAX_NODES * fx::MAX_BEAM];
            double lp[fx::MAX_NODES * fx::MAX_BEAM];
            for (int b = 0; b < n; ++b) {
                const fx::Head& h = cw.heads[(size_t)b];
                step_row[b] = h.row;
                if (h.finished) continue;   // beam_step reads no candidate of a finished node
                for (int i = 0; i < B; ++i) {
                    id[b * B + i] = (int)cand_id[(size_t)h.row * B + i];
                    lp[b * B + i] = cand_lp[(size_t)h.row * B + i];
                }
            }
            fx::Pick out[fx::MAX_NODES];
            const int n_out = fx::beam_step(cw.heads.data(), n, step_row, id, lp, B, (int)eot, out);
            Carried next;
            for (int i = 0; i < n_out; ++i) {
                const fx::Pick& o = out[i];
                next.heads.push_back(o.head);
                next.ids.push_back(cw.ids[(size_t)o.src]);
                next.lps.push_back(cw.lps[(size_t)o.src]);
                if (o.token < 0) continue;
                next.ids.back().push_back(o.token);
                next.lps.back().push_back((float)o.lp);   // the f32 the step scored the id with (transcribe.rs:291-299)
            }
            cw = std::move(next);
        }
    }
    *steps = n_steps;
    return c;
}

}  // namespace wb
