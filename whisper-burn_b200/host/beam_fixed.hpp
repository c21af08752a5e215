// One step of the reference's beam search (src/beam.rs:39-79, src/transcribe.rs:232-309) over fixed-capacity arrays, callable
// from host and device code.  decoder6.cu's beam mode runs it on the GPU, one warp per window; wb_beam_search_table_fixed runs
// it on the CPU.  It makes the same choices as host/beam.hpp + transcribe_windows (transcribe.cu), which stay the restatement
// the tests compare against:
//   * the continuations of a live beam are its (at most beam_size) candidates in ascending token id, as the reference
//     enumerates the vocabulary; score = parent log-prob + (double) candidate log-prob;
//   * get_top_elements: on exact ties the EARLIER element wins, output in ascending score;
//   * carried list = top beam_size of the continuations, then top beam_size of the beams that were already finished;
//   * max_by_last: the LAST maximum.  A beam is finished when its last token is eot; its continuations are discarded.
// Token sequences are not touched here: a Pick says which input node a carried node extends and by which token, and the caller
// copies sequences (the device does it warp-parallel).
#pragma once

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
}  // namespace wb
