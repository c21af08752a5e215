// Host-side beam search with the reference's exact semantics (src/beam.rs:1-110).
//
// Generic over the token type T and the `next` / `is_finished` callables like the Rust original;
// the decode loop of src/transcribe.rs:232-309 instantiates it with BeamSearchToken.  Tie-breaks
// that the reference inherits from its data structures are kept on purpose:
//   * get_top_elements (beam.rs:81-110): ascending insertion list, a candidate equal to the minimum
//     of a full list is inserted in front and evicted at once  ->  on exact ties the EARLIER
//     element wins; k = 1 is a first-index arg-max.  Output order: ascending score.
//   * beam_search (beam.rs:9-37): Rust Iterator::max_by returns the LAST maximum.  beam_search_final returns the carried list
//     it picks from (the n-best list, ranked by rank_final / beamfx::rank_final).
//   * beam_search_step (beam.rs:39-79): `next` sees every beam, finished ones included; up to
//     2*beam_size beams are carried (k live + k finished).
#pragma once

#include <cstddef>
#include <functional>
#include <utility>
#include <vector>

#include "beam_fixed.hpp"

namespace wb {
namespace beam {

template <typename T>
struct BeamNode {   // beam.rs:3-7
    std::vector<T> seq;
    double log_prob = 0.0;
};

// beam.rs:81-110 -- returns indices into `elems` in the reference's output order
template <typename E, typename ScoreFn>
std::vector<size_t> get_top_elements(const std::vector<E>& elems, ScoreFn score, size_t num) {
    std::vector<size_t> top;
    std::vector<double> scores;
    top.reserve(num + 1);
    scores.reserve(num + 1);
    for (size_t e = 0; e < elems.size(); ++e) {
        const double s = score(elems[e]);
        if (top.size() == num) {                 // "most common scenario"
            if (num == 0 || s < scores[0]) continue;
        }
        size_t idx = scores.size();
        for (size_t i = 0; i < scores.size(); ++i) {
            if (scores[i] >= s) { idx = i; break; }
        }
        top.insert(top.begin() + idx, e);
        scores.insert(scores.begin() + idx, s);
        if (top.size() > num) {
            top.erase(top.begin());
            scores.erase(scores.begin());
        }
    }
    return top;
}

// Iterator::max_by(partial_cmp): last maximum; -1 if empty
template <typename T>
int max_by_last(const std::vector<BeamNode<T>>& beams) {
    int best = -1;
    for (size_t i = 0; i < beams.size(); ++i) {
        if (best < 0 || !(beams[i].log_prob < beams[(size_t)best].log_prob)) best = (int)i;
    }
    return best;
}

// beam.rs:39-79.  next(beams) -> per beam a list of (token, cumulative log-prob) continuations.
template <typename T, typename NextFn, typename FinFn>
std::vector<BeamNode<T>> beam_search_step(const std::vector<BeamNode<T>>& beams, NextFn&& next, FinFn&& is_finished,
                                          size_t beam_size) {
    std::vector<BeamNode<T>> finished_beams, new_beams;
    const std::vector<std::vector<std::pair<T, double>>> continuations = next(beams);
    for (size_t b = 0; b < beams.size(); ++b) {
        if (is_finished(beams[b].seq)) {
            finished_beams.push_back(beams[b]);
        } else {
            const auto& conts = continuations[b];
            for (size_t i : get_top_elements(conts, [](const std::pair<T, double>& c) { return c.second; }, beam_size)) {
                BeamNode<T> nb;
                nb.seq = beams[b].seq;
                nb.seq.push_back(conts[i].first);
                nb.log_prob = conts[i].second;
                new_beams.push_back(std::move(nb));
            }
        }
    }
    std::vector<BeamNode<T>> out;
    auto score = [](const BeamNode<T>& n) { return n.log_prob; };
    for (size_t i : get_top_elements(new_beams, score, beam_size)) out.push_back(new_beams[i]);
    for (size_t i : get_top_elements(finished_beams, score, beam_size)) out.push_back(finished_beams[i]);
    return out;
}

// beam.rs:9-32: the carried list when the search stops (`beams` at beam.rs:33), in carried order
template <typename T, typename NextFn, typename FinFn>
std::vector<BeamNode<T>> beam_search_final(std::vector<BeamNode<T>> beams, NextFn&& next, FinFn&& is_finished, size_t beam_size,
                                           size_t max_depth) {
    for (size_t i = 0; i < max_depth; ++i) {
        const int best = max_by_last(beams);
        if (best >= 0 && is_finished(beams[(size_t)best].seq)) break;
        beams = beam_search_step(beams, next, is_finished, beam_size);
    }
    return beams;
}

// beam.rs:9-37
template <typename T, typename NextFn, typename FinFn>
std::vector<T> beam_search(std::vector<BeamNode<T>> beams, NextFn&& next, FinFn&& is_finished, size_t beam_size,
                           size_t max_depth) {
    beams = beam_search_final(std::move(beams), next, is_finished, beam_size, max_depth);
    const int best = max_by_last(beams);
    return best >= 0 ? beams[(size_t)best].seq : std::vector<T>();
}

// the n-best order of a final carried list (beamfx::rank_final): indices into `beams`, best first
template <typename T>
std::vector<int> rank_final(const std::vector<BeamNode<T>>& beams) {
    std::vector<double> lp(beams.size());
    for (size_t i = 0; i < beams.size(); ++i) lp[i] = beams[i].log_prob;
    std::vector<int> order(beams.size());
    beamfx::rank_final(lp.data(), (int)lp.size(), order.data());
    return order;
}

}  // namespace beam
}  // namespace wb
