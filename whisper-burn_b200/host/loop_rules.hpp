// Stopping rules of the reference's greedy loop (transcribe.rs:314-380), callable from host and device code.  Every persistent
// decoder applies them in its row finish (dec_common.cuh loop_finish) when a session decodes with WB_SEARCH_GREEDY_LOOP; the
// host build is checked against host/repeat.hpp, which stays the restatement of the reference's helpers.
//   * EOT test (:334-356): stop when exp(eot_logit - token_logit) > 0.5, in f64 on the two f32 logits;
//   * repetition cut (:358-377): find_repeated_tokens_index(tokens, 5, 4) over the whole sequence, prompt included; on a hit
//     the sequence is cut to `end` (the index of the SECOND window equal to the last one) and EOT follows.
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define WB_HD __host__ __device__
#else
#define WB_HD
#endif

namespace wb {
namespace loop {

constexpr int REPEAT_WINDOW = 5;   // transcribe.rs:358
constexpr int MIN_REPEATS = 4;     // transcribe.rs:359

WB_HD inline bool eot_stop(float eot_logit, float token_logit) {
    return exp((double)eot_logit - (double)token_logit) > 0.5;
}

// Whether the window of REPEAT_WINDOW tokens at i equals the last window of tokens[0, n); tok(j) returns token j.
template <class Tok>
WB_HD inline bool window_repeats(const Tok& tok, int n, int i) {
    const int last = n - REPEAT_WINDOW;
    for (int k = 0; k < REPEAT_WINDOW; ++k)
        if (tok(i + k) != tok(last + k)) return false;
    return true;
}

WB_HD inline int popc32(unsigned int m) {
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}
WB_HD inline int ctz32(unsigned int m) {   // m != 0
#if defined(__CUDA_ARCH__)
    return __ffs((int)m) - 1;
#else
    return __builtin_ctz(m);
#endif
}

// The repetition cut over tokens[0, n): `end` of find_repeated_tokens_index(tokens, REPEAT_WINDOW, MIN_REPEATS), or -1 for
// None.  The candidate windows i = 0 .. n - 2 * REPEAT_WINDOW are examined 32 at a time: ballot(base) returns a mask whose
// bit l says that window base + l repeats the last window (window_repeats; bits of i past the last candidate clear).  On the
// device a warp forms that mask with one __ballot_sync, lane l taking window base + l; on the host a loop does.  The scan
// stops once MIN_REPEATS repeats are found: the first two are then known, and later ones change nothing.
template <class Ballot>
WB_HD inline int repeat_cut(int n, const Ballot& ballot) {
    if (2 * REPEAT_WINDOW > n) return -1;
    const int n_cand = n - 2 * REPEAT_WINDOW + 1;
    int count = 0, first = -1, second = -1;
    for (int base = 0; base < n_cand; base += 32) {
        unsigned int m = ballot(base);
        count += popc32(m);
        while (m != 0u && second < 0) {
            const int i = base + ctz32(m);
            if (first < 0) first = i;
            else second = i;
            m &= m - 1u;
        }
        if (count >= MIN_REPEATS) return second;   // MIN_REPEATS >= 2: `second` is set
    }
    return -1;
}

// Host form of the same rule over an array (what the device computes with one warp)
template <class T>
inline int repeat_cut_host(const T* tokens, int n) {
    auto tok = [tokens](int j) { return tokens[j]; };
    return repeat_cut(n, [&](int base) {
        unsigned int m = 0u;
        for (int l = 0; l < 32; ++l)
            if (base + l + 2 * REPEAT_WINDOW <= n && window_repeats(tok, n, base + l)) m |= 1u << l;
        return m;
    });
}

}  // namespace loop
}  // namespace wb
