// The dynamic time warping of token alignment (openai-whisper whisper/timing.py: dtw_cpu, backtrace and the jump times of
// find_alignment), callable from host and device code: align.cu's DTW kernel runs the cell rule over anti-diagonals and the
// backtrace in one thread; the restatement the tests compare against is tests/oracle_align.py.
//
// On x [N][C] (the negated alignment matrix), cost [N + 1][C + 1] in f32 with cost[0][0] = 0 and inf elsewhere on the border:
//   cost[i][j] = x[i-1][j-1] + c,  c = the cost of the predecessor the rule picks among
//   c0 = cost[i-1][j-1] (diagonal, trace 0), c1 = cost[i-1][j] (up, trace 1), c2 = cost[i][j-1] (left, trace 2):
//   diagonal if c0 < c1 && c0 < c2, else up if c1 < c0 && c1 < c2, else left.
// The f32 add equals dtw_cpu's f64 add rounded to its f32 cost array (the f64 sum of two f32 values rounds once more to the
// same f32).  The backtrace walks from (N, C) to (0, 0) with row 0 read as left and column 0 as up; start[k] is the column
// (j - 1) where the path first enters row k + 1, end[k] = start[k + 1] and end[N - 1] = C.
#pragma once

#ifndef WB_HD
#if defined(__CUDACC__)
#define WB_HD __host__ __device__
#else
#define WB_HD
#endif
#endif

namespace wb {
namespace dtw {

enum : int { DIAG = 0, UP = 1, LEFT = 2 };

// the cell rule: returns the trace code, c receives the picked predecessor's cost
WB_HD inline int pick(float c0, float c1, float c2, float& c) {
    if (c0 < c1 && c0 < c2) { c = c0; return DIAG; }
    if (c1 < c0 && c1 < c2) { c = c1; return UP; }
    c = c2;
    return LEFT;
}

// trace(i, j) for 1 <= i <= N, 1 <= j <= C -> the code of that cell; writes start[0 .. N) and end[0 .. N)
template <typename Trace>
WB_HD inline void backtrace(int N, int C, Trace&& trace, int* start, int* end) {
    int i = N, j = C;
    while (i > 0 || j > 0) {
        if (i > 0) start[i - 1] = j - 1;   // the last write of a row is the path's first cell in it
        const int t = i == 0 ? LEFT : j == 0 ? UP : trace(i, j);
        if (t == DIAG) { --i; --j; }
        else if (t == UP) --i;
        else --j;
    }
    for (int k = 0; k + 1 < N; ++k) end[k] = start[k + 1];
    end[N - 1] = C;
}

}  // namespace dtw
}  // namespace wb
