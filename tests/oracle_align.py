"""Float64 restatement of token alignment (wb_session_align_tokens): openai-whisper's find_alignment (whisper/timing.py) on this
project's rows, from oracle/ alone, and a float32 restatement of its dtw_cpu and backtrace.

  cross_qk         the decoder's per-layer scaled cross q . k of every position (oracle.model's functions; fp16-rounded scaled
                   keys with kv="f16", as oracle.model.qkv_attention rounds them)
  alignment_matrix steps 2-5 of the header: crop to C columns, softmax, per-column normalisation over all L positions (biased
                   std, 0 where it is 0), width-7 median with torch reflect padding (none when C <= 3), mean over the heads in
                   ascending order, rows first - 1 .. L - 2.  Keyword options restate the mistakes the MARGIN check measures.
  dtw / dtw_loops  dtw_cpu's cost in float32 over float64 inputs (the anti-diagonal form and openai's own loop order)
  times            the backtrace and the jump times: start / end per row"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import model as o_model


# The GPU matrix against alignment_matrix, absolute (the matrix is a mean of z-scores, O(1)), on the GPU's own encoder output.
# Worst measured on one H100 80GB HBM3 (700 W power limit): f32 4.9e-5 (d = 1280), 3x margin; f16 2.3e-3 (d = 1280), 3x
# margin.  The fp16 figure is larger because a float64 key can round to the fp16 neighbour of the one the GPU's float32 key
# rounds to, and a z-score divides that by a column's spread.
MATRIX_TOL = {"f32": 1.5e-4, "f16": 7e-3}


def default_heads(dims):
    """openai's fallback: every head of decoder layers n_text_layer // 2 .."""
    return [(l, h) for l in range(dims.n_text_layer // 2, dims.n_text_layer) for h in range(dims.n_text_head)]


def cross_qk(w, dims, ids, xa, kv="f32", last_layer=None):
    """{layer: [H, L, T] float64} of the scaled cross q . k at every position of ids (one sequence) on xa [1, T, d], for layers
    0 .. last_layer (default all)."""
    opts = o_model.OracleOptions(kv_dtype=kv)
    H, d = dims.n_text_head, dims.n_text_state
    scale = o_model._f32((d / H) ** -0.25)
    toks = torch.tensor([ids], dtype=torch.int64)
    n = toks.shape[1]
    x = F.embedding(toks, w["decoder/token_embedding/weight"]) + w["decoder/positional_embedding"][0:n].unsqueeze(0)
    mask = o_model.attn_decoder_mask(dims.n_text_ctx, x.dtype)
    out = {}
    last = dims.n_text_layer - 1 if last_layer is None else last_layer
    for i in range(last + 1):
        p = f"decoder/block_{i}"
        x = x + o_model.self_attention(o_model.layer_norm(x, w, p + "/attn_ln", opts), w, p + "/attn", mask, H, opts)
        hc = o_model.layer_norm(x, w, p + "/cross_attn_ln", opts)
        q = o_model.linear(hc, w, p + "/cross_attn/query").reshape(1, n, H, d // H).transpose(1, 2) * scale
        k = o_model.linear(xa, w, p + "/cross_attn/key")
        k = k.reshape(1, k.shape[1], H, d // H).transpose(1, 2) * scale
        if kv == "f16":
            k = k.to(torch.float16).to(k.dtype)
        out[i] = torch.matmul(q, k.transpose(2, 3))[0].double().numpy()
        x = x + o_model.cross_attention(hc, xa, w, p + "/cross_attn", H, opts)
        x = x + o_model.mlp(o_model.layer_norm(x, w, p + "/mlp_ln", opts), w, p + "/mlp")
    return out


def softmax(x):
    e = np.exp(x - x.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def median_filter(x, width=7, pad="reflect"):
    """openai's median_filter along the last axis: torch reflect padding (numpy "reflect", scipy "mirror"); unchanged when the
    axis is not longer than width // 2.  pad="symmetric" is scipy's "reflect" (the edge repeated)."""
    half = width // 2
    if x.shape[-1] <= half:
        return x
    xp = np.pad(x, [(0, 0)] * (x.ndim - 1) + [(half, half)], mode=pad)
    win = np.lib.stride_tricks.sliding_window_view(xp, width, axis=-1)
    return np.sort(win, axis=-1)[..., half]


def alignment_matrix(qk, heads, C, first, softmax_first=False, ddof=0, width=7, pad="reflect", kept_rows_stats=False):
    """The float64 matrix [L - first, C] from cross_qk's result; the options restate the mistakes an implementation could make."""
    acc = None
    for l, h in sorted(heads):
        s = qk[l][h]
        L = s.shape[0]
        p = softmax(s)[:, :C] if softmax_first else softmax(s[:, :C])
        base = p[first - 1:L - 1] if kept_rows_stats else p
        mean, std = base.mean(axis=0), base.std(axis=0, ddof=ddof)
        z = np.where(std == 0, 0.0, (p - mean) / np.where(std == 0, 1.0, std))
        z = median_filter(z, width, pad)
        acc = z if acc is None else acc + z
    m = acc / len(heads)
    return m[first - 1:m.shape[0] - 1]


def window_columns(n_frames):
    """C = max(1, F // 2) (openai's num_frames // 2)"""
    return max(1, n_frames // 2)


# ---------------------------------------------------------------- DTW (float32 cost, as dtw_cpu)
def _pick(c0, c1, c2):
    if c0 < c1 and c0 < c2:
        return c0, 0
    if c1 < c0 and c1 < c2:
        return c1, 1
    return c2, 2


def dtw_loops(x):
    """openai's dtw_cpu loop order on x (float64 [N, M]) -> (cost float32, trace)"""
    x = np.asarray(x, dtype=np.float64)
    N, M = x.shape
    cost = np.full((N + 1, M + 1), np.inf, dtype=np.float32)
    trace = -np.ones((N + 1, M + 1), dtype=np.float32)
    cost[0, 0] = 0
    for j in range(1, M + 1):
        for i in range(1, N + 1):
            c, t = _pick(cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1])
            cost[i, j] = x[i - 1, j - 1] + c
            trace[i, j] = t
    return cost, trace


def dtw(x):
    """the same cost and trace, one anti-diagonal at a time (each cell reads only the two diagonals before it)"""
    x = np.asarray(x, dtype=np.float64)
    N, M = x.shape
    cost = np.full((N + 1, M + 1), np.inf, dtype=np.float32)
    trace = -np.ones((N + 1, M + 1), dtype=np.float32)
    cost[0, 0] = 0
    for s in range(2, N + M + 1):
        i = np.arange(max(1, s - M), min(N, s - 1) + 1)
        j = s - i
        c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
        diag = (c0 < c1) & (c0 < c2)
        up = ~diag & (c1 < c0) & (c1 < c2)
        t = np.where(diag, 0, np.where(up, 1, 2))
        c = np.where(diag, c0, np.where(up, c1, c2))
        cost[i, j] = (x[i - 1, j - 1] + c.astype(np.float64)).astype(np.float32)
        trace[i, j] = t
    return cost, trace


def backtrace(trace):
    """openai's backtrace -> (text_indices, time_indices)"""
    trace = trace.copy()
    i, j = trace.shape[0] - 1, trace.shape[1] - 1
    trace[0, :] = 2
    trace[:, 0] = 1
    result = []
    while i > 0 or j > 0:
        result.append((i - 1, j - 1))
        if trace[i, j] == 0:
            i -= 1
            j -= 1
        elif trace[i, j] == 1:
            i -= 1
        elif trace[i, j] == 2:
            j -= 1
        else:
            raise ValueError("Unexpected trace[i, j]")
    return np.array(result)[::-1, :].T


def times(matrix):
    """(start, end) int32 per row of DTW on -matrix (float32 matrix [N, C]): find_alignment's jump times in encoder positions"""
    N, C = matrix.shape
    _, trace = dtw(-np.asarray(matrix, dtype=np.float32).astype(np.float64))
    text, time = backtrace(trace)
    jumps = np.pad(np.diff(text), (1, 0), constant_values=1).astype(bool)
    start = time[jumps].astype(np.int32)
    assert len(start) == N, f"{len(start)} jumps for {N} rows"
    return start, np.append(start[1:], C).astype(np.int32)


def path_cost(x, text, time):
    return float(np.asarray(x, dtype=np.float64)[text, time].sum())
