"""Token alignment without a GPU: the float64 / float32 restatement of openai-whisper's find_alignment (tests/oracle_align.py)
against independent computations and hand-worked DTW cases, openai's head-mask format, the no-GPU error of wb_align_dtw, and
the MARGIN check that makes test_align_gpu.py able to fail: each mistake an implementation could make moves the oracle matrix
of the GPU tests' models by at least MARGIN times the fp32 K/V tolerance oracle_align.MATRIX_TOL["f32"].  The kernels after
the key load are the same for both K/V types; with the fp16 K/V tolerance (47 times larger, fp16 rounding flips) only the
softmax crop, the filter and the normalisation rows are claimed."""
import base64
import gzip

import numpy as np
import pytest
import scipy.ndimage
import torch

import harness as h
import oracle_align as oa
from oracle import model as o_model
from whisper_burn_b200 import ffi, transcribe
from whisper_burn_b200.synth import WhisperDims


# ---------------------------------------------------------------- median filter
@pytest.mark.parametrize("C", [4, 5, 7, 8, 59, 750])
def test_median_filter_is_scipy_mirror(C):
    x = np.random.default_rng(C).standard_normal((5, 9, C))
    want = scipy.ndimage.median_filter(x, size=(1, 1, 7), mode="mirror")
    assert np.array_equal(oa.median_filter(x), want)
    if C > 4:   # scipy's own "reflect" repeats the edge: a different filter
        assert not np.array_equal(scipy.ndimage.median_filter(x, size=(1, 1, 7), mode="reflect"), want)


@pytest.mark.parametrize("C", [1, 2, 3])
def test_median_filter_passes_short_rows_through(C):
    x = np.random.default_rng(C).standard_normal((3, 4, C))
    assert np.array_equal(oa.median_filter(x), x)


# ---------------------------------------------------------------- DTW
def dp_optimum(x):
    """the float64 minimum path cost by a plain DP (diagonal, up and left steps from (0, 0) to (N-1, C-1))"""
    N, C = x.shape
    D = np.full((N + 1, C + 1), np.inf)
    D[0, 0] = 0.0
    for i in range(1, N + 1):
        for j in range(1, C + 1):
            D[i, j] = x[i - 1, j - 1] + min(D[i - 1, j - 1], D[i - 1, j], D[i, j - 1])
    return D[N, C]


HAND = [
    # all equal: every interior tie goes left, so the path climbs column 0 and crosses the last row
    (np.zeros((3, 4)), [0, 0, 0], [0, 0, 4]),
    # a diagonal of ones: ties between equal costs still go left, so the path steps up before it steps right
    (np.eye(3), [0, 0, 1], [0, 1, 3]),
    # one row: the whole row
    (np.array([[0.1, 0.5, 0.2, 0.9, 0.3]]), [0], [5]),
    # one column: every row starts at column 0
    (np.array([[0.3], [0.1], [0.7], [0.2]]), [0, 0, 0, 0], [0, 0, 0, 1]),
    # N > C: rows 0-1 prefer column 0 and rows 2-4 column 1; the tie at cell (3, 2) (three costs of -10) goes left, so row 2
    # still starts in column 0 and the path steps right inside it
    (np.array([[5, 0], [5, 0], [0, 5], [0, 5], [0, 5]], dtype=np.float64), [0, 0, 0, 1, 1], [0, 0, 1, 1, 2]),
]


@pytest.mark.parametrize("case", range(len(HAND)))
def test_dtw_hand_worked(case):
    m, start, end = HAND[case]
    s, e = oa.times(np.asarray(m, dtype=np.float32))
    assert s.tolist() == start and e.tolist() == end, (s, e)


def tie_heavy(rng, N, C, kind):
    if kind == "equal":
        return np.full((N, C), 0.25, dtype=np.float32)
    if kind == "int":
        return rng.integers(-2, 3, size=(N, C)).astype(np.float32)
    return rng.standard_normal((N, C)).astype(np.float32)


@pytest.mark.parametrize("kind", ["equal", "int", "normal"])
def test_dtw_forms_agree_and_reach_the_optimum(kind):
    rng = np.random.default_rng(len(kind))
    for N, C in [(1, 1), (1, 7), (6, 1), (5, 3), (9, 9), (12, 5), (17, 40)]:
        m = tie_heavy(rng, N, C, kind)
        x = -m.astype(np.float64)
        c1, t1 = oa.dtw_loops(x)
        c2, t2 = oa.dtw(x)
        assert np.array_equal(c1, c2) and np.array_equal(t1, t2), (N, C)
        text, time = oa.backtrace(t2)
        assert text[0] == 0 and time[0] == 0 and text[-1] == N - 1 and time[-1] == C - 1
        assert np.all(np.diff(text) >= 0) and np.all(np.diff(time) >= 0) and np.all(np.diff(text) + np.diff(time) >= 1)
        # the path costs what the rule's own DP says; that is the optimum unless ties decided (a tie of the two cheapest
        # predecessors goes to the third), which random normal matrices do not have
        opt = dp_optimum(x)
        got = oa.path_cost(x, text, time)
        assert abs(got - float(c2[N, C])) <= 1e-5 * max(1.0, abs(got)), (N, C, got, c2[N, C])
        if kind == "normal":
            assert abs(got - opt) < 1e-4 * max(1.0, abs(opt)), (N, C, got, opt)
        else:
            assert got >= opt, (N, C, got, opt)
        start, end = oa.times(m)
        assert len(start) == N and end[-1] == C and np.all(start[1:] == end[:-1])


# ---------------------------------------------------------------- openai's head masks
def test_alignment_heads_round_trip():
    dims = WhisperDims(80, 1500, 768, 12, 12, 51864, 448, 768, 12, 12)
    rng = np.random.default_rng(3)
    mask = rng.random((12, 12)) < 0.1
    b85 = base64.b85encode(gzip.compress(mask.tobytes())).decode()
    pairs = transcribe.alignment_heads_from_openai(b85, dims)
    assert pairs == sorted((int(l), int(hd)) for l, hd in zip(*np.nonzero(mask)))
    back = np.zeros((12, 12), dtype=bool)
    for l, hd in pairs:
        back[l, hd] = True
    assert np.array_equal(back, mask)
    with pytest.raises(ValueError):
        transcribe.alignment_heads_from_openai(b85, WhisperDims(80, 1500, 384, 6, 4, 51864, 448, 384, 6, 4))


# ---------------------------------------------------------------- the entry points without a GPU
def test_align_dtw_argument_errors_come_before_the_device():
    lib = ffi.lib()
    s = np.zeros(449, dtype=np.int32)
    e = np.zeros(449, dtype=np.int32)
    m = np.zeros((449, 4), dtype=np.float32)
    call = lambda n, c, mp=ffi.fptr(m): lib.wb_align_dtw(0, mp, n, c, ffi.i32ptr(s), ffi.i32ptr(e))
    assert call(0, 4) == ffi.WB_ERR_INVALID_ARG
    assert call(449, 4) == ffi.WB_ERR_INVALID_ARG
    assert call(4, 0) == ffi.WB_ERR_INVALID_ARG
    assert call(448, 10 ** 6) == ffi.WB_ERR_INVALID_ARG      # the trace exceeds shared memory
    assert call(4, 4, None) == ffi.WB_ERR_INVALID_ARG
    assert lib.wb_session_align_tokens(None, 1, None, None, None, None, 0, None, None, None, None, 0) == ffi.WB_ERR_INVALID_ARG


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU error path")
def test_align_dtw_fails_loudly_without_gpu():
    with pytest.raises(ffi.WbError) as e:
        transcribe.align_dtw(np.zeros((3, 5), np.float32))
    assert e.value.code == ffi.WB_ERR_CUDA and "no CPU fallback" in e.value.msg


# ---------------------------------------------------------------- MARGIN: the GPU checks can fail
def margin_case(n_text_layer, kv):
    dims, _, _, w64 = h.shallow_weights(384, 6, 2051, n_text_layer, True)
    xa = o_model.forward_encoder(w64, dims, h.window_mel(dims))
    C = oa.window_columns(h.N_OF_T[65] // 160)
    ids = [int(t) for t in np.random.default_rng(11).integers(0, 2051, size=40)]
    return dims, w64, xa, C, ids


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_mistakes_move_the_matrix(kv):
    dims, w64, xa, C, ids = margin_case(2, kv)
    first = 4
    qk = oa.cross_qk(w64, dims, ids, xa, kv)
    heads = oa.default_heads(dims)
    base = oa.alignment_matrix(qk, heads, C, first)
    move = lambda m: float(np.abs(m - base).max())
    moved = {
        "softmax before the crop": move(oa.alignment_matrix(qk, heads, C, first, softmax_first=True)),
        "unbiased std": move(oa.alignment_matrix(qk, heads, C, first, ddof=1)),
        "median width 5": move(oa.alignment_matrix(qk, heads, C, first, width=5)),
        "scipy reflect padding": move(oa.alignment_matrix(qk, heads, C, first, pad="symmetric")),
        "normalisation over the kept rows": move(oa.alignment_matrix(qk, heads, C, first, kept_rows_stats=True)),
        "keys without the f16 rounding" if kv == "f16" else "keys with an f16 rounding":
            move(oa.alignment_matrix(oa.cross_qk(w64, dims, ids, xa, "f32" if kv == "f16" else "f16"), heads, C, first)),
    }
    h.check_moves(moved, oa.MATRIX_TOL["f32"], f"alignment matrix d=384 kv={kv}", "align")
    coarse = ("softmax before the crop", "median width 5", "scipy reflect padding", "normalisation over the kept rows")
    h.check_moves({k: moved[k] for k in coarse}, oa.MATRIX_TOL["f16"], f"alignment matrix d=384 kv={kv}, fp16 tolerance", "align")


def test_default_heads_layer_moves_the_matrix():
    """(L + 1) // 2 differs from L // 2 only at an odd layer count: the 3-layer decoder that
    test_align_gpu.py::test_odd_layer_count_default_heads_vs_float64 aligns with the default heads"""
    dims, w64, xa, C, ids = margin_case(3, "f32")
    qk = oa.cross_qk(w64, dims, ids, xa, "f32")
    base = oa.alignment_matrix(qk, oa.default_heads(dims), C, 4)
    wrong = [(l, hd) for l in range((dims.n_text_layer + 1) // 2, dims.n_text_layer) for hd in range(dims.n_text_head)]
    h.check_moves({"default heads from (L + 1) / 2": float(np.abs(oa.alignment_matrix(qk, wrong, C, 4) - base).max())},
                  max(oa.MATRIX_TOL.values()), "alignment matrix default heads, 3 layers", "align")
