"""GPU tests (-m gpu) of token alignment (wb_session_align_tokens, Session.align_tokens, wb_align_dtw): openai-whisper's
find_alignment on this project's rows (tests/oracle_align.py).

  1. the matrix against float64 within oracle_align.MATRIX_TOL, and start / end bit-equal to the float32 DTW restatement run on
     the returned matrix: d = 384, 768, 1280, fp32 and fp16 K/V, reference windows T = 750, 6, 65, 64 and a native T = 1500,
     sequence lengths 2, 63-65, 127-129 and 448, default heads, one head and all heads; tiny.en and small.en at their layer
     counts; a 3-layer decoder (default heads from layer 1); windows of C = 1 to 5 and 7 columns (the median filter's skip
     and its first reflect-padded width);
  2. wb_align_dtw bit-equal to the restatement on tie-heavy matrices up to 447 x 1500;
  3. bit-identical results alone, in a batch, split across groups, with heads in any order and on repeated calls;
  4. transcripts of every decode path align, and leave decode results untouched;
  5. every error code of the header contract."""
import numpy as np
import pytest
import torch

import harness as h
import oracle_align as oa
import wb200  # noqa: F401
from oracle import synth
from whisper_burn_b200 import ffi, model, transcribe

pytestmark = pytest.mark.gpu

LENS = (2, 63, 64, 65, 127, 128, 129, 448)


def frames_of(n_samples, n_audio_ctx, mode="reference"):
    """F: the kept mel frames of a waveform window"""
    limit = n_audio_ctx if mode == "reference" else 2 * n_audio_ctx
    return min(n_samples // 160, limit - 10)


def seqs_for(V, seed, lens=LENS):
    rng = np.random.default_rng(seed)
    seqs = [[int(t) for t in rng.integers(0, V, size=n)] for n in lens]
    return seqs, [1 if n == 2 else min(4, n - 1) for n in lens]


def check_against_oracle(sess, w64, dims, xa, Cs, seqs, wins, first, heads, kv, what):
    """align_tokens against the float64 matrix and the exact DTW of its own matrix; returns the worst matrix error"""
    out = sess.align_tokens(seqs, wins, first, heads=heads, return_matrix=True)
    sel = heads if heads is not None else oa.default_heads(dims)
    last = max(l for l, _ in sel)
    worst = 0.0
    for seq, w, f, (st, en, m) in zip(seqs, wins, first, out):
        C = Cs[w]
        assert m.shape == (len(seq) - f, C) and m.dtype == np.float32, f"{what}: matrix {m.shape}"
        want = oa.alignment_matrix(oa.cross_qk(w64, dims, seq, xa[w], kv, last), sel, C, f)
        err = float(np.abs(m - want).max())
        worst = max(worst, err)
        assert err < oa.MATRIX_TOL[kv], f"{what} len={len(seq)} C={C}: matrix error {err}"
        s2, e2 = oa.times(m)
        assert np.array_equal(st, s2) and np.array_equal(en, e2), f"{what} len={len(seq)}: DTW {st} {en} vs {s2} {e2}"
    return worst


# ---------------------------------------------------------------- 1. against float64
@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("d", [384, 768, 1280])
def test_matrix_vs_float64(d, kv):
    dims, wh, w64 = h.make_model(d, d // 64, 2051)
    Ts, waves = h.windows(4, seed=11 * d)
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    Cs = [oa.window_columns(frames_of(len(w), dims.n_audio_ctx)) for w in waves]
    seqs, first = seqs_for(dims.n_vocab, d)
    wins = [i % 4 for i in range(len(seqs))]
    H, L = dims.n_text_head, dims.n_text_layer
    worst = 0.0
    for heads in (None, [(0, H - 1)], [(l, hh) for l in range(L) for hh in range(H)]):
        worst = max(worst, check_against_oracle(sess, w64, dims, xa, Cs, seqs, wins, first, heads, kv, f"d={d} kv={kv} heads={heads}"))
    h.report(f"align matrix d={d} kv={kv} T={sorted(set(Ts))}", worst, oa.MATRIX_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_native_window_vs_float64(kv):
    dims, wh, w64 = h.make_model(384, 6, 2051)
    waves = [synth.waveform(480000, seed=3)]
    sess = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv), windows="native")
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, [1500])
    Cs = [oa.window_columns(frames_of(480000, dims.n_audio_ctx, "native"))]
    assert Cs == [1495]
    seqs, first = seqs_for(dims.n_vocab, 5, lens=(2, 65, 448))
    worst = check_against_oracle(sess, w64, dims, xa, Cs, seqs, [0] * 3, first, None, kv, f"native kv={kv}")
    h.report(f"align matrix native T=1500 kv={kv}", worst, oa.MATRIX_TOL[kv])


@pytest.mark.parametrize("name", ["tiny.en", "small.en"])
def test_real_layer_counts_vs_float64(name):
    dims, sp, wh, _, _, w64 = h.named_model(name, f64=True)
    waves = [synth.waveform(h.N_OF_T[T], seed=T) for T in (750, 65)]
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8)
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, [750, 65])
    Cs = [oa.window_columns(frames_of(len(w), dims.n_audio_ctx)) for w in waves]
    seqs, first = seqs_for(dims.n_vocab, 9, lens=(64, 129))
    worst = check_against_oracle(sess, w64, dims, xa, Cs, seqs, [0, 1], first, None, "f32", name)
    h.report(f"align matrix {name} ({dims.n_text_layer} layers)", worst, oa.MATRIX_TOL["f32"])


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_odd_layer_count_default_heads_vs_float64(kv):
    """3 text layers, the MARGIN model of test_align_cpu.py: the default heads start at layer 3 // 2 = 1, not (3 + 1) // 2 = 2"""
    dims, wh, w64 = h.make_model(384, 6, 2051, n_text_layer=3)
    Ts, waves = h.windows(2, seed=31, order=(65, 750))
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    Cs = [oa.window_columns(frames_of(len(w), dims.n_audio_ctx)) for w in waves]
    seqs, first = seqs_for(dims.n_vocab, 13, lens=(40, 129, 448))
    worst = check_against_oracle(sess, w64, dims, xa, Cs, seqs, [0, 1, 0], first, None, kv, f"3 layers kv={kv}")
    h.report(f"align matrix 3 text layers, default heads kv={kv}", worst, oa.MATRIX_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_filter_edges_vs_float64(kv):
    """C = 1, 2, 3 (no median filter), 4 (the first C with reflect padding), 5 and 7: windows of 400 to 2240 samples"""
    dims, wh, w64 = h.make_model(384, 6, 2051)
    n = [400, 700, 1000, 1300, 1600, 2240]
    waves = [synth.waveform(m, seed=40 + i) for i, m in enumerate(n)]
    Cs = [oa.window_columns(frames_of(m, dims.n_audio_ctx)) for m in n]
    assert Cs == [1, 2, 3, 4, 5, 7]
    Ts = [(m // 160 + 10 - 1) // 2 + 1 for m in n]
    sess = transcribe.Session(wh, max_windows=len(n), max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    seqs, first = seqs_for(dims.n_vocab, 17, lens=(2, 9, 65, 129, 64, 448))
    worst = 0.0
    for heads in (None, [(0, 3)]):
        worst = max(worst, check_against_oracle(sess, w64, dims, xa, Cs, seqs, list(range(len(n))), first, heads, kv,
                                                f"C=1..7 kv={kv} heads={heads}"))
    h.report(f"align matrix C = 1, 2, 3, 4, 5, 7 kv={kv}", worst, oa.MATRIX_TOL[kv])


# ---------------------------------------------------------------- 2. the DTW kernel alone
@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (7, 1), (3, 4), (30, 17), (200, 64), (447, 1500)])
def test_align_dtw_exact(shape):
    N, C = shape
    rng = np.random.default_rng(N * 7 + C)
    for kind in ("equal", "int", "normal", "coarse"):
        if kind == "equal":
            m = np.full((N, C), 0.5, np.float32)
        elif kind == "int":
            m = rng.integers(-2, 3, size=(N, C)).astype(np.float32)
        elif kind == "coarse":   # a diagonal band of exact ties
            m = np.round(rng.standard_normal((N, C)) * 2) / 4 - np.abs(np.arange(N)[:, None] * C / N - np.arange(C)[None, :]) / 8
            m = m.astype(np.float32)
        else:
            m = rng.standard_normal((N, C)).astype(np.float32)
        st, en = transcribe.align_dtw(m)
        s2, e2 = oa.times(m)
        assert np.array_equal(st, s2) and np.array_equal(en, e2), f"{shape} {kind}"


# ---------------------------------------------------------------- 3. invariance
@pytest.fixture(scope="module")
def small():
    dims, wh, w64 = h.make_model(384, 6, 2051)
    Ts, waves = h.windows(2, seed=23)
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8)
    sess.encode_waveforms(waves)
    return dims, wh, sess, waves


def same(a, b):
    return all(np.array_equal(x, y) for p, q in zip(a, b) for x, y in zip(p, q)) and len(a) == len(b)


def test_alone_batched_split_reordered_repeated(small):
    dims, _, sess, _ = small
    rng = np.random.default_rng(4)
    long = [int(t) for t in rng.integers(0, dims.n_vocab, size=448)]
    heads = [(1, 2), (0, 5), (1, 0)]
    alone = sess.align_tokens([long], [0], [4], heads=heads, return_matrix=True)[0]
    others, _ = seqs_for(dims.n_vocab, 8, lens=(65, 300, 3))
    batch = sess.align_tokens([others[0], long, others[1], others[2]], [1, 0, 0, 1], [4, 4, 4, 1], heads=heads, return_matrix=True)
    assert same([batch[1]], [alone])
    # 9 x 448 + 65 = 4097 rows: two groups of whole sequences
    split = sess.align_tokens([long] * 9 + [others[0]], [0] * 9 + [1], [4] * 10, heads=heads, return_matrix=True)
    assert same([split[0]], [alone]) and same([split[8]], [alone]) and same([split[9]], [batch[0]])
    for perm in ([(1, 0), (0, 5), (1, 2)], [(0, 5), (1, 0), (1, 2)]):
        assert same([sess.align_tokens([long], [0], [4], heads=perm, return_matrix=True)[0]], [alone])
    assert same([sess.align_tokens([long], [0], [4], heads=heads, return_matrix=True)[0]], [alone])
    st, en = sess.align_tokens([long], [0], [4], heads=heads)[0]
    assert np.array_equal(st, alone[0]) and np.array_equal(en, alone[1])


# ---------------------------------------------------------------- 4. transcripts of every decode path
def check_rows_align(sess, w64, dims, ids, first, kv="f32"):
    xa = [torch.from_numpy(sess.get_encoder_output(r)).double()[None] for r in range(len(ids))]
    Cs = [oa.window_columns(sess.get_mel(r).shape[1] - 10) for r in range(len(ids))]   # the kept frames: Tm - 10 zero frames
    keep = [r for r, t in enumerate(ids) if len(t) > first[r]]
    return check_against_oracle(sess, w64, dims, xa, Cs, [ids[r] for r in keep], keep, [first[r] for r in keep], None, kv,
                                "decoded rows") if keep else 0.0


def state_of(sess, n, nbest):
    lps = [sess.last_logprobs(r) for r in range(n)]
    nb = [sess.last_nbest(r) for r in range(n)] if nbest else None
    try:
        topk = sess.last_topk(n, 1)
    except ffi.WbError:   # a beam search's last launch kept more candidates per row
        topk = None
    return lps, nb, topk, sess.last_decoder()


def same_state(a, b):
    assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a[0], b[0]))
    if a[1] is not None:
        for x, y in zip(a[1], b[1]):
            for p, q in zip(x, y):
                assert p[0] == q[0] and np.array_equal(p[1], q[1]) and p[2] == q[2] and p[3] == q[3]
    if a[2] is not None:
        assert np.array_equal(a[2][0], b[2][0]) and np.array_equal(a[2][1], b[2][1])
    assert a[3] == b[3]


def test_decoded_transcripts_align(monkeypatch):
    dims, sp, wh, _, _, w64 = h.named_model("tiny.en", f64=True)
    waves = h.pool_waves(h.golden("tokens_beam"), 3)
    spec = h.is_special_of(sp)
    worst = 0.0
    cases = []
    sess = transcribe.Session(wh, max_windows=3, max_beams=5, max_text_len=40)
    cases.append((sess, sess.transcribe_windows(waves, sp, spec, beam_size=5, max_depth=30), True))   # device beam search
    assert sess.last_decoder() == 6
    h.use_decoder(monkeypatch, 3)
    host = transcribe.Session(wh, max_windows=3, max_beams=5, max_text_len=40)
    h.use_decoder(monkeypatch, 0)
    cases.append((host, host.transcribe_windows(waves, sp, spec, beam_size=5, max_depth=30), True))   # host beam search
    g1 = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=40)
    cases.append((g1, g1.transcribe_windows(waves, sp, spec, beam_size=1, max_depth=30), True))
    loop = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=40, search="greedy_loop")
    cases.append((loop, [t[:40] for t in loop.transcribe_windows(waves, sp, None, beam_size=1, max_depth=30)], False))
    for s, ids, nbest in cases:
        before = state_of(s, len(ids), nbest)
        worst = max(worst, check_rows_align(s, w64, dims, ids, [4] * len(ids)))
        if nbest:
            rank1 = [s.last_nbest(r)[0][0] for r in range(len(ids))]
            assert rank1 == ids
            worst = max(worst, check_rows_align(s, w64, dims, rank1, [4] * len(ids)))
        same_state(before, state_of(s, len(ids), nbest))
    # previous-text prompts: the aligned ids start after each row's prompt
    prev = [[], [int(t) for t in range(10, 17)], [int(t) for t in range(30, 33)]]
    pp = transcribe.Session(wh, max_windows=3, max_beams=5, max_text_len=60)
    ids = pp.transcribe_windows_prev(waves, prev, sp, spec, beam_size=5, max_depth=30)
    first = [4 if not p else 1 + len(p) + 4 for p in prev]
    before = state_of(pp, 3, True)
    worst = max(worst, check_rows_align(pp, w64, dims, ids, first))
    same_state(before, state_of(pp, 3, True))
    h.report("align decoded rows tiny.en (every decode path)", worst, oa.MATRIX_TOL["f32"])


# ---------------------------------------------------------------- 5. error codes
def raw_align(sess, seqs, wins, first, heads=None, matrix=False, cap=None):
    lens = np.asarray([len(s) for s in seqs], dtype=np.int64)
    toks = np.asarray([t for s in seqs for t in s] or [0], dtype=np.int64)
    w = np.asarray(wins, dtype=np.int32)
    f = np.asarray(first, dtype=np.int64)
    hs = np.asarray(heads if heads is not None else [], dtype=np.int32).reshape(-1, 2)
    n = max(int(lens.sum()), 1)
    st, en = np.zeros(n, np.int32), np.zeros(n, np.int32)
    m = np.zeros(max(cap or 1, 1), np.float32)
    return ffi.lib().wb_session_align_tokens(sess._h, len(lens), ffi.i32ptr(w), ffi.i64ptr(toks), ffi.i64ptr(lens), ffi.i64ptr(f),
                                             len(hs), ffi.i32ptr(hs) if len(hs) else None, ffi.i32ptr(st), ffi.i32ptr(en),
                                             ffi.fptr(m) if matrix else None, cap or 0)


def test_error_codes(small):
    dims, wh, _, waves = small
    V, n_ctx, L, H = dims.n_vocab, dims.n_text_ctx, dims.n_text_layer, dims.n_text_head
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8)
    assert raw_align(sess, [[1, 2]], [0], [1]) == ffi.WB_ERR_STATE
    sess.encode_waveforms(waves)
    C0 = oa.window_columns(frames_of(len(waves[0]), dims.n_audio_ctx))
    assert raw_align(sess, [[1, 2]], [0], [1]) == ffi.WB_OK
    assert raw_align(sess, [[1]], [0], [1]) == ffi.WB_ERR_INVALID_ARG                       # lens 1
    assert raw_align(sess, [[1] * (n_ctx + 1)], [0], [4]) == ffi.WB_ERR_INVALID_ARG         # lens > n_text_ctx
    assert raw_align(sess, [[1, 2, 3]], [0], [0]) == ffi.WB_ERR_INVALID_ARG                 # first 0
    assert raw_align(sess, [[1, 2, 3]], [0], [3]) == ffi.WB_ERR_INVALID_ARG                 # first = len
    assert raw_align(sess, [[1, V]], [0], [1]) == ffi.WB_ERR_INVALID_ARG                    # id >= n_vocab
    assert raw_align(sess, [[1, -1]], [0], [1]) == ffi.WB_ERR_INVALID_ARG
    assert raw_align(sess, [[1, 2]], [2], [1]) == ffi.WB_ERR_INVALID_ARG                    # window not encoded
    assert raw_align(sess, [[1, 2]], [-1], [1]) == ffi.WB_ERR_INVALID_ARG
    assert raw_align(sess, [[1, 2]], [0], [1], heads=[(L, 0)]) == ffi.WB_ERR_INVALID_ARG    # layer outside
    assert raw_align(sess, [[1, 2]], [0], [1], heads=[(0, H)]) == ffi.WB_ERR_INVALID_ARG    # head outside
    assert raw_align(sess, [[1, 2]], [0], [1], heads=[(0, -1)]) == ffi.WB_ERR_INVALID_ARG
    assert raw_align(sess, [[1, 2]], [0], [1], heads=[(1, 1), (0, 2), (1, 1)]) == ffi.WB_ERR_INVALID_ARG   # listed twice
    assert raw_align(sess, [[1, 2, 3]], [0], [1], matrix=True, cap=2 * C0 - 1) == ffi.WB_ERR_INVALID_ARG  # capacity
    assert raw_align(sess, [[1, 2, 3]], [0], [1], matrix=True, cap=2 * C0) == ffi.WB_OK
    sess.close()
    dims_x, w_np, _, _ = h.synthetic("test-a", 3, exact=False, f64=False)
    wx = model.Whisper(dims_x, w_np)
    sx = transcribe.Session(wx, max_windows=1, max_beams=1, max_text_len=8)
    sx.encode_waveforms(waves[:1])
    assert raw_align(sx, [[1, 2]], [0], [1]) == ffi.WB_ERR_UNSUPPORTED
