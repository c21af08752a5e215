"""GPU tests (-m gpu) of wb_session_last_nbest: each window's n-best list, the beam search's final carried list ranked by
max_by_last applied repeatedly (host/beam.hpp beamfx::rank_final), from the on-device search (decoder6 beam mode) and
from the host search.  Lists are checked against the oracle's (tests/golden/nbest_beam.json, make_golden_nbest.py): ids,
lengths, finished flags and order; log-probs against float64 teacher forcing; rank 0 against the returned row."""
import ctypes as C

import numpy as np
import pytest
import torch

import harness as h
import oracle_prev_prompt as opp
import wb200  # noqa: F401
from harness import is_special_of, pool_waves
from oracle import synth, transcribe as o_tr
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    return h.golden("nbest_beam")


@pytest.fixture(scope="module")
def small():
    return h.named_model("test-a", f64=True)


@pytest.fixture(scope="module")
def tiny():
    return h.named_model("tiny.en", f64=True)


def session(wh, n, depth, kv, monkeypatch, decoder=0, prompt_len=4, max_beams=7):
    h.use_decoder(monkeypatch, decoder)
    try:
        return transcribe.Session(wh, max_windows=n, max_beams=max_beams, max_text_len=prompt_len + depth + 1,
                                  kv_dtype=h.kv_code(kv))
    finally:
        h.use_decoder(monkeypatch, 0)


def f64_sum(lps):
    total = 0.0
    for x in np.asarray(lps, dtype=np.float32).astype(np.float64):
        total += float(x)
    return total


def check_list(sess, index, row, nb, n_prompt, eot):
    """the list's own rules: rank 0 is the row and its last_logprobs bit for bit, prompts score 0, scores are the f64 sums"""
    assert nb[0][0] == row
    assert np.array_equal(nb[0][1], sess.last_logprobs(index))
    for ids, lps, score, fin in nb:
        assert lps.dtype == np.float32 and len(lps) == len(ids) and ids[:n_prompt] == row[:n_prompt]
        assert np.all(lps[:n_prompt] == 0.0) and np.all(lps[n_prompt:] <= 0.0)
        assert score == f64_sum(lps)
        assert fin == (ids[-1] == eot)
    scores = [h[2] for h in nb]
    assert all(scores[i] >= scores[i + 1] for i in range(len(scores) - 1))


def match_golden(nb, want, kv):
    """ids, lengths, finished flags and order equal the golden list's; two ranks may come out swapped only where their golden
    scores differ by less than the log-prob tolerance times the sequence length"""
    tol = h.GREEDY_LP_TOL[kv]
    got_ids = [h[0] for h in nb]
    want_ids = [h["ids"] for h in want["hyps"]]
    assert len(got_ids) == len(want_ids) and sorted(map(tuple, got_ids)) == sorted(map(tuple, want_ids)), (got_ids, want_ids)
    for r, (ids, _, score, fin) in enumerate(nb):
        w = want["hyps"][want_ids.index(ids)]
        assert fin == w["finished"]
        assert abs(score - w["score"]) < tol * len(ids)
        if ids != want_ids[r]:
            gap = abs(want["hyps"][r]["score"] - w["score"])
            assert gap < tol * len(ids), f"rank {r} swapped across a golden gap of {gap}"


def check_f64(sess, w64, dims, sp, window, nb, kv, n_prompt=4, seen=None):
    """every hypothesis's log-probs against float64 teacher forcing along its own ids"""
    xa = torch.from_numpy(sess.get_encoder_output(window)).double()[None]
    worst = 0.0
    for ids, lps, _, _ in nb:
        if seen is not None:
            if (window, tuple(ids)) in seen:
                continue
            seen.add((window, tuple(ids)))
        ref = h.along(h.path_rows(w64, dims, sp, xa, ids, kv, n_prompt=n_prompt), ids, n_prompt)
        err = float(np.abs(lps[n_prompt:].astype(np.float64) - ref).max(initial=0.0))
        assert err < h.GREEDY_LP_TOL[kv], f"window {window} {ids}: {lps[n_prompt:]} vs float64 {ref}"
        worst = max(worst, err)
    return worst


def run(sess, waves, sp, b, depth):
    ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=b, max_depth=depth)
    return ids, [sess.last_nbest(i) for i in range(len(waves))]


def same_lists(a, b):
    """ids, order and finished flags"""
    return [[(h[0], h[3]) for h in x] for x in a] == [[(h[0], h[3]) for h in x] for x in b]


# ---------------------------------------------------------------- 1, 2. device and host search against the golden lists
@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("b", [2, 3, 4, 5, 6, 7])
def test_nbest_device_test_a(small, gold, monkeypatch, b, kv):
    dims, sp, wh, _, _, w64 = small
    depth = gold["depth_test_a"]
    want = gold["test_a"][kv][str(b)]
    n_max = 24 // b
    sess = session(wh, n_max, depth, kv, monkeypatch)
    for n in range(1, n_max + 1):
        ids, nbs = run(sess, pool_waves(gold, n), sp, b, depth)
        assert sess.last_decoder() == 6, n
        for i, nb in enumerate(nbs):
            assert len(nb) <= 2 * b
            check_list(sess, i, ids[i], nb, 4, sp.eot)
            match_golden(nb, want[i % len(gold["pool"])], kv)
    seen: set = set()
    worst = max(check_f64(sess, w64, dims, sp, i, nb, kv, seen=seen) for i, nb in enumerate(nbs))
    h.report(f"last_nbest device beam test-a B={b} kv={kv}", worst, h.GREEDY_LP_TOL[kv])
    hs = session(wh, n_max, depth, kv, monkeypatch, decoder=3)
    hids, hnbs = run(hs, pool_waves(gold, n_max), sp, b, depth)
    assert hs.last_decoder() == 3 and hids == ids and same_lists(hnbs, nbs)


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_nbest_tiny_en_device_and_host(tiny, gold, monkeypatch, kv):
    dims, sp, wh, _, _, w64 = tiny
    te = h.golden("tokens_tiny_en")
    chunk = synth.chunk_waveform(0)
    waves = [chunk[s:e] for s, e in te["bounds"]]
    depth = gold["depth_tiny_en"]
    sess = session(wh, 3, depth, kv, monkeypatch)
    ids, nbs = run(sess, waves, sp, 5, depth)
    assert sess.last_decoder() == 6
    hs = session(wh, 3, depth, kv, monkeypatch, decoder=3)
    hids, hnbs = run(hs, waves, sp, 5, depth)
    assert hs.last_decoder() == 3 and hids == ids and same_lists(hnbs, nbs)
    for i in range(3):
        for s, lists in ((sess, nbs), (hs, hnbs)):
            check_list(s, i, ids[i], lists[i], 4, sp.eot)
            match_golden(lists[i], gold["tiny_en"][kv]["5"][i], kv)
    seen: set = set()
    worst = max(check_f64(sess, w64, dims, sp, i, nb, kv, seen=seen) for i, nb in enumerate(nbs))
    h.report(f"last_nbest device beam tiny.en B=5 kv={kv}", worst, h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 3. EOT, depth limit, previous-text prompts
@pytest.mark.parametrize("decoder", [0, 3])
def test_nbest_eot_and_depth_limit(small, gold, monkeypatch, decoder):
    """EOT declared to be a token the search emits: both windows stop early with a finished best and live hypotheses carried
    behind it, one several steps before the other; at depth 12 (test-a, default EOT) every list is live hypotheses only"""
    dims, sp, wh, _, _, w64 = small
    sp2 = o_tr.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, gold["eot"], sp.first_special, sp.n_vocab)
    chunk = synth.chunk_waveform(0)
    waves = [chunk[:238559], chunk[:98882]]
    sess = session(wh, 2, gold["depth_eot"], "f32", monkeypatch, decoder=decoder)
    ids, nbs = run(sess, waves, sp2, 5, gold["depth_eot"])
    assert sess.last_decoder() == (decoder or 6)
    for i, nb in enumerate(nbs):
        check_list(sess, i, ids[i], nb, 4, sp2.eot)
        want = gold["eot_case"]["f32"]["5"][i]
        match_golden(nb, want, "f32")
        fin = [h[3] for h in nb]
        assert fin[0] and not all(fin) and fin == [h["finished"] for h in want["hyps"]]
    check_f64(sess, w64, dims, sp2, 0, nbs[0], "f32")
    assert len(ids[0]) != len(ids[1])
    for lst in gold["test_a"]["f32"]["5"]:
        assert not any(h["finished"] for h in lst["hyps"]) and len(lst["hyps"]) == 5


@pytest.mark.parametrize("decoder", [0, 3])
def test_nbest_prev_prompt_mixed_lengths(small, gold, monkeypatch, decoder):
    """one launch over windows whose prompts hold 4, 7, 10 and 6 ids: each hypothesis starts with its window's own prompt,
    whose ids score 0"""
    dims, sp, wh, _, _, w64 = small
    depth = gold["depth_test_a"]
    prevs = gold["prev_ids"]
    prompts = [opp.build_prompt(sp, p) for p in prevs]
    sess = session(wh, 4, depth, "f32", monkeypatch, decoder=decoder, prompt_len=max(map(len, prompts)))
    ids = sess.transcribe_windows_prev(pool_waves(gold, 4), prevs, sp, is_special_of(sp), beam_size=5, max_depth=depth)
    assert sess.last_decoder() == (decoder or 6)
    for i in range(4):
        nb = sess.last_nbest(i)
        check_list(sess, i, ids[i], nb, len(prompts[i]), sp.eot)
        assert all(h[0][:len(prompts[i])] == prompts[i] for h in nb)
        match_golden(nb, gold["prev"]["f32"]["5"][i], "f32")
        if decoder == 0:
            check_f64(sess, w64, dims, sp, i, nb, "f32", n_prompt=len(prompts[i]))


# ---------------------------------------------------------------- 4. beam_size 1, max_depth 0, the greedy loop, state rules
def nbest_status(sess, index, max_hyps=14, capacity=64):
    ids = np.zeros((max_hyps, capacity), dtype=np.int64)
    lens = np.zeros(max_hyps, dtype=np.int64)
    scores = np.zeros(max_hyps, dtype=np.float64)
    n = C.c_int64(0)
    return ffi.lib().wb_session_last_nbest(sess._h, index, max_hyps, capacity, ffi.i64ptr(ids), None, ffi.i64ptr(lens),
                                           scores.ctypes.data_as(C.POINTER(C.c_double)), None, C.byref(n))


def test_nbest_greedy_depth0_loop_and_state_rules(small, gold, monkeypatch):
    dims, sp, wh, *_ = small
    waves = pool_waves(gold, 3)
    sess = session(wh, 3, 12, "f32", monkeypatch)
    assert nbest_status(sess, 0) == ffi.WB_ERR_STATE                   # before the first decode call
    # beam_size 1: one hypothesis, the row, score = the f64 sum of its log-probs
    ids, nbs = run(sess, waves, sp, 1, 12)
    for i, nb in enumerate(nbs):
        assert len(nb) == 1
        check_list(sess, i, ids[i], nb, 4, sp.eot)
    # max_depth 0: the prompt, score 0
    ids0, nbs0 = run(sess, waves, sp, 5, 0)
    for i, nb in enumerate(nbs0):
        assert [(h[0], h[2], h[3]) for h in nb] == [([sp.sot, sp.lang, sp.transcribe, sp.notimestamps], 0.0, False)]
        assert nb[0][0] == ids0[i] and np.array_equal(nb[0][1], np.zeros(4, np.float32))
    # a beam-5 list, then the rules around it
    ids5, nbs5 = run(sess, waves, sp, 5, 12)
    assert nbest_status(sess, 3) == ffi.WB_ERR_INVALID_ARG             # index out of range
    assert nbest_status(sess, 0, max_hyps=len(nbs5[0]) - 1) == ffi.WB_ERR_INVALID_ARG
    assert nbest_status(sess, 0, capacity=len(ids5[0]) - 1) == ffi.WB_ERR_INVALID_ARG
    # wb_session_score_tokens leaves it as it was
    sess.score_tokens([h[0] for h in nbs5[1]], [1] * len(nbs5[1]), apply_special_mask=True, is_special=is_special_of(sp))
    assert same_lists([sess.last_nbest(i) for i in range(3)], nbs5)
    # a call rejected before it encodes (beam_size above max_beams) leaves it as it was
    with pytest.raises(ffi.WbError) as e:
        sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=8, max_depth=12)
    assert e.value.code == ffi.WB_ERR_INVALID_ARG
    assert same_lists([sess.last_nbest(i) for i in range(3)], nbs5)
    # a call that fails after decoding (a row beyond capacity) leaves none
    ws = [np.ascontiguousarray(w, dtype=np.float32) for w in waves]
    ptrs = (ffi._F * 3)(*[ffi.fptr(w) for w in ws])
    lens = np.asarray([len(w) for w in ws], dtype=np.int64)
    out = np.zeros((3, 5), dtype=np.int64)
    out_len = np.zeros(3, dtype=np.int64)
    st = ffi.lib().wb_transcribe_windows(sess._h, ptrs, ffi.i64ptr(lens), 3, 5, 12, C.byref(transcribe._special_ids(sp)),
                                         ffi.u8ptr(is_special_of(sp)), ffi.i64ptr(out), 5, ffi.i64ptr(out_len))
    assert st == ffi.WB_ERR_INVALID_ARG
    assert nbest_status(sess, 0) == ffi.WB_ERR_STATE
    # the greedy loop carries no list
    loop = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=4 + 12 + 1, search="greedy_loop")
    loop.transcribe_windows(waves, sp, None, beam_size=1, max_depth=12)
    assert nbest_status(loop, 0) == ffi.WB_ERR_STATE
    with pytest.raises(ffi.WbError):
        loop.last_nbest(0)


# ---------------------------------------------------------------- 5. waveform calls
@pytest.mark.parametrize("prev_prompt", [False, True])
def test_nbest_waveforms_to_tokens_per_window(tiny, monkeypatch, prev_prompt):
    """two waveforms (30 s and 7 s) at beam 5: window k in waveform-major order has the n-best transcribe_windows(_prev) gives
    for the same slice, prompt and batch"""
    dims, sp, wh, *_ = tiny
    depth = 20
    chunk = synth.chunk_waveform(0)
    wave_b = synth.chunk_waveform(1)[:112000]
    sess = session(wh, 4, depth, "f32", monkeypatch, prompt_len=10)
    if prev_prompt:
        sess.set_prev_prompt(sp.startofprev)
    merged = sess.waveforms_to_tokens([chunk, wave_b], sp, is_special_of(sp), beam_size=5, max_depth=depth)
    assert sess.last_decoder() == 6
    wl = transcribe.window_samples(dims.n_audio_ctx)
    slices = [(0, chunk[s:e]) for s, e in transcribe.window_bounds(len(chunk), 16000, wl)]
    slices += [(1, wave_b[s:e]) for s, e in transcribe.window_bounds(len(wave_b), 16000, wl)]
    assert len(slices) == 4
    got = [sess.last_nbest(k) for k in range(len(slices))]
    with pytest.raises(ffi.WbError):
        sess.last_nbest(len(slices))
    ref = session(wh, 4, depth, "f32", monkeypatch, prompt_len=10)
    if not prev_prompt:   # one batch of all windows
        ref.transcribe_windows([w for _, w in slices], sp, is_special_of(sp), beam_size=5, max_depth=depth)
        want = [ref.last_nbest(k) for k in range(4)]
    else:                 # round i: window i of every waveform that has one, prompted by its waveform's merged ids so far
        want = [None] * 4
        done = {0: [], 1: []}
        rounds = [[0, 3], [1], [2]]
        for rnd in rounds:
            prevs = [opp.prev_nonspecial(done[slices[k][0]], sp.is_special) for k in rnd]
            rows = ref.transcribe_windows_prev([slices[k][1] for k in rnd], prevs, sp, is_special_of(sp), beam_size=5,
                                               max_depth=depth)
            for j, k in enumerate(rnd):
                want[k] = ref.last_nbest(j)
                ov = o_tr.find_chunk_overlap(done[slices[k][0]], rows[j], 40, 3)
                m = done[slices[k][0]]
                done[slices[k][0]] = m[:ov[0]] + rows[j][ov[1]:] if ov is not None else m + rows[j]
        assert [done[0], done[1]] == merged
    for k in range(4):
        assert len(got[k]) == len(want[k])
        for g, w in zip(got[k], want[k]):
            assert g[0] == w[0] and g[2] == w[2] and g[3] == w[3] and np.array_equal(g[1], w[1]), k


# ---------------------------------------------------------------- 6. rescoring round trip
@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_nbest_rescoring_round_trip(small, gold, monkeypatch, kv):
    """score_tokens on every hypothesis of a window reproduces the log-probs the search scored its generated ids with"""
    _, sp, wh, *_ = small
    sess = session(wh, 2, gold["depth_test_a"], kv, monkeypatch)
    ids, nbs = run(sess, pool_waves(gold, 2), sp, 5, gold["depth_test_a"])
    for w in range(2):
        hyps = nbs[w]
        scored = sess.score_tokens([h[0] for h in hyps], [w] * len(hyps), apply_special_mask=True, is_special=is_special_of(sp))
        for (hid, hlp, _, _), (lp, _) in zip(hyps, scored):
            assert np.abs(lp[4:].astype(np.float64) - hlp[4:]).max() < h.GREEDY_LP_TOL[kv], hid
        assert same_lists([sess.last_nbest(i) for i in range(2)], nbs)
