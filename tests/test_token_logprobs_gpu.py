"""GPU tests (-m gpu) of the per-token log-probs of a transcription (wb_session_last_logprobs, Session.last_logprobs): the
BeamSearchToken.log_prob of every id the reference's search returns (src/transcribe.rs:142-146, 205-208, 291-299).

  1. on every path a row has one value per id, 0 for the 4 prompt ids, finite and <= 0 elsewhere except a rule's EOT;
  2. greedy on decoder3 / 4 / 5 / 6, fp32 and fp16 K/V: each value against float64 teacher forcing of the GPU's own ids
     (greedy_path_log_probs on the reduced-depth real-width models of harness.make_model, harness.GREEDY_LP_TOL);
  3. real shapes: small.en 8 chunks and medium chunk 0 against the top-1 log-probs of tests/golden/tokens_real.json, the
     native windows against tokens_native.json (harness.REAL_LP_TOL), wherever the ids match;
  4. the greedy loop on every decoder (the cases of test_greedy_loop_gpu.py): NaN exactly at the rule-appended EOTs, the
     arg-max values against the oracle loop's unmasked log-softmax;
  5. beam: the device search (decoder6) and the host search (decoder5, decoder3) against float64 teacher forcing, and device
     and host values equal within tolerance wherever their ids agree;
  6. the merge of waveform(s)_to_tokens equals the oracle merge of transcribe_windows' per-window rows of the same batch;
  7. the getter's contract."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
import torch

import harness as h
import oracle_logprobs as olp
import wb200  # noqa: F401
from harness import check_against_f64, is_special_of, pool_waves, rows_of
from oracle import audio as o_audio, model as o_model, synth
from whisper_burn_b200 import ffi, model, transcribe

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- 2. greedy, every decoder, against float64
# (decoder, d, heads, rows): decoder4 and decoder6 at d = 384, decoder5 at d = 256, decoder3 at d = 384
GREEDY_CASES = [(4, 384, 6, 4), (6, 384, 6, 9), (5, 256, 4, 9), (3, 384, 6, 4)]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("decoder,d,H,rows", GREEDY_CASES)
def test_greedy_logprobs_every_decoder_vs_float64(decoder, d, H, rows, kv, monkeypatch):
    dims, wh, w64 = h.make_model(d, H, 2051)
    sp = synth.special_tokens(dims)
    Ts, waves = h.windows(rows, seed=11 * d + rows)
    h.use_decoder(monkeypatch, decoder)
    sess = transcribe.Session(wh, max_windows=rows, max_beams=1, max_text_len=4 + h.DEPTH + 1, kv_dtype=h.kv_code(kv))
    h.use_decoder(monkeypatch, 0)
    ids = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=h.DEPTH)
    assert sess.last_decoder() == decoder
    lps = rows_of(sess, ids)
    for r, t in enumerate(ids):   # the greedy value of the last step is what wb_session_last_topk reports
        if len(t) == 4 + h.DEPTH:
            tk, tl = sess.last_topk(rows, 1)
            assert int(tk[r, 0]) == t[-1] and float(tl[r, 0]) == float(lps[r][-1])
    worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
    h.report(f"last_logprobs greedy decoder{decoder} d={d} rows={rows} kv={kv}", worst, h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 3. real shapes against the fixtures' top-1 log-probs
def check_top1(got_ids, lps, recs):
    worst = 0.0
    for r, (t, rec) in enumerate(zip(got_ids, recs)):
        want = rec["tokens"]
        for s, (top_ids, top_lp) in enumerate(rec["top5"]):
            j = 4 + s
            if j >= len(t) or t[:j + 1] != want[:j + 1]:
                break
            err = abs(float(lps[r][j]) - top_lp[0])
            worst = max(worst, err)
            assert err < h.REAL_LP_TOL, f"row {r} position {j}: {lps[r][j]} vs oracle {top_lp[0]}"
    return worst


def test_small_en_8_chunks_and_medium_vs_golden_top1():
    g = h.golden("tokens_real")
    dims, w_np, _ = synth.make_weights("small.en", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    waves, recs = h.real_windows("small.en", "f32")
    sess = transcribe.Session(wh, max_windows=24, max_beams=1, max_text_len=105)
    ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 5
    h.report("last_logprobs small.en 24 windows greedy f32 vs golden top-1", check_top1(ids, rows_of(sess, ids), recs), h.REAL_LP_TOL)
    sess.close()
    del sess, wh
    gm = g["medium"]
    dims, w_np, _ = synth.make_weights("medium", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    chunk = synth.chunk_waveform(0)
    sess = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=35)
    ids = sess.transcribe_windows([chunk[s:e] for s, e in gm["bounds"]], sp, is_special_of(sp), beam_size=1, max_depth=30)
    assert sess.last_decoder() == 5
    h.report("last_logprobs medium chunk 0 greedy f32 vs golden top-1", check_top1(ids, rows_of(sess, ids), gm["f32"]), h.REAL_LP_TOL)


@pytest.mark.parametrize("case,max_windows", [("tiny.en", 4), ("small.en", 2)])
def test_native_windows_vs_golden_top1(case, max_windows):
    g = h.golden("tokens_native")[case]
    dims, w_np, _ = synth.make_weights(case, seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    for kv in ("f32", "f16"):
        sess = transcribe.Session(wh, max_windows=max_windows, max_beams=1, max_text_len=105, kv_dtype=h.kv_code(kv),
                                  windows="native")
        waves = [synth.chunk_waveform(c)[:n] for c, n in g["windows"]]
        ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
        h.report(f"last_logprobs native {case} greedy kv={kv} vs golden top-1", check_top1(ids, rows_of(sess, ids), g[kv]),
                   h.REAL_LP_TOL)
        sess.close()


# ---------------------------------------------------------------- 4. the greedy loop
_LOOP = {}


def loop_oracle(name, i, sp, max_depth, kv):
    key = (name, i, sp.eot, max_depth, kv)
    if key not in _LOOP:
        dims, _, _, _, w_t, _ = h.loop_model(name)
        tr = {}
        ids, lps = olp.greedy_loop_logprobs(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(h.loop_window(i))[None]), max_depth,
                                            o_model.OracleOptions(kv_dtype=kv), trace=tr)
        _LOOP[key] = (ids, lps, tr)
    return _LOOP[key]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("dec,name,n,t_max,rules", h.LOOP_CASES)
def test_greedy_loop_logprobs(monkeypatch, dec, name, n, t_max, rules, kv):
    dims = h.loop_model(name).dims
    sp = dataclasses.replace(synth.special_tokens(dims), eot=h.LOOP_EOT_ID)
    monkeypatch.setenv("WB200_DECODER", str(dec))
    s = h.loop_session(name, n, t_max, kv)
    monkeypatch.delenv("WB200_DECODER")
    waves = [h.loop_window(i) for i in range(n)]
    tol = h.GREEDY_LP_TOL[kv]
    stops, worst = set(), 0.0
    for max_depth in (t_max - 4, 3):
        got = s.transcribe_windows(waves, sp, None, beam_size=1, max_depth=max_depth)
        assert s.last_decoder() == dec
        lps = rows_of(s, got, [[len(t) - 1] for t in got])
        for i in range(n):
            want, want_lp, tr = loop_oracle(name, i, sp, max_depth, kv)
            stops.add(tr["stop"])
            if got[i] != want:   # a near tie the GPU resolved the other way (test_greedy_loop_gpu.py): compare the prefix
                assert h.same_up_to_ties(got[i], want, tr)
                n_common = min(len(got[i]), len(want))
                m = next((j for j in range(n_common) if got[i][j] != want[j]), n_common)
                a, b = lps[i][4:m].astype(np.float64), np.asarray(want_lp[4:m])
                assert np.abs(a - b).max(initial=0.0) < tol
                continue
            assert olp.same(np.isnan(lps[i]), np.isnan(want_lp)), f"window {i}: NaN at {np.isnan(lps[i]).nonzero()}"
            ok = ~np.isnan(lps[i])
            err = np.abs(lps[i][ok].astype(np.float64) - np.asarray(want_lp)[ok]).max()
            worst = max(worst, float(err))
            assert err < tol, f"window {i}: {lps[i]} vs oracle {want_lp}"
    assert stops == rules, stops
    h.report(f"last_logprobs greedy loop decoder{dec} {name} kv={kv} vs oracle", worst, tol)
    s.close()


# ---------------------------------------------------------------- 5. beam: device and host search
def beam_run(wh, waves, sp, b, depth, kv, monkeypatch, decoder=0):
    h.use_decoder(monkeypatch, decoder)
    sess = transcribe.Session(wh, max_windows=len(waves), max_beams=7, max_text_len=4 + depth + 1, kv_dtype=h.kv_code(kv))
    h.use_decoder(monkeypatch, 0)
    ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=b, max_depth=depth)
    return sess, ids, rows_of(sess, ids)


def check_beam_sums(lps):
    """a beam row's f64 left-to-right sum is finite: the score its search kept it by (checked exactly by the CPU tests)"""
    for v in lps:
        total = 0.0
        for x in v.astype(np.float64):
            total += x
        assert math.isfinite(total) and total <= 0.0


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_beam_test_a_device_and_host_vs_float64(monkeypatch, kv):
    beam_gold = h.golden("tokens_beam")
    dims, sp, wh, _, _, w64 = h.named_model("test-a", f64=True)
    depth = beam_gold["depth_test_a"]
    for b in range(2, 8):
        waves = pool_waves(beam_gold, 24 // b)
        sess, ids, lps = beam_run(wh, waves, sp, b, depth, kv, monkeypatch)
        assert sess.last_decoder() == 6
        check_beam_sums(lps)
        worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
        h.report(f"last_logprobs device beam test-a B={b} kv={kv}", worst, h.GREEDY_LP_TOL[kv])
        if b == 5:   # the host search (decoder3) returns the same ids; its values agree within tolerance
            hs, hids, hlps = beam_run(wh, waves, sp, b, depth, kv, monkeypatch, decoder=3)
            assert hs.last_decoder() == 3 and hids == ids
            for r in range(len(ids)):
                assert np.abs(hlps[r].astype(np.float64) - lps[r]).max() < h.GREEDY_LP_TOL[kv]
            check_against_f64(hs, w64, dims, sp, hids, hlps, kv)


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_beam_tiny_en_device_vs_float64(monkeypatch, kv):
    beam_gold = h.golden("tokens_beam")
    dims, sp, wh, _, _, w64 = h.named_model("tiny.en", f64=True)
    te = h.golden("tokens_tiny_en")
    chunk = synth.chunk_waveform(0)
    sess, ids, lps = beam_run(wh, [chunk[s:e] for s, e in te["bounds"]], sp, 5, beam_gold["depth_tiny_en"], kv, monkeypatch)
    assert sess.last_decoder() == 6 and ids == beam_gold["tiny_en"][kv]["5"]
    worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
    h.report(f"last_logprobs device beam tiny.en B=5 kv={kv}", worst, h.GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_beam_host_search_decoder5_vs_float64(monkeypatch, kv):
    dims, wh, w64 = h.make_model(256, 4, 2051)
    sp = synth.special_tokens(dims)
    _, waves = h.windows(3, seed=41)
    sess, ids, lps = beam_run(wh, waves, sp, 5, h.DEPTH, kv, monkeypatch)
    assert sess.last_decoder() == 5
    check_beam_sums(lps)
    worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
    h.report(f"last_logprobs host beam decoder5 d=256 B=5 kv={kv}", worst, h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 6. the merge
@pytest.mark.parametrize("beam_size", [1, 5])
@pytest.mark.parametrize("windows", ["reference", "native"])
def test_merge_carries_logprobs_with_their_ids(windows, beam_size):
    dims, sp, wh, *_ = h.named_model("test-a")
    bitmap = is_special_of(sp)
    waves = [synth.waveform(16000 * 70, seed=78), synth.waveform(16000 * 40, seed=79)]
    wl = transcribe.window_samples(dims.n_audio_ctx, windows)
    bounds = [transcribe.window_bounds(len(w), 16000, wl) for w in waves]
    n_win = sum(len(b) for b in bounds)
    assert all(len(b) >= 2 for b in bounds)
    sess = transcribe.Session(wh, max_windows=n_win, max_beams=5, max_text_len=4 + 20 + 1, windows=windows)
    # the same windows in the same batch through transcribe_windows, merged by the oracle
    flat = [w[s:e] for w, b in zip(waves, bounds) for s, e in b]
    ids = sess.transcribe_windows(flat, sp, bitmap, beam_size=beam_size, max_depth=20)
    lps = rows_of(sess, ids)
    per, k = [], 0
    for b in bounds:
        per.append(olp.merge([(ids[k + i], list(lps[k + i])) for i in range(len(b))]))
        k += len(b)
    got = sess.waveforms_to_tokens(waves, sp, bitmap, beam_size=beam_size, max_depth=20)
    for i in range(len(waves)):
        assert got[i] == per[i][0]
        assert olp.same(sess.last_logprobs(i), np.asarray(per[i][1], np.float32))
    flat0 = flat[:len(bounds[0])]   # waveform_to_tokens: the windows of waves[0] alone
    ids0 = sess.transcribe_windows(flat0, sp, bitmap, beam_size=beam_size, max_depth=20)
    want = olp.merge([(t, list(sess.last_logprobs(i))) for i, t in enumerate(ids0)])
    assert sess.waveform_to_tokens(waves[0], sp, bitmap, beam_size=beam_size, max_depth=20) == want[0]
    assert olp.same(sess.last_logprobs(0), np.asarray(want[1], np.float32))


# ---------------------------------------------------------------- 7. the getter's contract
def test_getter_contract():
    dims, sp, wh, *_ = h.named_model("test-a")
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=12)
    lib, n = ffi.lib(), C.c_int64(-1)
    buf = np.zeros(64, np.float32)
    assert lib.wb_session_last_logprobs(sess._h, 0, ffi.fptr(buf), 64, C.byref(n)) == ffi.WB_ERR_STATE
    ids = sess.transcribe_windows([h.loop_window(0), h.loop_window(1)], sp, is_special_of(sp), beam_size=1, max_depth=6)
    for i in (-1, 2):
        assert lib.wb_session_last_logprobs(sess._h, i, ffi.fptr(buf), 64, C.byref(n)) == ffi.WB_ERR_INVALID_ARG
    assert lib.wb_session_last_logprobs(sess._h, 1, None, 0, C.byref(n)) == ffi.WB_OK and n.value == len(ids[1])
    assert lib.wb_session_last_logprobs(sess._h, 1, ffi.fptr(buf), n.value - 1, C.byref(n)) == ffi.WB_ERR_INVALID_ARG
    assert lib.wb_session_last_logprobs(sess._h, 1, ffi.fptr(buf), 64, C.byref(n)) == ffi.WB_OK
    assert olp.same(buf[:n.value], sess.last_logprobs(1))
