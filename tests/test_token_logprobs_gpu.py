"""GPU tests (-m gpu) of the per-token log-probs of a transcription (wb_session_last_logprobs, Session.last_logprobs): the
BeamSearchToken.log_prob of every id the reference's search returns (src/transcribe.rs:142-146, 205-208, 291-299).

  1. on every path a row has one value per id, 0 for the 4 prompt ids, finite and <= 0 elsewhere except a rule's EOT;
  2. greedy on decoder3 / 4 / 5 / 6, fp32 and fp16 K/V: each value against float64 teacher forcing of the GPU's own ids
     (greedy_path_log_probs on the reduced-depth real-width models of test_f64_reference_gpu.py, its GREEDY_LP_TOL);
  3. real shapes: small.en 8 chunks and medium chunk 0 against the top-1 log-probs of tests/golden/tokens_real.json, the
     native windows against tokens_native.json (LP_TOL of test_real_shapes_gpu.py), wherever the ids match;
  4. the greedy loop on every decoder (the cases of test_greedy_loop_gpu.py): NaN exactly at the rule-appended EOTs, the
     arg-max values against the oracle loop's unmasked log-softmax;
  5. beam: the device search (decoder6) and the host search (decoder5, decoder3) against float64 teacher forcing, and device
     and host values equal within tolerance wherever their ids agree;
  6. the merge of waveform(s)_to_tokens equals the oracle merge of transcribe_windows' per-window rows of the same batch;
  7. the getter's contract."""
import ctypes as C
import dataclasses
import json
import math
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_logprobs as olp
import test_f64_reference_gpu as f64
import test_greedy_loop_gpu as gl
import wb200  # noqa: F401
from oracle import audio as o_audio, model as o_model, synth, transcribe as o_tr
from whisper_burn_b200 import ffi, model, transcribe

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"
LP_TOL = 2e-4   # test_real_shapes_gpu.py: GPU log-probs against the float32 oracle's at real shapes


def is_special_of(sp):
    return (np.arange(sp.n_vocab) >= sp.first_special).astype(np.uint8)


def rows_of(sess, ids, rule_eots=None):
    """last_logprobs of every row, checked for shape, prompt and range; rule_eots[r]: the positions of row r that may be
    NaN (an EOT a rule appended)."""
    out = []
    for r, t in enumerate(ids):
        lps = sess.last_logprobs(r)
        assert lps.dtype == np.float32 and len(lps) == len(t), f"row {r}"
        assert np.all(lps[:4] == 0.0), f"row {r}: prompt log-probs {lps[:4]}"
        allowed = set(rule_eots[r]) if rule_eots else set()
        for j in range(4, len(t)):
            if j in allowed:
                continue
            assert math.isfinite(lps[j]) and lps[j] <= 0.0, f"row {r} position {j}: {lps[j]}"
        out.append(lps)
    return out


def teacher_forced(w, dims, sp, xa, ids, kv, unmask=False, ln_eps_mode="outside"):
    """The log-prob of ids[j], j >= 4, given ids[:j]: one greedy_path_log_probs pass over the path (mask of the beam rule, or
    none for the greedy loop)."""
    rows = o_tr.greedy_path_log_probs(w, dims, olp.unmasked(sp) if unmask else sp, xa, ids,
                                      opts=o_model.OracleOptions(ln_eps_mode=ln_eps_mode, kv_dtype=kv))
    return np.array([float(rows[j - 4][ids[j]]) for j in range(4, len(ids))])


def check_against_f64(sess, w64, dims, sp, ids, lps, kv, unmask=False, skip_nan=False, ln_eps_mode="outside"):
    worst = 0.0
    for r, t in enumerate(ids):
        xa = torch.from_numpy(sess.get_encoder_output(r)).double()[None]
        ref = teacher_forced(w64, dims, sp, xa, t, kv, unmask, ln_eps_mode)
        got = lps[r][4:].astype(np.float64)
        ok = ~np.isnan(got) if skip_nan else np.ones(len(got), bool)
        err = np.abs(got[ok] - ref[ok]).max(initial=0.0)
        worst = max(worst, float(err))
        assert err < f64.GREEDY_LP_TOL[kv], f"row {r}: log-probs {got} vs float64 {ref}"
    return worst


# ---------------------------------------------------------------- 2. greedy, every decoder, against float64
# (decoder, d, heads, rows): decoder4 and decoder6 at d = 384, decoder5 at d = 256, decoder3 at d = 384
GREEDY_CASES = [(4, 384, 6, 4), (6, 384, 6, 9), (5, 256, 4, 9), (3, 384, 6, 4)]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("decoder,d,H,rows", GREEDY_CASES)
def test_greedy_logprobs_every_decoder_vs_float64(decoder, d, H, rows, kv, monkeypatch):
    dims, wh, w64 = f64.make_model(d, H, 2051)
    sp = synth.special_tokens(dims)
    Ts, waves = f64.windows(rows, seed=11 * d + rows)
    f64.use_decoder(monkeypatch, decoder)
    sess = transcribe.Session(wh, max_windows=rows, max_beams=1, max_text_len=4 + f64.DEPTH + 1, kv_dtype=f64.kv_code(kv))
    f64.use_decoder(monkeypatch, 0)
    ids = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=f64.DEPTH)
    assert sess.last_decoder() == decoder
    lps = rows_of(sess, ids)
    for r, t in enumerate(ids):   # the greedy value of the last step is what wb_session_last_topk reports
        if len(t) == 4 + f64.DEPTH:
            tk, tl = sess.last_topk(rows, 1)
            assert int(tk[r, 0]) == t[-1] and float(tl[r, 0]) == float(lps[r][-1])
    worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
    f64.report(f"last_logprobs greedy decoder{decoder} d={d} rows={rows} kv={kv}", worst, f64.GREEDY_LP_TOL[kv])


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
            assert err < LP_TOL, f"row {r} position {j}: {lps[r][j]} vs oracle {top_lp[0]}"
    return worst


def test_small_en_8_chunks_and_medium_vs_golden_top1():
    g = json.loads((G / "tokens_real.json").read_text())
    dims, w_np, _ = synth.make_weights("small.en", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    waves, recs = [], []
    for c, rec in enumerate(g["small.en"]["chunks"]):
        chunk = synth.chunk_waveform(c)
        for (s, e), r in zip(rec["bounds"], rec["f32"]):
            waves.append(chunk[s:e])
            recs.append(r)
    sess = transcribe.Session(wh, max_windows=24, max_beams=1, max_text_len=105)
    ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 5
    f64.report("last_logprobs small.en 24 windows greedy f32 vs golden top-1", check_top1(ids, rows_of(sess, ids), recs), LP_TOL)
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
    f64.report("last_logprobs medium chunk 0 greedy f32 vs golden top-1", check_top1(ids, rows_of(sess, ids), gm["f32"]), LP_TOL)


@pytest.mark.parametrize("case,max_windows", [("tiny.en", 4), ("small.en", 2)])
def test_native_windows_vs_golden_top1(case, max_windows):
    g = json.loads((G / "tokens_native.json").read_text())[case]
    dims, w_np, _ = synth.make_weights(case, seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    for kv in ("f32", "f16"):
        sess = transcribe.Session(wh, max_windows=max_windows, max_beams=1, max_text_len=105, kv_dtype=f64.kv_code(kv),
                                  windows="native")
        waves = [synth.chunk_waveform(c)[:n] for c, n in g["windows"]]
        ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
        f64.report(f"last_logprobs native {case} greedy kv={kv} vs golden top-1", check_top1(ids, rows_of(sess, ids), g[kv]),
                   LP_TOL)
        sess.close()


# ---------------------------------------------------------------- 4. the greedy loop
_LOOP = {}


def loop_oracle(name, i, sp, max_depth, kv):
    key = (name, i, sp.eot, max_depth, kv)
    if key not in _LOOP:
        dims, w_t, _ = gl.weights(name)
        tr = {}
        ids, lps = olp.greedy_loop_logprobs(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(gl.window(i))[None]), max_depth,
                                            o_model.OracleOptions(kv_dtype=kv), trace=tr)
        _LOOP[key] = (ids, lps, tr)
    return _LOOP[key]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("dec,name,n,t_max,rules", gl.CASES)
def test_greedy_loop_logprobs(monkeypatch, dec, name, n, t_max, rules, kv):
    dims, _, _ = gl.weights(name)
    sp = dataclasses.replace(synth.special_tokens(dims), eot=gl.EOT_ID)
    monkeypatch.setenv("WB200_DECODER", str(dec))
    s = gl.session(name, n, t_max, kv)
    monkeypatch.delenv("WB200_DECODER")
    waves = [gl.window(i) for i in range(n)]
    tol = f64.GREEDY_LP_TOL[kv]
    stops, worst = set(), 0.0
    for max_depth in (t_max - 4, 3):
        got = s.transcribe_windows(waves, sp, None, beam_size=1, max_depth=max_depth)
        assert s.last_decoder() == dec
        lps = rows_of(s, got, [[len(t) - 1] for t in got])
        for i in range(n):
            want, want_lp, tr = loop_oracle(name, i, sp, max_depth, kv)
            stops.add(tr["stop"])
            if got[i] != want:   # a near tie the GPU resolved the other way (test_greedy_loop_gpu.py): compare the prefix
                assert gl.same_up_to_ties(got[i], want, tr)
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
    f64.report(f"last_logprobs greedy loop decoder{dec} {name} kv={kv} vs oracle", worst, tol)
    s.close()


# ---------------------------------------------------------------- 5. beam: device and host search
@pytest.fixture(scope="module")
def beam_gold():
    return json.loads((G / "tokens_beam.json").read_text())


def pool_waves(gold, n):
    chunk = synth.chunk_waveform(0)
    return [chunk[off:off + m] for off, m in (gold["pool"][i % len(gold["pool"])] for i in range(n))]


def beam_run(wh, waves, sp, b, depth, kv, monkeypatch, decoder=0):
    f64.use_decoder(monkeypatch, decoder)
    sess = transcribe.Session(wh, max_windows=len(waves), max_beams=7, max_text_len=4 + depth + 1, kv_dtype=f64.kv_code(kv))
    f64.use_decoder(monkeypatch, 0)
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
def test_beam_test_a_device_and_host_vs_float64(beam_gold, monkeypatch, kv):
    dims, w_np, w_t = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    w64 = o_model.as_dtype(w_t)
    depth = beam_gold["depth_test_a"]
    for b in range(2, 8):
        waves = pool_waves(beam_gold, 24 // b)
        sess, ids, lps = beam_run(wh, waves, sp, b, depth, kv, monkeypatch)
        assert sess.last_decoder() == 6
        check_beam_sums(lps)
        worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
        f64.report(f"last_logprobs device beam test-a B={b} kv={kv}", worst, f64.GREEDY_LP_TOL[kv])
        if b == 5:   # the host search (decoder3) returns the same ids; its values agree within tolerance
            hs, hids, hlps = beam_run(wh, waves, sp, b, depth, kv, monkeypatch, decoder=3)
            assert hs.last_decoder() == 3 and hids == ids
            for r in range(len(ids)):
                assert np.abs(hlps[r].astype(np.float64) - lps[r]).max() < f64.GREEDY_LP_TOL[kv]
            check_against_f64(hs, w64, dims, sp, hids, hlps, kv)


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_beam_tiny_en_device_vs_float64(beam_gold, monkeypatch, kv):
    dims, w_np, w_t = synth.make_weights("tiny.en", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    w64 = o_model.as_dtype(w_t)
    te = json.loads((G / "tokens_tiny_en.json").read_text())
    chunk = synth.chunk_waveform(0)
    sess, ids, lps = beam_run(wh, [chunk[s:e] for s, e in te["bounds"]], sp, 5, beam_gold["depth_tiny_en"], kv, monkeypatch)
    assert sess.last_decoder() == 6 and ids == beam_gold["tiny_en"][kv]["5"]
    worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
    f64.report(f"last_logprobs device beam tiny.en B=5 kv={kv}", worst, f64.GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_beam_host_search_decoder5_vs_float64(monkeypatch, kv):
    dims, wh, w64 = f64.make_model(256, 4, 2051)
    sp = synth.special_tokens(dims)
    _, waves = f64.windows(3, seed=41)
    sess, ids, lps = beam_run(wh, waves, sp, 5, f64.DEPTH, kv, monkeypatch)
    assert sess.last_decoder() == 5
    check_beam_sums(lps)
    worst = check_against_f64(sess, w64, dims, sp, ids, lps, kv)
    f64.report(f"last_logprobs host beam decoder5 d=256 B=5 kv={kv}", worst, f64.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 6. the merge
@pytest.mark.parametrize("beam_size", [1, 5])
@pytest.mark.parametrize("windows", ["reference", "native"])
def test_merge_carries_logprobs_with_their_ids(windows, beam_size):
    dims, w_np, _ = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
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
    dims, w_np, _ = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=12)
    lib, n = ffi.lib(), C.c_int64(-1)
    buf = np.zeros(64, np.float32)
    assert lib.wb_session_last_logprobs(sess._h, 0, ffi.fptr(buf), 64, C.byref(n)) == ffi.WB_ERR_STATE
    ids = sess.transcribe_windows([gl.window(0), gl.window(1)], sp, is_special_of(sp), beam_size=1, max_depth=6)
    for i in (-1, 2):
        assert lib.wb_session_last_logprobs(sess._h, i, ffi.fptr(buf), 64, C.byref(n)) == ffi.WB_ERR_INVALID_ARG
    assert lib.wb_session_last_logprobs(sess._h, 1, None, 0, C.byref(n)) == ffi.WB_OK and n.value == len(ids[1])
    assert lib.wb_session_last_logprobs(sess._h, 1, ffi.fptr(buf), n.value - 1, C.byref(n)) == ffi.WB_ERR_INVALID_ARG
    assert lib.wb_session_last_logprobs(sess._h, 1, ffi.fptr(buf), 64, C.byref(n)) == ffi.WB_OK
    assert olp.same(buf[:n.value], sess.last_logprobs(1))
