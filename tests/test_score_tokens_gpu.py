"""GPU tests (-m gpu) of teacher-forced token scoring (wb_session_score_tokens, Session.score_tokens): forward_decoder
(mod.rs:131-157) + log_softmax (transcribe.rs:276) at every position of given sequences, in one sequence-parallel pass.

  1. against float64 (oracle.model.forward_decoder on the real-width models of harness.make_model): d = 384, 768,
     1280, fp32 and fp16 K/V, reference windows of T = 6, 64, 65, 750 and native windows of T = 1500 and 1025, random
     sequences (special ids included) of lengths around the 64-row tiles up to n_text_ctx, several on one window;
  2. the special-token mask of the beam rule (greedy_path_log_probs from the prompt on; -inf targets at j = 4, 5 only);
  3. agreement with decoding: the rows transcribe_windows returned score what last_logprobs reports (greedy, beam 5 on the
     device and on the host, the greedy loop unmasked), and the greedy arg-max is the decoded id;
  4. real shapes: small.en 8 chunks and medium chunk 0 along tests/golden/tokens_real.json;
  5. sequence parallel and independent: a fixed launch count, bit-identical values alone, in a batch and as prefixes;
  6. the session's decode results are untouched;
  7. every error code of the header contract."""
import numpy as np
import pytest
import torch

import harness as h
import wb200  # noqa: F401
from harness import GAP, check_rows, is_special_of, random_seqs
from oracle import synth
from whisper_burn_b200 import ffi, model, transcribe

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- 1. against float64
def score_vs_f64(d, kv, windows, Ts, waves, seed):
    dims, wh, w64 = h.make_model(d, d // 64, 2051)
    sess = transcribe.Session(wh, max_windows=len(waves), max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv), windows=windows)
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    seqs = random_seqs(dims.n_vocab, seed)
    wins = [i % len(waves) for i in range(len(seqs))]
    out = sess.score_tokens(seqs, wins)
    worst = 0.0
    for i, (seq, w) in enumerate(zip(seqs, wins)):
        lp, am = out[i]
        assert lp.dtype == np.float32 and am.dtype == np.int64 and len(lp) == len(seq)
        ref = h.forward_rows(w64, dims, [xa[w]], [seq], kv)[0] if len(seq) > 1 else None
        worst = max(worst, check_rows(lp, am, ref, seq, kv, f"d={d} kv={kv} T={Ts[w]} len={len(seq)}"))
    h.report(f"score_tokens d={d} {windows} windows T={sorted(set(Ts))} kv={kv}", worst, h.GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("d", [384, 768, 1280])
def test_score_vs_float64(d, kv):
    Ts, waves = h.windows(4, seed=7 * d)
    score_vs_f64(d, kv, "reference", Ts, waves, seed=d)


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_score_native_windows_vs_float64(kv):
    # T = 1500: a full 30 s window; T = 1025: 2039 frames -> (2039 + 10 - 1) // 2 + 1
    waves = [synth.waveform(480000, seed=3), synth.waveform(2039 * 160, seed=4)]
    score_vs_f64(384, kv, "native", [1500, 1025], waves, seed=5)


# ---------------------------------------------------------------- 2. the special-token mask
@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_mask_rule_matches_greedy_path_log_probs(kv):
    dims, wh, w64 = h.make_model(384, 6, 2051)
    sp = synth.special_tokens(dims)
    Ts, waves = h.windows(2, seed=17)
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    seqs = h.masked_seqs(sp, 9)   # special ids at j = 4, 5, 6, 9
    wins = [r % 2 for r in range(4)]
    out = sess.score_tokens(seqs, wins, apply_special_mask=True, is_special=is_special_of(sp))
    worst = 0.0
    for seq, w, (lp, _) in zip(seqs, wins, out):
        assert np.isneginf(lp[4]) and np.isneginf(lp[5]), lp[:8]
        assert np.all(np.isfinite(lp[6:])), lp[6:12]
        want = h.along(h.path_rows(w64, dims, sp, xa[w], seq, kv), seq)
        assert np.array_equal(np.isneginf(want), np.isneginf(lp[4:]))
        ok = np.isfinite(want)
        err = float(np.abs(lp[4:][ok].astype(np.float64) - want[ok]).max())
        worst = max(worst, err)
        assert err < h.GREEDY_LP_TOL[kv]
    h.report(f"score_tokens masked rows d=384 kv={kv}", worst, h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 3. agreement with decoding
def close_to_decoding(sess, ids, sp, kv, masked=True, greedy=False, gaps=None):
    out = sess.score_tokens(ids, list(range(len(ids))), apply_special_mask=masked, is_special=is_special_of(sp) if masked else None)
    worst = 0.0
    for r, (t, (lp, am)) in enumerate(zip(ids, out)):
        want = sess.last_logprobs(r)[4:len(t)].astype(np.float64)
        got = lp[4:].astype(np.float64)
        ok = ~np.isnan(want)   # an EOT the greedy loop's rules appended has no log-prob
        err = float(np.abs(got[ok] - want[ok]).max(initial=0.0))
        worst = max(worst, err)
        assert err < h.GREEDY_LP_TOL[kv], f"row {r}: scored {got} vs decoded {want}"
        if greedy:
            for j in range(4, len(t)):
                if ok[j - 4] and (gaps is None or gaps[r][j] >= GAP):
                    assert am[j] == t[j], f"row {r} position {j}: arg-max {am[j]} vs decoded id {t[j]}"
    return worst


def f64_gaps(w64, dims, sess, ids, kv):
    """per row and position j >= 1 the float64 top-1 / top-2 gap of the masked row that chose ids[j]"""
    sp = synth.special_tokens(dims)
    gaps = []
    for r, t in enumerate(ids):
        xa = torch.from_numpy(sess.get_encoder_output(r)).double()[None]
        rows = h.path_rows(w64, dims, sp, xa, t, kv)
        g = np.full(len(t), np.inf)
        for j in range(4, len(t)):
            top2 = np.sort(rows[j - 4])[-2:]
            g[j] = top2[1] - top2[0]
        gaps.append(g)
    return gaps


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_scores_agree_with_decoding(kv, monkeypatch):
    for name in ("test-a", "tiny.en"):
        dims, sp, wh, _, _, w64 = h.named_model(name, f64=True)
        waves = h.pool_waves(h.golden("tokens_beam"), 4)
        sess = transcribe.Session(wh, max_windows=4, max_beams=5, max_text_len=40, kv_dtype=h.kv_code(kv))
        ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=30)
        worst = close_to_decoding(sess, ids, sp, kv, greedy=True, gaps=f64_gaps(w64, dims, sess, ids, kv))
        h.report(f"score_tokens vs greedy last_logprobs {name} kv={kv}", worst, h.GREEDY_LP_TOL[kv])
        ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=5, max_depth=30)
        assert sess.last_decoder() == 6
        worst = close_to_decoding(sess, ids, sp, kv)
        h.report(f"score_tokens vs device beam last_logprobs {name} kv={kv}", worst, h.GREEDY_LP_TOL[kv])
        h.use_decoder(monkeypatch, 3)
        hs = transcribe.Session(wh, max_windows=4, max_beams=5, max_text_len=40, kv_dtype=h.kv_code(kv))
        h.use_decoder(monkeypatch, 0)
        hids = hs.transcribe_windows(waves, sp, is_special_of(sp), beam_size=5, max_depth=30)
        assert hs.last_decoder() == 3
        worst = close_to_decoding(hs, hids, sp, kv)
        h.report(f"score_tokens vs host beam last_logprobs {name} kv={kv}", worst, h.GREEDY_LP_TOL[kv])
        hs.close()
        loop = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=40, kv_dtype=h.kv_code(kv), search="greedy_loop")
        lids = loop.transcribe_windows(waves, sp, None, beam_size=1, max_depth=30)
        lids = [t[:min(len(t), 40)] for t in lids]   # a context-stop EOT past the token buffer is not scored
        worst = close_to_decoding(loop, lids, sp, kv, masked=False)
        h.report(f"score_tokens unmasked vs greedy loop last_logprobs {name} kv={kv}", worst, h.GREEDY_LP_TOL[kv])
        loop.close()
        sess.close()


# ---------------------------------------------------------------- 4. real shapes
def check_fixture_rows(sess, sp, recs, with_lp):
    ids = [r["tokens"] for r in recs]
    out = sess.score_tokens(ids, list(range(len(ids))), apply_special_mask=True, is_special=is_special_of(sp))
    worst = 0.0
    for r, (rec, (lp, am)) in enumerate(zip(recs, out)):
        for s, t in enumerate(rec["tokens"][4:]):
            j = 4 + s
            assert am[j] == t, f"row {r} position {j}: arg-max {am[j]} vs fixture id {t}"
            if with_lp:
                top_ids, top_lp = rec["top5"][s]
                if top_lp[0] - top_lp[1] >= GAP:
                    assert am[j] == top_ids[0]
                err = abs(float(lp[j]) - top_lp[0])
                worst = max(worst, err)
                assert err < h.REAL_LP_TOL, f"row {r} position {j}: {lp[j]} vs oracle {top_lp[0]}"
    return worst


def test_real_shapes_vs_golden():
    g = h.golden("tokens_real")
    dims, w_np, _ = synth.make_weights("small.en", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    for kv in ("f32", "f16"):
        waves, recs = h.real_windows("small.en", kv)
        sess = transcribe.Session(wh, max_windows=24, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
        sess.encode_waveforms(waves)
        worst = check_fixture_rows(sess, sp, recs, with_lp=kv == "f32")
        h.report(f"score_tokens small.en 24 windows kv={kv} vs golden", worst, h.REAL_LP_TOL)
        sess.close()
    del sess, wh
    gm = g["medium"]
    dims, w_np, _ = synth.make_weights("medium", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    chunk = synth.chunk_waveform(0)
    sess = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=8)
    sess.encode_waveforms([chunk[s:e] for s, e in gm["bounds"]])
    h.report("score_tokens medium chunk 0 f32 vs golden", check_fixture_rows(sess, sp, gm["f32"], with_lp=True), h.REAL_LP_TOL)


# ---------------------------------------------------------------- 5-7. shape of the pass, state, contract
@pytest.fixture(scope="module")
def small_model():
    dims, wh, _ = h.make_model(384, 6, 2051)
    return dims, wh


def test_launch_count_and_independence(small_model):
    dims, wh = small_model
    Ts, waves = h.windows(2, seed=23)
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8)
    sess.encode_waveforms(waves)
    lib = ffi.lib()
    rng = np.random.default_rng(4)
    long = [int(t) for t in rng.integers(0, dims.n_vocab, size=448)]
    counts = []
    for seq in (long[:8], long):
        lib.wb_kernel_launch_count_reset()
        sess.score_tokens([seq], [1])
        counts.append(lib.wb_kernel_launch_count())
    assert counts[0] == counts[1] > 0, counts
    alone = sess.score_tokens([long], [1])[0][0]
    others = random_seqs(dims.n_vocab, 8, lengths=(65, 300, 3))
    batch = sess.score_tokens([others[0], long, others[1], long[:129], others[2], long[:64]], [0, 1, 1, 1, 0, 1])
    assert np.array_equal(batch[1][0], alone)
    assert np.array_equal(batch[3][0], alone[:129]) and np.array_equal(batch[5][0], alone[:64])
    assert np.array_equal(sess.score_tokens([long[:200]], [1])[0][0], alone[:200])


def test_decode_state_untouched(small_model):
    dims, wh = small_model
    sp = synth.special_tokens(dims)
    Ts, waves = h.windows(3, seed=29)
    sess = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=4 + h.DEPTH + 1)
    ids = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=h.DEPTH)
    before = ([sess.last_logprobs(r) for r in range(3)], sess.last_topk(3, 1), sess.last_decoder())
    sess.score_tokens(ids + random_seqs(dims.n_vocab, 2, lengths=(448,)), [0, 1, 2, 0], apply_special_mask=True,
                      is_special=is_special_of(sp))
    after = ([sess.last_logprobs(r) for r in range(3)], sess.last_topk(3, 1), sess.last_decoder())
    for a, b in zip(before[0], after[0]):
        assert np.array_equal(a, b, equal_nan=True)
    assert np.array_equal(before[1][0], after[1][0]) and np.array_equal(before[1][1], after[1][1])
    assert before[2] == after[2]
    assert sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=h.DEPTH) == ids


def raw_score(sess, seqs, wins, mask=0, special=None):
    lens = np.asarray([len(s) for s in seqs], dtype=np.int64)
    toks = np.asarray([t for s in seqs for t in s], dtype=np.int64)
    w = np.asarray(wins, dtype=np.int32)
    lp = np.empty(max(len(toks), 1), dtype=np.float32)
    return ffi.lib().wb_session_score_tokens(sess._h, len(lens), ffi.i32ptr(w), ffi.i64ptr(toks), ffi.i64ptr(lens), mask,
                                             None if special is None else ffi.u8ptr(special), ffi.fptr(lp), None)


def test_error_codes(small_model):
    dims, wh = small_model
    sp = synth.special_tokens(dims)
    V, n_ctx = dims.n_vocab, dims.n_text_ctx
    Ts, waves = h.windows(2, seed=31)
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8)
    assert raw_score(sess, [[1, 2]], [0]) == ffi.WB_ERR_STATE
    sess.encode_waveforms(waves)
    assert raw_score(sess, [[1, 2]], [0]) == ffi.WB_OK
    assert raw_score(sess, [[]], [0]) == ffi.WB_ERR_INVALID_ARG                       # lens 0
    assert raw_score(sess, [[1] * (n_ctx + 1)], [0]) == ffi.WB_ERR_INVALID_ARG        # lens > n_text_ctx
    assert raw_score(sess, [[1, V]], [0]) == ffi.WB_ERR_INVALID_ARG                   # token >= n_vocab
    assert raw_score(sess, [[1, -1]], [0]) == ffi.WB_ERR_INVALID_ARG                  # token < 0
    assert raw_score(sess, [[1, 2]], [2]) == ffi.WB_ERR_INVALID_ARG                   # window not encoded
    assert raw_score(sess, [[1, 2]], [-1]) == ffi.WB_ERR_INVALID_ARG
    assert raw_score(sess, [[1, 2]], [0], mask=1) == ffi.WB_ERR_INVALID_ARG           # mask without is_special
    assert raw_score(sess, [[1, 2]], [0], mask=1, special=is_special_of(sp)) == ffi.WB_OK
    sess.close()
    # the non-fp16-exact model of test_non_fp16_exact_weights_use_fp32_storage
    dims_x, w_np, _, _ = h.synthetic("test-a", 3, exact=False, f64=False)
    wx = model.Whisper(dims_x, w_np)
    assert not wx.weights_fp16_exact
    sx = transcribe.Session(wx, max_windows=1, max_beams=1, max_text_len=8)
    sx.encode_waveforms(waves[:1])
    assert raw_score(sx, [[1, 2]], [0]) == ffi.WB_ERR_UNSUPPORTED
    with pytest.raises(ffi.WbError) as e:
        sx.score_tokens([[1, 2]], [0])
    assert e.value.code == ffi.WB_ERR_UNSUPPORTED
