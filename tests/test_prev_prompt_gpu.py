"""GPU tests (-m gpu) of the previous-text prompt (wb_transcribe_windows_prev, wb_session_set_prev_prompt): windows whose
prompts differ in length share one decoder launch, each row committing from its own prompt's last position on.

  1. a ragged batch (previous-id lists of 0, 1, 5 and a long one past a self-attention key-count edge) on decoder3 / 4 / 5 /
     6 with fp32 and fp16 K/V: every row starts with its prompt, stops at EOT or at exactly Lp + max_depth ids, and its
     log-probs match float64 teacher forcing of the GPU's own path (greedy_path_log_probs with n_prompt = Lp);
  2. all-empty previous lists give bit-identical ids and log-probs to wb_transcribe_windows (greedy and beam);
  3. each window of a ragged batch decodes to the same ids alone;
  4. the returned log-probs match wb_session_score_tokens with the special-id mask on the returned rows;
  5. beam search with ragged prompts: the device search (decoder6), the host search (decoder3 / decoder5) and the oracle give
     the same ids;
  6. the waveform rule of waveform(s)_to_tokens against the oracle restatement (tests/oracle_prev_prompt.py), and batched
     waveforms against each waveform alone;
  7. every error case of the two entry points."""
from ctypes import byref as C_byref, c_int64 as C_int64

import numpy as np
import pytest
import torch

import harness as h
import oracle_prev_prompt as opp
import wb200  # noqa: F401
from oracle import audio as o_audio, synth, transcribe as o_tr
from whisper_burn_b200 import ffi, model, transcribe

pytestmark = pytest.mark.gpu
DEPTH = h.DEPTH


def prev_lists(sp, n, long_len, seed):
    """n previous-id lists of lengths 0, 1, 5, long_len, 0, 1, ... of non-special ids"""
    rng = np.random.default_rng(seed)
    lens = [(0, 1, 5, long_len)[i % 4] for i in range(n)]
    return [[int(t) for t in rng.integers(0, sp.first_special, size=k)] for k in lens]


# (decoder, d, heads, rows, long previous list): the long list crosses decoder6's 32-key slot, and the 128-key turn elsewhere
RAGGED_CASES = [(4, 384, 6, 4, 130), (6, 384, 6, 9, 40), (6, 128, 2, 8, 40), (5, 256, 4, 9, 130), (3, 384, 6, 4, 130)]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("decoder,d,H,rows,long_len", RAGGED_CASES)
def test_ragged_greedy_vs_float64(decoder, d, H, rows, long_len, kv, monkeypatch):
    dims, wh, w64 = h.make_model(d, H, 2051)
    sp = synth.special_tokens(dims)
    _, waves = h.windows(rows, seed=7 * d + rows)
    prev = prev_lists(sp, rows, long_len, seed=d + rows)
    t_max = long_len + 5 + DEPTH + 1
    h.use_decoder(monkeypatch, decoder)
    sess = transcribe.Session(wh, max_windows=rows, max_beams=1, max_text_len=t_max, kv_dtype=h.kv_code(kv))
    h.use_decoder(monkeypatch, 0)
    ids = sess.transcribe_windows_prev(waves, prev, sp, sp.is_special_bitmap(), beam_size=1, max_depth=DEPTH)
    assert sess.last_decoder() == decoder
    worst = 0.0
    for r, t in enumerate(ids):
        prompt = opp.build_prompt(sp, prev[r])
        lp0 = len(prompt)
        assert t[:lp0] == prompt, f"row {r}"
        assert len(t) == lp0 + DEPTH or (t[-1] == sp.eot and len(t) < lp0 + DEPTH), f"row {r}: {len(t)} ids, prompt {lp0}"
        lps = sess.last_logprobs(r)
        assert len(lps) == len(t) and np.all(lps[:lp0] == 0.0)
        xa = torch.from_numpy(sess.get_encoder_output(r)).double()[None]
        ref = h.along(h.path_rows(w64, dims, opp.oracle_special(sp), xa, t, kv, n_prompt=lp0), t, lp0)
        err = float(np.abs(lps[lp0:].astype(np.float64) - ref).max(initial=0.0))
        worst = max(worst, err)
        assert err < h.GREEDY_LP_TOL[kv], f"row {r}: {lps[lp0:]} vs float64 {ref}"
    h.report(f"prev prompt ragged greedy decoder{decoder} d={d} rows={rows} kv={kv}", worst, h.GREEDY_LP_TOL[kv])


def test_deep_rows_stop_at_their_own_length(monkeypatch):
    """EOT declared as an id no row emits: every row runs to exactly Lp + max_depth ids on every greedy decoder."""
    dims, wh, _ = h.make_model(384, 6, 2051)
    sp0 = synth.special_tokens(dims)
    sp = synth.SpecialTokens(sot=sp0.sot, lang=sp0.lang, transcribe=sp0.transcribe, notimestamps=sp0.notimestamps,
                             eot=sp0.n_vocab - 1, first_special=sp0.first_special, n_vocab=sp0.n_vocab, startofprev=sp0.startofprev)
    _, waves = h.windows(4, seed=5)
    prev = prev_lists(sp, 4, 40, seed=3)
    for decoder in (4, 6, 3):
        h.use_decoder(monkeypatch, decoder)
        sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=45 + DEPTH + 1)
        h.use_decoder(monkeypatch, 0)
        ids = sess.transcribe_windows_prev(waves, prev, sp, sp.is_special_bitmap(), beam_size=1, max_depth=DEPTH)
        assert sess.last_decoder() == decoder
        if any(sp.eot in t for t in ids):
            pytest.skip("a row emitted the stand-in EOT")
        assert [len(t) for t in ids] == [len(opp.build_prompt(sp, p)) + DEPTH for p in prev], f"decoder{decoder}"
        sess.close()


@pytest.mark.parametrize("beam_size", [1, 3])
def test_empty_prev_is_bit_identical(beam_size):
    dims, _, wh, *_ = h.named_model("test-a")
    sp = synth.special_tokens(dims)
    waves = [synth.waveform(48000, seed=40 + i) for i in range(4)]
    sess = transcribe.Session(wh, max_windows=4, max_beams=beam_size, max_text_len=4 + 20 + 1)
    a = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=beam_size, max_depth=20)
    la = [sess.last_logprobs(r) for r in range(4)]
    b = sess.transcribe_windows_prev(waves, [[]] * 4, sp, sp.is_special_bitmap(), beam_size=beam_size, max_depth=20)
    lb = [sess.last_logprobs(r) for r in range(4)]
    assert a == b
    for x, y in zip(la, lb):
        assert np.array_equal(x, y)


def test_ragged_batch_equals_each_window_alone_and_scoring():
    dims, _, wh, *_ = h.named_model("test-a")
    sp = synth.special_tokens(dims)
    waves = [synth.waveform(48000, seed=60 + i) for i in range(6)]
    prev = prev_lists(sp, 6, 12, seed=9)
    sess = transcribe.Session(wh, max_windows=6, max_beams=1, max_text_len=17 + 30 + 1)
    ids = sess.transcribe_windows_prev(waves, prev, sp, sp.is_special_bitmap(), beam_size=1, max_depth=30)
    lps = [sess.last_logprobs(r) for r in range(6)]
    for r in range(6):
        one = sess.transcribe_windows_prev([waves[r]], [prev[r]], sp, sp.is_special_bitmap(), beam_size=1, max_depth=30)
        assert one[0] == ids[r], f"window {r}"
        assert np.abs(sess.last_logprobs(0) - lps[r]).max() < 1e-5
    sess.encode_waveforms(waves)
    scored = sess.score_tokens(ids, list(range(6)), apply_special_mask=True, is_special=sp.is_special_bitmap())
    for r, (lp, _) in enumerate(scored):
        lp0 = len(opp.build_prompt(sp, prev[r]))
        assert np.abs(lp[lp0:] - lps[r][lp0:]).max(initial=0.0) < 2e-5, f"window {r}"


def oracle_rows(w_t, dims, sp, waves, prev, beam_size, max_depth):
    out = []
    for wv, p in zip(waves, prev):
        mel = o_audio.prep_audio(torch.from_numpy(wv)[None])
        out.append(opp.mels_to_tokens(w_t, dims, sp, mel, opp.build_prompt(sp, p), beam_size, max_depth))
    return out


@pytest.mark.parametrize("name,host_decoder", [("test-a", 3), ("tiny.en", 3), ("test-d", 5)])
def test_ragged_beam_device_host_oracle(name, host_decoder, monkeypatch):
    dims, _, wh, _, w_t, _ = h.named_model(name)
    sp = synth.special_tokens(dims)
    n = 4
    waves = [synth.waveform(48000, seed=80 + i) for i in range(n)]
    prev = prev_lists(sp, n, 9, seed=21)
    depth, beam_size = 12, 3
    want = oracle_rows(w_t, dims, sp, waves, prev, beam_size, depth)
    runs = []
    for dec in ((6, host_decoder) if dims.n_text_state in (128, 384) else (host_decoder,)):
        h.use_decoder(monkeypatch, dec)
        sess = transcribe.Session(wh, max_windows=n, max_beams=beam_size, max_text_len=14 + depth + 1)
        h.use_decoder(monkeypatch, 0)
        got = sess.transcribe_windows_prev(waves, prev, sp, sp.is_special_bitmap(), beam_size=beam_size, max_depth=depth)
        assert sess.last_decoder() == dec
        for r, t in enumerate(got):
            lp = sess.last_logprobs(r)
            assert np.all(lp[:len(opp.build_prompt(sp, prev[r]))] == 0.0)
        runs.append(got)
        sess.close()
    for got in runs:
        assert got == want


def test_waveform_rule_vs_oracle_and_batched():
    dims, _, wh, _, w_t, _ = h.named_model("test-a")
    sp = synth.special_tokens(dims)
    win = o_audio.max_waveform_samples(dims.n_audio_ctx - 10)
    shift = win - 3 * 16000
    lens = [win // 2, win + 2 * shift - 100, win + 5 * shift - 100]   # 1, 3 and 6 windows
    waves = [synth.waveform(n, seed=100 + i) for i, n in enumerate(lens)]
    depth = 16
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=10 + depth + 1)
    sess.set_prev_prompt(sp.startofprev)
    alone = []
    for wv in waves:
        per = []
        want = opp.waveform_to_tokens(w_t, dims, sp, wv, 1, depth, per_window=per)
        got = sess.waveform_to_tokens(wv, sp, sp.is_special_bitmap(), beam_size=1, max_depth=depth)
        assert got == want
        assert np.all(sess.last_logprobs(0)[:4] == 0.0)
        alone.append((got, sess.last_logprobs(0)))
        assert all(len(p) > 4 for p, _ in per[1:])   # every later window is prompted with earlier text
    batched = sess.waveforms_to_tokens(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=depth)
    for i, (got, lp) in enumerate(alone):
        assert batched[i] == got
        assert np.abs(sess.last_logprobs(i) - lp).max() < 1e-5
    sess.set_prev_prompt(-1)
    assert sess.waveform_to_tokens(waves[1], sp, sp.is_special_bitmap(), beam_size=1, max_depth=depth) == \
        o_tr.waveform_to_tokens(w_t, dims, opp.oracle_special(sp), waves[1], beam_size=1, max_depth=depth)


def test_errors():
    dims, _, wh, *_ = h.named_model("test-a")
    sp = synth.special_tokens(dims)
    waves = [synth.waveform(48000, seed=1)]
    sess = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=12 + 8 + 1)
    bm = sp.is_special_bitmap()

    def call(prev, startofprev=None, max_depth=8, cap=None, is_special=bm):
        ws = [np.ascontiguousarray(w, dtype=np.float32) for w in waves]
        ptrs = (ffi._F * 1)(*[ffi.fptr(w) for w in ws])
        lens = np.asarray([len(ws[0])], dtype=np.int64)
        pl = np.asarray([len(prev)], dtype=np.int64) if not isinstance(prev, int) else np.asarray([prev], dtype=np.int64)
        pt = np.asarray(list(prev) if not isinstance(prev, int) else [0], dtype=np.int64)
        pt = np.concatenate([pt, [0]]).astype(np.int64)
        lp0 = (len(prev) + 5) if (not isinstance(prev, int) and len(prev)) else 4
        cap = lp0 + max_depth + 1 if cap is None else cap
        out = np.zeros(cap, dtype=np.int64)
        out_len = np.zeros(1, dtype=np.int64)
        ids = ffi.SpecialIds(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, sp.eot)
        sop = sp.startofprev if startofprev is None else startofprev
        sp_ptr = None if is_special is None else ffi.u8ptr(is_special)
        return ffi.lib().wb_transcribe_windows_prev(sess._h, ptrs, ffi.i64ptr(lens), 1, ffi.i64ptr(pt), ffi.i64ptr(pl), sop, 1,
                                                    max_depth, C_byref(ids), sp_ptr, ffi.i64ptr(out), cap, ffi.i64ptr(out_len))

    bad = ffi.WB_ERR_INVALID_ARG
    assert call([1, 2, 3]) == 0
    assert call([1, 2], startofprev=dims.n_vocab) == bad
    assert call([1, 2], startofprev=-1) == bad
    assert call([1, dims.n_vocab]) == bad
    assert call([1, -1]) == bad
    assert call(-1) == bad
    assert call([1, 2, 3], max_depth=14) == bad             # 8 + 14 > max_text_len
    assert call([1, 2, 3], cap=8 + 8) == bad                # capacity < Lp + max_depth + 1
    ffi.check(ffi.lib().wb_session_set_search(sess._h, ffi.WB_SEARCH_GREEDY_LOOP))
    assert call([1, 2]) == bad
    assert call([]) == 0
    sess.set_prev_prompt(sp.startofprev)
    assert ffi.lib().wb_waveform_to_tokens(sess._h, ffi.fptr(np.ascontiguousarray(waves[0], dtype=np.float32)), len(waves[0]), 16000, 1, 8,
                                           C_byref(ffi.SpecialIds(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, sp.eot)),
                                           ffi.u8ptr(bm), ffi.i64ptr(np.zeros(64, np.int64)), 64,
                                           C_byref(C_int64(0))) == bad
    ffi.check(ffi.lib().wb_session_set_search(sess._h, ffi.WB_SEARCH_BEAM))
    assert ffi.lib().wb_waveform_to_tokens(sess._h, ffi.fptr(np.ascontiguousarray(waves[0], dtype=np.float32)), len(waves[0]), 16000, 1, 8,
                                           C_byref(ffi.SpecialIds(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, sp.eot)),
                                           None, ffi.i64ptr(np.zeros(64, np.int64)), 64, C_byref(C_int64(0))) == bad
    assert ffi.lib().wb_session_set_prev_prompt(sess._h, dims.n_vocab) == bad
    assert ffi.lib().wb_session_set_prev_prompt(sess._h, -2) == bad
    assert ffi.lib().wb_session_set_prev_prompt(sess._h, -1) == 0



# ---------------------------------------------------------------- real shapes against tests/golden/tokens_prev_prompt.json
TIE_TOL = 1e-4  # ids are compared up to the first step whose oracle top-1/top-2 gap is below this


def _prefix_until_tie(rec):
    lp0 = len(rec["prompt"])
    if "margins" not in rec:
        return len(rec["tokens"])
    return next((lp0 + s for s, v in enumerate(rec["margins"]) if v < TIE_TOL), len(rec["tokens"]))


def _check_windows(sess, got, recs, beam):
    for i, (g, r) in enumerate(zip(got, recs)):
        n = _prefix_until_tie(r)
        assert g[:n] == r["tokens"][:n], f"window {i}"
        lps = sess.last_logprobs(i)
        lp0 = len(r["prompt"])
        assert np.all(lps[:lp0] == 0.0)
        if beam == 1:
            m = min(n, len(g)) - lp0
            err = np.abs(lps[lp0:lp0 + m] - np.asarray(r["lps"][:m], dtype=np.float32)).max(initial=0.0)
            assert err < h.REAL_LP_TOL, f"window {i}: log-prob error {err}"


@pytest.mark.parametrize("case", ["tiny.en-f32", "tiny.en-f16", "tiny.en-beam", "small.en-f32", "small.en-f16", "small.en-beam",
                                  "tiny.en-native", "ragged"])
def test_real_shapes_vs_golden(case):
    """Every window decoded from the fixture's prompt (one ragged batch per case), ids up to the first near tie and
    log-probs within harness.REAL_LP_TOL; for the waveform-rule cases without a near tie also the merged ids of waveform_to_tokens."""
    g = h.golden("tokens_prev_prompt")[case]
    dims, w_np, _ = synth.make_weights(g["model"], seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    recs = g["windows"]
    if case == "ragged":
        waves = [synth.chunk_waveform(r["chunk"])[r["bounds"][0]:r["bounds"][1]] for r in recs]
        wave = None
    else:
        wave = synth.waveform(1120000, seed=2024, kind="mix") if g["waveform"] == "long" else synth.chunk_waveform(0)
        waves = [wave[r["bounds"][0]:r["bounds"][1]] for r in recs]
    prev = [r["prompt"][1:-4] if len(r["prompt"]) > 4 else [] for r in recs]
    sess = transcribe.Session(wh, max_windows=len(recs), max_beams=max(g["beam"], 1),
                              max_text_len=max(len(r["prompt"]) for r in recs) + g["depth"] + 1,
                              kv_dtype=h.kv_code(g["kv"]), windows="native" if g.get("native") else "reference")
    got = sess.transcribe_windows_prev(waves, prev, sp, sp.is_special_bitmap(), beam_size=g["beam"], max_depth=g["depth"])
    _check_windows(sess, got, recs, g["beam"])
    if wave is not None and all(_prefix_until_tie(r) == len(r["tokens"]) for r in recs):
        sess.set_prev_prompt(sp.startofprev)
        merged = sess.waveform_to_tokens(wave, sp, sp.is_special_bitmap(), beam_size=g["beam"], max_depth=g["depth"])
        assert merged == g["merged"]
