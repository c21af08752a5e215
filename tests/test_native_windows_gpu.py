"""Native windowing on the GPU: sessions whose windows give the encoder up to 2 * n_audio_ctx mel frames, i.e. T up to 1500
encoder positions (the reference's windowing stops at 750).

  (a) log-mel of native windows against the oracle (the suite's mel bar);
  (b) the encoder at real widths against float64, T = 1500 and ragged T > 750 in one batch, tensor-core and fp32 paths;
  (c) every persistent decoder's cross attention over T > 750 keys against float64: greedy top-1 log-probs per step and
      wb_session_step candidates (the helpers and bars of harness.py);
  (d) token ids against tests/golden/tokens_native.json (make_golden_native.py): greedy, the device and the host beam search;
  (e) long-form waveform_to_tokens (native windowing + overlap merge) against the same fixture;
  (f) a reference and a native session of one model side by side, each with its own frame limit.

The oracle's native mode is the oracle on dims with n_audio_ctx doubled: it reads n_audio_ctx only as the frame limit."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import harness as h
import wb200  # noqa: F401
from harness import is_special_of, kv_code
from oracle import audio as o_audio, model as o_model, synth, transcribe as o_tr
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu
MEL_TOL = 1e-4   # the suite's log-mel bar (test_parity_gpu.py), relative to scale


def samples_of_T(T):
    """Waveform samples whose native window has T encoder positions: F = 2T - 11 frames -> Tm = 2T - 1 (T <= 1500)."""
    return 160 * (2 * T - 11)


def native(dims):
    return dataclasses.replace(dims, n_audio_ctx=2 * dims.n_audio_ctx)


# ---------------------------------------------------------------- (a) log-mel
def test_logmel_native_windows_vs_oracle():
    dims, _, wh, *_ = h.named_model("test-a")
    lens = [480000, 478560, samples_of_T(1025), 64000]
    waves = [synth.waveform(n, seed=20 + i) for i, n in enumerate(lens)]
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8, windows="native")
    sess.encode_waveforms(waves)
    worst = 0.0
    for i, wv in enumerate(waves):
        got = sess.get_mel(i)
        want = o_tr.pad_mel(o_audio.prep_audio(torch.from_numpy(wv)[None]), 3000).numpy()[0]
        assert got.shape == want.shape == (80, min(len(wv) // 160, 2990) + 10)
        e = h.rel_to_scale(got, want)
        worst = max(worst, e)
        assert e < MEL_TOL, f"window {i}: {e}"
    h.report("native log-mel (4 windows, Tm up to 3000)", worst, MEL_TOL)


# ---------------------------------------------------------------- (b) encoder at real widths
ENC_TS = (1500, 751, 1025, 205)


@pytest.mark.parametrize("exact", [True, False], ids=["tensor-core", "fp32"])
@pytest.mark.parametrize("d,H", [(384, 6), (768, 12), (1024, 16), (1280, 20)])
def test_encoder_native_windows_vs_float64(d, H, exact):
    """Encoder output of windows with T = 1500, 751, 1025, 205 packed in one batch (conv stems over Tm up to 3000 mel rows,
    24 attention key tiles with a ragged last one), against the float64 encoder of each window's padded mel."""
    dims, wh, w64 = h.make_model(d, H, 2051, exact=exact, n_text_layer=1)
    waves = [synth.waveform(samples_of_T(T) if T != 1500 else 480000, seed=850 + d + i) for i, T in enumerate(ENC_TS)]
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8, windows="native")
    sess.encode_waveforms(waves)
    worst = h.encoder_error(sess, w64, native(dims), ENC_TS, h.ENC_REL_TOL)
    h.report(f"native encoder d={d} {'tensor-core' if exact else 'fp32'}", worst, h.ENC_REL_TOL)


# ---------------------------------------------------------------- (c) decoders over T > 750 cross keys
# T on either side of 1024 (a multiple of every key chunk and batch: decoder6's 32 / 64-key ring chunks, decoder4's 8 / 16-key
# bulk batches over 16 CTAs' warps, decoder5's and decoder3's ceil(T / S) splits), the first length past the reference's 750,
# and 1500 (ragged last chunk everywhere).  DESIGN.md section 2 lists the edges.
DEC_TS = (1500, 751, 1025, 1024)


# (decoder, d, rows, exact): decoder4 <= 7 rows, decoder6 8..24 rows, decoder5 d % 256 == 0, decoder3 (both weight types)
NATIVE_DEC_CASES = [(4, 384, 1, True), (4, 384, 4, True), (6, 384, 8, True), (6, 128, 24, True), (5, 256, 9, True),
                    (5, 768, 4, True), (3, 384, 4, True), (3, 192, 3, False)]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("decoder,d,rows,exact", NATIVE_DEC_CASES)
def test_decoder_greedy_native_T_vs_float64(decoder, d, rows, exact, kv, monkeypatch):
    dims, wh, _ = h.make_model(d, d // 64, 51864 if d == 384 else 2051, exact=exact)
    h.use_decoder(monkeypatch, decoder)
    seed = 2000 + 10 * decoder + rows
    Ts = [DEC_TS[i % len(DEC_TS)] for i in range(rows)]
    waves = [synth.waveform(480000 if T == 1500 else samples_of_T(T), seed=seed + i) for i, T in enumerate(Ts)]
    try:
        worst = h.check_greedy(dims, wh, kv, rows, decoder, seed, inputs=(Ts, waves), mode="native")
    except ffi.WbError as e:
        if decoder == 4 and rows > 1 and e.code == ffi.WB_ERR_UNSUPPORTED:
            pytest.skip(f"decoder4 does not cover {rows} rows on this GPU (co-resident 16-CTA clusters)")
        raise
    h.report(f"native decoder{decoder} d={d} rows={rows} kv={kv}", worst, h.GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("decoder,d", [(3, 384), (5, 256)])
def test_session_step_k7_native_T_vs_float64(decoder, d, kv, monkeypatch):
    """wb_session_step with k = 7 on two windows of T = 1500 and 1025: every candidate against float64 CachedDecoder rows."""
    dims, wh, w64 = h.make_model(d, d // 64, 51864 if d == 384 else 2051)
    h.use_decoder(monkeypatch, decoder)
    sp = synth.special_tokens(dims)
    bitmap = sp.is_special_bitmap()
    K = 7
    waves = [synth.waveform(480000, seed=2500), synth.waveform(samples_of_T(1025), seed=2501)]
    sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=12, kv_dtype=kv_code(kv), windows="native")
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, [1500, 1025])
    opts = o_model.OracleOptions(kv_dtype=kv)
    prompt = sp.prompt()
    sess.begin(prompt)
    ref = [o_model.CachedDecoder(w64, dims, xa[w], opts) for w in range(2)]
    for dec in ref:
        for t in prompt[:-1]:
            dec.step(torch.tensor([t], dtype=torch.int64))
    maskout = torch.from_numpy(sp.maskout())
    tol = h.STEP_LP_TOL[kv]
    worst = 0.0
    rows = [(0, 0), (1, 0)]          # GPU row -> (window, row of that window's float64 decoder)

    def step(parents, tokens, masked):
        nonlocal rows, worst
        win = [rows[p][0] for p in parents]
        ids, lps = sess.step(win, parents, tokens, masked, bitmap, K)
        assert sess.last_decoder() == decoder
        for w in range(2):
            mine = [i for i in range(len(parents)) if win[i] == w]
            ref[w].reorder([rows[parents[i]][1] for i in mine])
            logits = ref[w].step(torch.tensor([tokens[i] for i in mine], dtype=torch.int64))
            if masked:
                logits = logits + maskout
            lp = o_model.log_softmax_last(logits).numpy()
            for j, i in enumerate(mine):
                have = lp[j][ids[i]]
                err = float(np.abs(lps[i] - have).max())
                worst = max(worst, err)
                assert err < tol, f"row {i}: log-probs {lps[i]} vs float64 {have}"
                assert np.abs(have - np.sort(lp[j])[::-1][:K]).max() < tol, f"row {i}: ids out of float64 order"
        rows = [(win[i], sum(1 for q in range(i) if win[q] == win[i])) for i in range(len(parents))]
        return ids

    ids = step([0, 1], [prompt[-1]] * 2, True)
    ids = step([0, 0, 0, 1, 1, 1], [int(ids[0, j]) for j in range(3)] + [int(ids[1, j]) for j in range(3)], True)
    ids = step([2, 0, 1, 5, 3, 4], [int(ids[p, 1]) for p in (2, 0, 1, 5, 3, 4)], False)
    step([1, 2, 0, 4, 5, 3], [int(ids[p, 2]) for p in (1, 2, 0, 4, 5, 3)], False)
    h.report(f"native step k=7 decoder{decoder} d={d} kv={kv}", worst, tol)


# ---------------------------------------------------------------- (d), (e) token ids against the native fixture
def _windows(case):
    return [synth.chunk_waveform(c)[:n] for c, n in case["windows"]]


@pytest.fixture(scope="module")
def tiny_en():
    return h.named_model("tiny.en")


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_tiny_en_greedy_native_golden(tiny_en, kv):
    """One batch of T = 1500, 1500, 1005 and 205, greedy depth 100, on the default decoder."""
    dims, sp, wh, *_ = tiny_en
    g = h.golden("tokens_native")["tiny.en"]
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=105, kv_dtype=kv_code(kv), windows="native")
    got = sess.transcribe_windows(_windows(g), sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert [sess.get_encoder_output(i).shape[0] for i in range(4)] == [r["T"] for r in g[kv]] == [1500, 1500, 1005, 205]
    print(f"\n[native] tiny.en greedy kv={kv}: decoder{sess.last_decoder()}")
    h.check_ids_where_separated(got, g[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_tiny_en_device_beam_native_golden(tiny_en, kv):
    """Beam 5, depth 30, 2 windows (T = 1500, 1005): the whole search in one decoder6 launch."""
    dims, sp, wh, *_ = tiny_en
    g = h.golden("tokens_native")["tiny.en-beam"]
    sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=35, kv_dtype=kv_code(kv), windows="native")
    got = sess.transcribe_windows(_windows(g), sp, is_special_of(sp), beam_size=5, max_depth=30)
    assert sess.last_decoder() == 6
    assert got == [r["tokens"] for r in g[kv]], f"oracle min margin {g['min_margin_' + kv]}"


@pytest.fixture(scope="module")
def small_en():
    return h.named_model("small.en")


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_small_en_greedy_native_golden(small_en, kv):
    dims, sp, wh, *_ = small_en
    g = h.golden("tokens_native")["small.en"]
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=105, kv_dtype=kv_code(kv), windows="native")
    got = sess.transcribe_windows(_windows(g), sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 5
    h.check_ids_where_separated(got, g[kv])
    if kv == "f32":   # the one or two tokens these models decode carry little evidence: the 5 best log-probs of every step
        recs = g[kv]
        sess.encode_waveforms(_windows(g))
        sess.begin(sp.prompt())
        last, rows, worst = [sp.prompt()[-1]] * 2, [0, 1], 0.0
        for step in range(100):
            ids, lps = sess.step(rows, rows, last, step + 4 <= 5, is_special_of(sp) if step == 0 else None, 5)
            for r in range(2):
                want_ids, want_lp = recs[r]["top5"][step]
                worst = max(worst, float(np.abs(lps[r] - np.asarray(want_lp, np.float32)).max()))
                last[r] = recs[r]["tokens"][4 + step]
                assert int(ids[r, 0]) == last[r]
        h.report("native small.en 2 rows x 100 steps, top-5 log-probs vs oracle", worst, 2e-4)
        assert worst < 2e-4


def test_small_en_host_beam_native_golden(small_en):
    """Beam 5, depth 20, one window of T = 1500: the host search over decoder5 steps."""
    dims, sp, wh, *_ = small_en
    g = h.golden("tokens_native")["small.en-beam"]
    sess = transcribe.Session(wh, max_windows=1, max_beams=5, max_text_len=25, windows="native")
    got = sess.transcribe_windows(_windows(g), sp, is_special_of(sp), beam_size=5, max_depth=20)
    assert sess.last_decoder() == 5
    assert got == [r["tokens"] for r in g["f32"]], f"oracle min margin {g['min_margin_f32']}"


def test_tiny_en_long_form_native_golden(tiny_en):
    """waveform_to_tokens over 70 s: three native windows (T = 1500, 1500, 814) and the overlap merge."""
    dims, sp, wh, *_ = tiny_en
    g = h.golden("tokens_native")["tiny.en-long"]
    wave = np.concatenate([synth.chunk_waveform(c) for c in g["chunks"]])[:g["samples"]]
    assert transcribe.window_bounds(len(wave), 16000, transcribe.window_samples(1500, "native")) == \
        [tuple(b) for b in g["bounds"]]
    sess = transcribe.Session(wh, max_windows=3, max_beams=1, max_text_len=105, windows="native")
    assert sess.waveform_to_tokens(wave, sp, is_special_of(sp), beam_size=1, max_depth=100) == g["tokens"]


# ---------------------------------------------------------------- (f) both modes side by side
def test_reference_and_native_sessions_side_by_side(tiny_en):
    dims, sp, wh, *_ = tiny_en
    ref = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=8)
    nat = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=8, windows="native")
    wave = synth.chunk_waveform(0)
    ref.encode_waveforms([wave])
    nat.encode_waveforms([wave])
    assert ref.get_mel(0).shape == (80, 1500) and ref.get_encoder_output(0).shape == (1500 // 2, 384)
    assert nat.get_mel(0).shape == (80, 3000) and nat.get_encoder_output(0).shape == (1500, 384)
    rng = np.random.default_rng(5)
    for sess, ok, too_long in ((ref, 1500, 1501), (nat, 3000, 3001)):
        sess.encode_mels(rng.standard_normal((1, 80, ok)).astype(np.float32))
        assert sess.get_encoder_output(0).shape == ((ok - 1) // 2 + 1, 384)
        with pytest.raises(ffi.WbError) as e:
            sess.encode_mels(rng.standard_normal((1, 80, too_long)).astype(np.float32))
        assert e.value.code == ffi.WB_ERR_INVALID_ARG
    h = C.c_void_p()
    assert ffi.lib().wb_session_create_windows(wh.handle, 1, 1, 8, ffi.WB_KV_F32, 2, C.byref(h)) == ffi.WB_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        transcribe.Session(wh, max_windows=1, windows="30s")
