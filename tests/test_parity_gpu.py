"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on
the same seeded inputs and against the committed golden fixtures.

Bars (north_star): log-mel within 1e-4 relative -- measured as max|a-b| / max|ref| (relative to the
tensor's scale; element-wise relative error is reported too, with an absolute floor, because bins at
the f32 rounding-noise floor differ between ANY two f32 DFT implementations, SURVEY section 7);
decoded token ids identical under greedy (and under beam 5)."""
import numpy as np
import pytest
import torch

import harness as h
import wb200  # noqa: F401
from harness import G, is_special_of, kv_code, rel_to_scale
from oracle import audio as o_audio, model as o_model, synth, transcribe as o_tr
from whisper_burn_b200 import audio, ffi, model, transcribe

pytestmark = pytest.mark.gpu
MEL_TOL = 1e-4


@pytest.fixture(scope="module")
def small():
    return h.named_model("test-a")


@pytest.fixture(scope="module")
def tiny():
    return h.named_model("tiny.en")


@pytest.fixture(scope="module")
def wide():
    """d = 256: the configuration class the batched tensor-core decoder (decoder5.cu) covers (small.en / medium / large)."""
    return h.named_model("test-c")


# ---------------------------------------------------------------- log-mel (audio.rs)
@pytest.mark.parametrize("n,kind", [(400, "noise"), (401, "mix"), (559, "mix"), (16000, "chirp"), (16000, "mix"),
                                    (4000, "click"), (98882, "mix"), (238559, "mix"), (480000, "mix")])
def test_prep_audio_vs_oracle(n, kind):
    w = synth.waveform(n, seed=11, kind=kind)
    got = audio.prep_audio(w[None])
    want = o_audio.prep_audio(torch.from_numpy(w)[None]).numpy()
    assert got.shape == want.shape == (1, 80, n // 160)
    assert rel_to_scale(got, want) < MEL_TOL
    ew = np.abs(got - want) / np.maximum(np.abs(want), 0.05)      # element-wise, 0.05 absolute floor
    assert ew.max() < 2e-3, "element-wise relative error (reported metric)"


def test_prep_audio_silence_and_batch_global_max():
    z = np.zeros((1, 3200), np.float32)
    got = audio.prep_audio(z)
    assert np.array_equal(got, o_audio.prep_audio(torch.from_numpy(z)).numpy())     # log10(1e-10) path, all equal
    w = np.stack([synth.waveform(16000, seed=1), 0.01 * synth.waveform(16000, seed=2)])
    got = audio.prep_audio(w)                                                         # ONE max over the call (audio.rs:50)
    assert rel_to_scale(got, o_audio.prep_audio(torch.from_numpy(w)).numpy()) < MEL_TOL


def test_prep_audio_golden_and_errors():
    z = np.load(G / "mel_golden.npz")
    for key in z.files:
        n, kind, seed, stride = key.split("_")
        w = synth.waveform(int(n), seed=int(seed), kind=kind)
        got = audio.prep_audio(w[None])[0][:, ::int(stride)]
        assert rel_to_scale(got, z[key]) < MEL_TOL, key
    with pytest.raises(ffi.WbError) as e:
        audio.prep_audio(np.zeros((1, 399), np.float32))                             # audio.rs:292 panics
    assert e.value.code == ffi.WB_ERR_INVALID_ARG


def test_prep_audio_scale_property_full_size():
    """Size-independent property at the full 30 s size: scaling the waveform by 1/4 shifts every
    log-mel value by log10(1/16)/4 (power scales by 1/16; the max-8 clamp floor shifts with the max)."""
    w = synth.chunk_waveform(3) * 0.5
    a = audio.prep_audio(w[None])
    b = audio.prep_audio((w * 0.25)[None])
    assert a.shape == (1, 80, 3000)
    assert np.abs((a - b) - np.log10(16.0) / 4.0).max() < 2e-6


# ---------------------------------------------------------------- encoder / decoder (mod.rs)
@pytest.mark.parametrize("n_ctx", [1, 2, 301, 628, 1500])
def test_forward_encoder_vs_oracle(small, n_ctx):
    dims, _, wh, _, w_t, _ = small
    mel = torch.from_numpy(np.random.default_rng(n_ctx).standard_normal((2, 80, n_ctx)).astype(np.float32) * 0.5)
    got = wh.forward_encoder(mel.numpy())
    want = o_model.forward_encoder(w_t, dims, mel).numpy()
    assert got.shape == want.shape == (2, (n_ctx - 1) // 2 + 1, dims.n_audio_state)
    assert rel_to_scale(got, want) < 2e-5


def test_forward_encoder_contract_violations(small):
    dims, _, wh, *_ = small
    for shape in ((1, 80, 1501), (1, 81, 100)):                                      # mod.rs:231-241 asserts
        with pytest.raises(ffi.WbError) as e:
            wh.forward_encoder(np.zeros(shape, np.float32))
        assert e.value.code == ffi.WB_ERR_INVALID_ARG


def test_forward_decoder_stateless_vs_oracle(small):
    dims, sp, wh, _, w_t, _ = small
    rng = np.random.default_rng(0)
    xa = rng.standard_normal((3, 50, dims.n_audio_state)).astype(np.float32)
    toks = rng.integers(0, dims.n_vocab, size=(3, 9)).astype(np.int64)
    got = wh.forward_decoder(toks, xa)
    want = o_model.forward_decoder(w_t, dims, torch.from_numpy(toks), torch.from_numpy(xa)).numpy()
    assert got.shape == want.shape == (3, 9, dims.n_vocab)
    assert rel_to_scale(got, want) < 2e-5
    with pytest.raises(ffi.WbError) as e:
        wh.forward_decoder(np.zeros((1, dims.n_text_ctx + 1), np.int64), xa[:1])     # mod.rs:134-139
    assert e.value.code == ffi.WB_ERR_INVALID_ARG


def test_encoder_golden_tiny_en(tiny):
    dims, _, wh, *_ = tiny
    z = np.load(G / "encoder_golden.npz")
    chunk = synth.chunk_waveform(0)
    sess = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=8)
    sess.encode_waveforms([chunk[381118:480000]])
    enc = sess.get_encoder_output(0)
    assert enc.shape == (314, 384)                                                    # SURVEY F6: 628 mel frames -> 314
    assert rel_to_scale(enc[::16], z["tiny_en_enc_w2"]) < 2e-5
    mel = sess.get_mel(0)
    assert mel.shape == (80, 628) and np.all(mel[:, 618:] == 0.0)                     # 10 zero frames (transcribe.rs:171-177)


def test_layernorm_eps_mode_inside(small):
    dims, _, _, w_np, w_t, _ = small
    wh = model.Whisper(dims, w_np, ln_eps_outside=False)
    mel = torch.from_numpy(np.random.default_rng(5).standard_normal((1, 80, 200)).astype(np.float32) * 0.5)
    want = o_model.forward_encoder(w_t, dims, mel, o_model.OracleOptions("inside")).numpy()
    assert rel_to_scale(wh.forward_encoder(mel.numpy()), want) < 2e-5


def test_non_fp16_exact_weights_use_fp32_storage():
    dims, w_np, w_t, _ = h.synthetic("test-a", 3, exact=False, f64=False)    # no longer fp16-representable
    wh = model.Whisper(dims, w_np)
    assert not wh.weights_fp16_exact
    sp = synth.special_tokens(dims)
    wave = synth.waveform(40000, seed=4)
    sess = transcribe.Session(wh, 1, 1, 4 + 16 + 1)
    got = sess.transcribe_windows([wave], sp, is_special_of(sp), beam_size=1, max_depth=16)[0]
    want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(wave)[None]), beam_size=1, max_depth=16)
    assert got == want


# ---------------------------------------------------------------- decoding (transcribe.rs + beam.rs)
@pytest.mark.parametrize("beam_size,depth", [(1, 30), (5, 12)])
def test_tokens_small_model_vs_oracle_and_golden(small, beam_size, depth):
    dims, sp, wh, _, w_t, _ = small
    ta = h.golden("tokens_test_a")
    chunk = synth.chunk_waveform(0)
    waves = [chunk[:238559], chunk[:98882]]
    sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=4 + depth + 1)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=beam_size, max_depth=depth)
    for name, g, wv in zip(("w238559", "w98882"), got, waves):
        assert g == ta["cases"][f"{name}_beam{beam_size}_depth{depth}"]["tokens"]
        live = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(wv)[None]), beam_size=beam_size, max_depth=depth)
        assert g == live
    # batching invariance: one window at a time gives the same ids
    solo = transcribe.Session(wh, max_windows=1, max_beams=5, max_text_len=4 + depth + 1)
    assert solo.transcribe_windows(waves[1:], sp, is_special_of(sp), beam_size=beam_size, max_depth=depth)[0] == got[1]


@pytest.mark.parametrize("key,beam_size", [("eot_case", 1), ("eot_case_beam5", 5)])
def test_eot_stops_search(small, key, beam_size):
    dims, sp, wh, *_ = small
    ta = h.golden("tokens_test_a")
    e = ta[key]
    sp2 = o_tr.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, e["eot"], sp.first_special, sp.n_vocab)
    sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=4 + 30 + 1)
    chunk = synth.chunk_waveform(0)
    got = sess.transcribe_windows([chunk[:238559], chunk[:98882]], sp2, is_special_of(sp), beam_size=beam_size, max_depth=30)
    assert got[0] == e["tokens"]                       # the other window keeps going / stops on its own


def test_session_step_api_matches_forward_decoder(small):
    """wb_session_step (cached, top-k) against the stateless wb_forward_decoder + host log_softmax."""
    dims, sp, wh, _, w_t, _ = small
    wave = synth.waveform(60000, seed=9)
    sess = transcribe.Session(wh, max_windows=1, max_beams=3, max_text_len=16)
    sess.encode_waveforms([wave])
    enc = sess.get_encoder_output(0)[None]
    prompt = sp.prompt()
    sess.begin(prompt)
    ids, lps = sess.step([0], [0], [prompt[-1]], True, is_special_of(sp), 3)
    logits = wh.forward_decoder(np.asarray([prompt], np.int64), enc)[0, -1]
    logits = torch.from_numpy(logits) + torch.from_numpy(sp.maskout())
    lp = o_model.log_softmax_last(logits[None])[0].numpy()
    order = np.lexsort((np.arange(len(lp)), -lp))[:3]
    assert list(ids[0]) == [int(i) for i in order]
    assert np.abs(lps[0] - lp[order]).max() < 1e-5
    # fan out to 3 beams from row 0, then continue two of them from different parents
    ids2, _ = sess.step([0, 0, 0], [0, 0, 0], list(ids[0]), True, None, 2)
    ids3, lps3 = sess.step([0, 0], [2, 0], [int(ids2[2, 0]), int(ids2[0, 1])], False, None, 2)
    for r, (par, t2) in enumerate(((2, int(ids2[2, 0])), (0, int(ids2[0, 1])))):
        seq = prompt + [int(ids[0, par]), t2]
        lg = wh.forward_decoder(np.asarray([seq], np.int64), enc)[0, -1]
        lp = o_model.log_softmax_last(torch.from_numpy(lg)[None])[0].numpy()
        assert int(ids3[r, 0]) == int(np.argmax(lp)) and abs(float(lps3[r, 0]) - float(lp.max())) < 1e-5


def test_tiny_en_chunk_greedy_golden(tiny):
    """BASELINE config 2: tiny.en, one 30 s chunk (3 reference windows), greedy to depth 100."""
    dims, sp, wh, *_ = tiny
    te = h.golden("tokens_tiny_en")
    chunk = synth.chunk_waveform(0)
    sess = transcribe.Session(wh, max_windows=3, max_beams=5, max_text_len=105)
    waves = [chunk[s:e] for s, e in te["bounds"]]
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert sess.last_decoder() == 4      # <= 7 rows: cluster / DSMEM decoder (decoder4.cu)
    assert got == te["windows"], f"min oracle margin {te['min_margin']}"
    merged = sess.waveform_to_tokens(chunk, sp, is_special_of(sp), beam_size=1, max_depth=100)
    assert merged == te["merged"]
    b5 = sess.transcribe_windows(waves[2:], sp, is_special_of(sp), beam_size=5, max_depth=30)[0]
    assert b5 == te["window2_beam5_depth30"]


def test_greedy_equals_beam1_host_path_full_size(tiny):
    """Property at full size: the on-device greedy loop and the host beam search driven through
    wb_session_step with k = 1 are two code paths for the same search (beam.rs with beam_size 1)."""
    dims, sp, wh, *_ = tiny
    chunk = synth.chunk_waveform(5)
    wave = chunk[:238559]
    sess = transcribe.Session(wh, max_windows=1, max_beams=2, max_text_len=105)
    greedy = sess.transcribe_windows([wave], sp, is_special_of(sp), beam_size=1, max_depth=100)[0]
    sess.encode_waveforms([wave])
    sess.begin(sp.prompt())
    seq = sp.prompt()
    for step in range(100):
        ids, _ = sess.step([0], [0], [seq[-1]], len(seq) <= 5, is_special_of(sp) if step == 0 else None, 1)
        seq = seq + [int(ids[0, 0])]
    assert seq == greedy


@pytest.mark.parametrize("beam_size,depth", [(1, 30), (5, 10)])
def test_fp16_kv_cache_matches_oracle_f16_mode(small, beam_size, depth):
    """WB_KV_F16 (the north star's persistent fp16 K/V cache): scaled keys and values are rounded to fp16 where
    they enter the cache; the oracle restates exactly that rounding (OracleOptions.kv_dtype = "f16")."""
    dims, sp, wh, _, w_t, _ = small
    chunk = synth.chunk_waveform(0)
    waves = [chunk[:238559], chunk[:98882]]
    sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=4 + depth + 1, kv_dtype=ffi.WB_KV_F16)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=beam_size, max_depth=depth)
    opts = o_model.OracleOptions(kv_dtype="f16")
    for g, wv in zip(got, waves):
        want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(wv)[None]), beam_size=beam_size,
                                   max_depth=depth, opts=opts)
        assert g == want


def test_npy_tree_round_trip(small, tmp_path):
    """wb_model_load_npy_tree (load::load_whisper, src/model/load.rs:295-310) == tensors set one by one."""
    from whisper_burn_b200 import npytree
    dims, sp, wh, w_np, *_ = small
    npytree.save_npy_tree(tmp_path, dims, w_np)
    wh2 = model.Whisper.from_npy_tree(tmp_path)
    assert wh2.config == dims and wh2.weights_fp16_exact
    mel = np.random.default_rng(3).standard_normal((1, 80, 200)).astype(np.float32) * 0.5
    assert np.array_equal(wh.forward_encoder(mel), wh2.forward_encoder(mel))
    wave = synth.waveform(40000, seed=2)
    a = transcribe.Session(wh, 1, 1, 24).transcribe_windows([wave], sp, is_special_of(sp), beam_size=1, max_depth=16)
    b = transcribe.Session(wh2, 1, 1, 24).transcribe_windows([wave], sp, is_special_of(sp), beam_size=1, max_depth=16)
    assert a == b


def test_batched_waveforms_equal_one_by_one(small):
    """wb_waveforms_to_tokens (all windows in one batch) == wb_waveform_to_tokens per waveform (transcribe.rs:23-74)."""
    dims, sp, wh, *_ = small
    waves = [synth.waveform(60000 + 9000 * i, seed=20 + i) for i in range(3)]
    sess = transcribe.Session(wh, 4, 1, 24)
    one = [sess.waveform_to_tokens(w, sp, is_special_of(sp), 16000, 1, 12) for w in waves]
    assert sess.waveforms_to_tokens(waves, sp, is_special_of(sp), 16000, 1, 12) == one


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_batched_tensor_core_decoder_greedy_vs_oracle(wide, kv):
    """decoder5.cu (mma.sync swap-AB, hi/lo fp16 split of the activations): 10 windows decoded in one batch,
    token ids identical to the oracle's per-window greedy search (transcribe.rs:148-383)."""
    dims, sp, wh, _, w_t, _ = wide
    waves = [synth.waveform(30000 + 7000 * i, seed=40 + i) for i in range(10)]
    sess = transcribe.Session(wh, max_windows=10, max_beams=1, max_text_len=4 + 14 + 1,
                              kv_dtype=kv_code(kv))
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=14)
    assert sess.last_decoder() == 5
    assert got == h.golden("tokens_wide")[f"test-c_greedy_depth14_{kv}"]      # committed oracle ids
    opts = o_model.OracleOptions(kv_dtype=kv)
    for g, wv in zip(got, waves):
        want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(wv)[None]), beam_size=1, max_depth=14, opts=opts)
        assert g == want
    # batching invariance across decoders: one window alone takes the same path with a single n-tile
    solo = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=4 + 14 + 1, kv_dtype=kv_code(kv))
    assert solo.transcribe_windows(waves[3:4], sp, is_special_of(sp), beam_size=1, max_depth=14)[0] == got[3]


def test_batched_tensor_core_decoder_unsplit_cross_attention():
    """20 rows x 8 heads >= one (row, head) unit per SM: decoder5.cu runs cross attention unsplit (S = 1) and writes its output
    directly as tensor-core planes -- the configuration class of the small.en / medium batches in BASELINE.json."""
    dims, sp, wh, _, w_t, _ = h.named_model("test-d")
    waves = [synth.waveform(24000 + 3000 * i, seed=80 + i) for i in range(20)]
    sess = transcribe.Session(wh, max_windows=20, max_beams=1, max_text_len=4 + 6 + 1)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=6)
    assert sess.last_decoder() == 5
    gold = h.golden("tokens_wide")["test-d_greedy_depth6_f32"]
    assert all(got[int(i)] == t for i, t in gold.items())
    for i in (0, 7, 13, 19):
        want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(waves[i])[None]), beam_size=1, max_depth=6)
        assert got[i] == want


def test_batched_tensor_core_decoder_small_en_width():
    """d = 768: decoder5.cu splits MLP2 (K = 4d) into 3 slabs of 1024 columns (fewer rounds of tiles than 4 slabs)."""
    dims, sp, wh, _, w_t, _ = h.named_model("test-e")
    waves = [synth.waveform(20000 + 2500 * i, seed=120 + i) for i in range(9)]
    sess = transcribe.Session(wh, max_windows=9, max_beams=1, max_text_len=4 + 6 + 1)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=1, max_depth=6)
    assert sess.last_decoder() == 5
    gold = h.golden("tokens_wide")["test-e_greedy_depth6_f32"]
    assert all(got[int(i)] == t for i, t in gold.items())
    for i in (0, 4, 8):
        want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(waves[i])[None]), beam_size=1, max_depth=6)
        assert got[i] == want


def test_batched_tensor_core_decoder_beams_and_logits(wide):
    dims, sp, wh, _, w_t, _ = wide
    waves = [synth.waveform(42000 + 9000 * i, seed=60 + i) for i in range(3)]
    sess = transcribe.Session(wh, max_windows=3, max_beams=5, max_text_len=4 + 8 + 1)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=5, max_depth=8)      # 15 rows, ancestry table
    assert sess.last_decoder() == 5
    assert got == h.golden("tokens_wide")["test-c_beam5_depth8_f32"]
    for g, wv in zip(got, waves):
        assert g == o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(wv)[None]), beam_size=5, max_depth=8)
    # stateless forward_decoder (full logits) against the oracle's decoder (mod.rs:131-157)
    sess.encode_waveforms(waves[:1])
    enc = sess.get_encoder_output(0)[None]
    toks = np.asarray([sp.prompt() + [17, 300, 5]], np.int64)
    lg = wh.forward_decoder(toks, enc)
    ref = o_model.forward_decoder(w_t, dims, torch.from_numpy(toks), torch.from_numpy(enc)).numpy()
    assert rel_to_scale(lg, ref) < 2e-5


def test_launch_counter_counts_kernels(small):
    dims, sp, wh, *_ = small
    ffi.lib().wb_kernel_launch_count_reset()
    sess = transcribe.Session(wh, 1, 1, 16)
    sess.transcribe_windows([synth.waveform(16000, seed=1)], sp, is_special_of(sp), beam_size=1, max_depth=4)
    assert ffi.lib().wb_kernel_launch_count() > 20     # log-mel 2 + encoder ~27 + cross K/V + 1 persistent decoder launch


@pytest.mark.parametrize("beam_size", [1, 5])
def test_batched_decoder_row_groups(wide, beam_size):
    """More rows than one launch of decoder5.cu takes (the shape of BASELINE configs[4]: beams of many windows per GPU): the session
    runs row groups of 32, one launch each; greedy 40 windows = 2 groups, beam 5 x 9 windows = 45 rows = 2 groups with the ancestry
    table addressing absolute cache rows."""
    dims, sp, wh, _, w_t, _ = wide
    n = 40 if beam_size == 1 else 9
    waves = [synth.waveform(28000 + 1500 * i, seed=200 + i) for i in range(n)]
    sess = transcribe.Session(wh, max_windows=n, max_beams=beam_size, max_text_len=4 + 8 + 1)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=beam_size, max_depth=8)
    assert sess.last_decoder() == 5
    for i in (range(0, n, 7) if beam_size == 1 else range(n)):
        want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(waves[i])[None]), beam_size=beam_size, max_depth=8)
        assert got[i] == want, f"window {i}"
