"""CPU tests of the oracle (oracle/): golden vectors, reference quirks, host-logic restatements.
The reference has no tests (SURVEY.md F4); these pin the oracle against the committed fixtures."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import audio, beam, model, synth, transcribe

G = Path(__file__).resolve().parent / "golden"


def test_max_waveform_samples_and_windows():
    assert audio.max_waveform_samples(1490) == 238559          # audio.rs:12-17 with n_ctx 1500 - 10
    b = transcribe.window_bounds(480000, 16000, 238559)         # SURVEY F6: a 30 s chunk = 3 windows
    assert b == [(0, 238559), (190559, 429118), (381118, 480000)]
    assert transcribe.window_bounds(1, 16000, 238559) == [(0, 1)]
    assert transcribe.window_bounds(0, 16000, 238559) == [(0, 0)]   # iter_len = 0.saturating_sub(1)/shift + 1 = 1


def test_mel_golden():
    z = np.load(G / "mel_golden.npz")
    for key in z.files:
        n, kind, seed, stride = key.split("_")
        w = synth.waveform(int(n), seed=int(seed), kind=kind)
        m = audio.prep_audio(torch.from_numpy(w)[None]).numpy()[0][:, ::int(stride)]
        assert m.shape == z[key].shape
        # same library family on possibly another CPU: allow fp32 reassociation noise only
        assert np.abs(m - z[key]).max() <= 2e-5 * max(1.0, np.abs(z[key]).max()), key


def test_mel_shape_and_quirks():
    w = synth.waveform(16000, seed=1)
    m = audio.prep_audio(torch.from_numpy(w)[None])
    assert m.shape == (1, 80, 100)                               # n/160 frames: the last STFT frame is dropped
    assert float(m.max() - m.min()) <= 2.0 + 1e-6                # clamp to max-8 then /4
    with pytest.raises(AssertionError):
        audio.prep_audio(torch.zeros(1, 399))                    # audio.rs:292
    # the reference's f32-angle DFT is close to, but not, an exact STFT (SURVEY section 7)
    exact = audio.prep_audio_f64(w[None])
    d = np.abs(m.numpy() - exact)
    assert 0 < d.max() < 1e-3
    # batch call: ONE max over the whole tensor (audio.rs:50)
    wb = np.stack([w, 0.01 * w])
    mb = audio.prep_audio(torch.from_numpy(wb)).numpy()
    assert np.allclose(mb[0], m.numpy()[0], atol=1e-6)
    assert not np.allclose(mb[1], audio.prep_audio(torch.from_numpy(wb[1:])).numpy()[0], atol=1e-3)


def test_mel_filters_match_librosa_formula():
    f = audio.get_mel_filters().numpy()
    assert f.shape == (80, 201)
    assert (f >= 0).all() and (f.sum(axis=1) > 0).all()
    # Slaney area normalisation: each filter integrates to ~ 2/(f_hi - f_lo) * area of a triangle
    peak = f.argmax(axis=1)
    assert (np.diff(peak) >= 0).all()


def test_beam_tie_break_table():
    cases = json.loads((G / "beam_ties.json").read_text())
    for c in cases:
        idx = list(range(len(c["scores"])))
        assert beam.get_top_elements(idx, lambda i: c["scores"][i], c["num"]) == c["expect"]
    # hand-traced against beam.rs:81-110
    assert beam.get_top_elements([0, 1, 2, 3, 4], lambda i: [1.0, 3.0, 3.0, 2.0, 3.0][i], 2) == [2, 1]
    assert beam.get_top_elements([0, 1, 2, 3], lambda i: 5.0, 1) == [0]
    assert beam.get_top_elements([0, 1], lambda i: [2.0, 1.0][i], 5) == [1, 0]


def test_find_chunk_overlap():
    assert transcribe.find_chunk_overlap([1, 2, 3, 4, 5, 6], [4, 5, 6, 7], 40, 3) == (3, 0)
    assert transcribe.find_chunk_overlap([1, 2, 3], [7, 8, 9], 40, 3) is None
    assert transcribe.find_chunk_overlap([], [1, 2, 3], 40, 3) is None
    assert transcribe.find_chunk_overlap([9, 1, 2, 3, 8], [1, 2, 3, 8, 5], 40, 3) == (1, 0)


def test_tokens_golden_small_model_and_cache_equivalence():
    ta = json.loads((G / "tokens_test_a.json").read_text())
    dims, _, w = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    chunk = synth.chunk_waveform(0)
    mel = audio.prep_audio(torch.from_numpy(chunk[:98882])[None])
    for bs, depth in ((1, 30), (5, 12)):
        want = ta["cases"][f"w98882_beam{bs}_depth{depth}"]
        assert want["min_margin"] > 1e-5
        cached = transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=bs, max_depth=depth, use_cache=True)
        full = transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=bs, max_depth=depth, use_cache=False, exact_topk=True)
        assert cached == want["tokens"]
        assert full == want["tokens"]          # reference-cost path == KV-cached path
    # EOT: search stops as soon as the best beam ends in EOT (beam.rs:22-27)
    e = ta["eot_case"]
    base = ta["cases"]["w238559_beam1_depth30"]["tokens"]
    assert e["tokens"][-1] == e["eot"] and e["tokens"].count(e["eot"]) == 1
    assert e["tokens"] == base[:len(e["tokens"])] and len(e["tokens"]) < len(base)


def test_encoder_golden_and_shapes():
    z = np.load(G / "encoder_golden.npz")
    dims, _, w = synth.make_weights("test-a", seed=0)
    chunk = synth.chunk_waveform(0)
    mel = transcribe.pad_mel(audio.prep_audio(torch.from_numpy(chunk[:98882])[None]), dims.n_audio_ctx)
    assert mel.shape == (1, 80, 628)                                   # 618 frames + 10 zero frames
    enc = model.forward_encoder(w, dims, mel).numpy()
    assert enc.shape == (1, 314, dims.n_audio_state)                   # conv2 stride 2 (SURVEY F6)
    assert np.abs(enc[0, ::8] - z["test_a_enc_w98882"]).max() < 5e-5
    with pytest.raises(AssertionError):
        model.forward_encoder(w, dims, torch.zeros(1, 80, 1501))       # mod.rs:236-241
    with pytest.raises(AssertionError):
        model.forward_encoder(w, dims, torch.zeros(1, 81, 100))        # mod.rs:231-235


def test_layernorm_eps_placement_is_a_real_switch():
    """burn 0.9 LayerNorm divides by (sqrt(var) + eps); later burn releases by sqrt(var + eps).  The
    burn source is not vendored (SURVEY 8c item 10), so both are restated.  The difference is NOT
    negligible where the variance is small (first decoder LayerNorm sees tok_emb + pos_emb with
    var ~ 5e-4, eps 1e-5 -> ~1 % change), so the mode is an explicit option on both sides."""
    dims, _, w = synth.make_weights("test-a", seed=0)
    x = (w["decoder/token_embedding/weight"][:4] + w["decoder/positional_embedding"][:4]).unsqueeze(0)
    a = model.layer_norm(x, w, "decoder/block_0/attn_ln", model.OracleOptions("outside"))
    b = model.layer_norm(x, w, "decoder/block_0/attn_ln", model.OracleOptions("inside"))
    rel = float((a - b).abs().max() / a.abs().max())
    assert 1e-4 < rel < 5e-2
    big = torch.randn(1, 4, dims.n_text_state) * 3.0
    a = model.layer_norm(big, w, "decoder/ln", model.OracleOptions("outside"))
    b = model.layer_norm(big, w, "decoder/ln", model.OracleOptions("inside"))
    assert float((a - b).abs().max()) < 1e-4


def test_special_mask_only_first_two_steps():
    dims, _, w = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    mel = audio.prep_audio(torch.from_numpy(synth.chunk_waveform(0)[:98882])[None])
    tr = {}
    transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=1, max_depth=4, trace=tr)
    lp = tr["log_probs"]
    assert np.isneginf(lp[0][0][sp.first_special:]).all() and np.isneginf(lp[1][0][sp.first_special:]).all()
    assert np.isfinite(lp[2][0][sp.first_special:]).all()             # transcribe.rs:271: max_seq_len > 5


def test_wide_model_tokens_golden():
    """The oracle reproduces the committed ids of the batched-decoder test models (tests/golden/make_golden_wide.py): greedy with the
    fp32 and the fp16 K/V cache, and beam 5."""
    import json
    gold = json.loads((G / "tokens_wide.json").read_text())
    dims, _, w = synth.make_weights("test-c", seed=0)
    sp = synth.special_tokens(dims)
    for i in (0, 9):
        mel = audio.prep_audio(torch.from_numpy(synth.waveform(30000 + 7000 * i, seed=40 + i))[None])
        assert transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=1, max_depth=14) == gold["test-c_greedy_depth14_f32"][i]
        assert transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=1, max_depth=14, opts=model.OracleOptions(kv_dtype="f16")) == gold["test-c_greedy_depth14_f16"][i]
    mel = audio.prep_audio(torch.from_numpy(synth.waveform(42000 + 9000 * 2, seed=62))[None])
    assert transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=5, max_depth=8) == gold["test-c_beam5_depth8_f32"][2]


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_float64_oracle_restates_the_float32_graph(kv):
    """The oracle run on float64 weights and inputs is the same graph as the float32 oracle: encoder output, stateless
    decoder logits and the teacher-forced greedy log-probs agree to float32 noise.  The GPU tests compare the kernels against
    this float64 mode.  With the fp16 K/V cache the rounding keeps the input dtype; there the few K/V elements whose float32
    and float64 values lie on opposite sides of an fp16 rounding boundary move by one fp16 ulp (2^-11 relative), which
    shows as ~6e-5 in the logits and ~9e-5 in the log-probs of this model, so the bound is wider for f16."""
    rel_tol, lp_tol = (5e-6, 1e-5) if kv == "f32" else (2e-4, 3e-4)
    dims, _, w = synth.make_weights("test-a", seed=0)
    w64 = model.as_dtype(w)
    sp = synth.special_tokens(dims)
    opts = model.OracleOptions(kv_dtype=kv)
    raw = audio.prep_audio(torch.from_numpy(synth.waveform(20000, seed=3))[None])
    mel = transcribe.pad_mel(raw, dims.n_audio_ctx)
    enc = model.forward_encoder(w, dims, mel, opts)
    enc64 = model.forward_encoder(w64, dims, mel.double(), opts)
    assert enc64.dtype == torch.float64
    assert float((enc64 - enc).abs().max() / enc64.abs().max()) < 5e-6       # the encoder has no K/V cache

    toks = torch.tensor([sp.prompt() + [17, 300, 5, 911, 2]], dtype=torch.int64)
    lg = model.forward_decoder(w, dims, toks, enc, opts)
    lg64 = model.forward_decoder(w64, dims, toks, enc64, opts)
    assert lg64.dtype == torch.float64
    assert float((lg64 - lg).abs().max() / lg64.abs().max()) < rel_tol

    path = transcribe.mels_to_tokens(w, dims, sp, raw, beam_size=1, max_depth=8, opts=opts)
    lp = transcribe.greedy_path_log_probs(w, dims, sp, enc, path, opts=opts)
    lp64 = transcribe.greedy_path_log_probs(w64, dims, sp, enc64, path, opts=opts)
    assert lp64.dtype == torch.float64 and lp64.shape == (len(path) - 4, dims.n_vocab)
    assert torch.isneginf(lp64[:2, sp.first_special:]).all() and torch.isfinite(lp64[2:]).all()   # mask on the first two steps
    fin = torch.isfinite(lp64)
    assert float((lp64 - lp)[fin].abs().max()) < lp_tol
    # the path is the float32 greedy path: its tokens are the argmax of every row (up to float32 ties)
    assert [int(i) for i in lp.argmax(dim=1)] == path[4:]
    # and the cached scoring equals the stateless decoder's last-position log-softmax
    full = model.log_softmax_last(model.forward_decoder(w64, dims, torch.tensor([path[:-1]]), enc64, opts)[0, 4 - 1:])
    assert float((full - lp64)[2:].abs().max()) < 1e-9


def test_repetition_heuristics_known_answers():
    """Hand-evaluated cases of transcribe.rs:385-447."""
    t = [0, 9] + [1, 2, 3] * 5
    assert transcribe.repetition_period(t, 4) == 3          # suffix [1,2,3] preceded by four equal blocks
    assert transcribe.repetition_period(t, 5) is None       # only four blocks precede the suffix
    assert transcribe.repetition_period([1, 2, 3, 4], 1) is None
    assert transcribe.first_repetition_end(t, 3) == 5       # first mismatch walking back: tokens[1..4] = [9,1,2] vs tokens[4..7] = [3,1,2] at i = 4
    assert transcribe.first_repetition_end([5, 5, 5, 5], 1) == 1
    s = [4, 4, 1, 2, 3, 4, 5, 0, 1, 2, 3, 4, 5, 7, 1, 2, 3, 4, 5, 6, 6, 1, 2, 3, 4, 5, 1, 2, 3, 4, 5]
    assert transcribe.find_repeated_tokens_index(s, 5, 4) == (2, 8)
    assert transcribe.find_repeated_tokens_index(s, 5, 5) is None
    assert transcribe.find_repeated_tokens_index([1, 2, 3], 2, 1) is None    # 2 * window > len
