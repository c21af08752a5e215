"""GPU tests (-m gpu): every LayerNorm implementation reads its own LayerNorm's eps and the placement switch
(wb_model_set_layernorm_eps_mode), on the per-LayerNorm-eps models of tests/layernorm_eps.py, in both placements, against
the float64 oracle on the same eps and placement (test_layernorm_eps_cpu.py shows that a wrong eps or placement at any one
LayerNorm moves what these compare by at least 10x the tolerance):

  1. the encoder, fp16-exact weights (layernorm_f16_kernel) and fp32 weights (layernorm_kernel), T = 6, 64, 65, 750 in one
     batch, d = 384 and 768, against forward_encoder of the session's own mel (ENC_REL_TOL);
  2. greedy on every persistent decoder (decoder4 both row-count instances, decoder6, decoder5, decoder3 with fp16 and fp32
     weights), fp32 and fp16 K/V: every last_logprobs value against float64 teacher forcing of the GPU's own ids on the
     GPU's own encoder output (GREEDY_LP_TOL);
  3. the device beam search (decoder6, beam 5) at d = 128 and 384, the same comparison for each returned sequence;
  4. the scoring pass (score_tokens, whose decoder LayerNorms run in layernorm_f16_kernel) at d = 384, every position
     against float64 log-softmax rows;
  5. an npy tree of these weights loaded with wb_model_load_npy_tree gives the bits of the same tensors set one by one."""
import numpy as np
import pytest

import harness as h
import layernorm_eps as lne
import wb200  # noqa: F401
from harness import check_against_f64, rows_of
from oracle import model as o_model, synth
from whisper_burn_b200 import ffi, model, npytree, transcribe

pytestmark = pytest.mark.gpu
V = 2051


# ---------------------------------------------------------------- 1. encoder
@pytest.mark.parametrize("mode", lne.MODES)
@pytest.mark.parametrize("exact", [True, False], ids=["fp16-exact", "fp32"])
@pytest.mark.parametrize("d,H", [(384, 6), (768, 12)])
def test_encoder_vs_float64(d, H, exact, mode):
    dims, _, wh, w64 = lne.make_model(d, H, V, mode, exact=exact, n_text_layer=1)
    Ts, waves = h.windows(4, seed=810 + d, order=(6, 64, 65, 750))
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8)
    sess.encode_waveforms(waves)
    worst = h.encoder_error(sess, w64, dims, Ts, h.ENC_REL_TOL, o_model.OracleOptions(ln_eps_mode=mode))
    h.report(f"eps {mode}: encoder d={d} {'fp16-exact' if exact else 'fp32'} weights", worst, h.ENC_REL_TOL)


# ---------------------------------------------------------------- 2. greedy, every decoder
# (decoder, d, rows, fp16-exact weights): decoder4's RC = 4 and RC = 8 instances, decoder6, decoder5, decoder3 on both
# weight types
GREEDY_CASES = [(4, 128, 4, True), (4, 128, 5, True), (4, 384, 4, True), (4, 384, 5, True), (6, 128, 9, True),
                (6, 384, 9, True), (5, 256, 9, True), (3, 384, 6, True), (3, 384, 6, False)]


@pytest.mark.parametrize("mode", lne.MODES)
@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("decoder,d,rows,exact", GREEDY_CASES)
def test_greedy_every_decoder_vs_float64(decoder, d, rows, exact, kv, mode, monkeypatch):
    dims, _, wh, w64 = lne.make_model(d, d // 64, V, mode, exact=exact)
    sp = synth.special_tokens(dims)
    _, waves = h.windows(rows, seed=2100 + d + rows)
    h.use_decoder(monkeypatch, decoder)
    sess = transcribe.Session(wh, max_windows=rows, max_beams=1, max_text_len=4 + h.DEPTH + 1, kv_dtype=h.kv_code(kv))
    h.use_decoder(monkeypatch, 0)
    try:
        ids = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=h.DEPTH)
    except ffi.WbError as e:
        # decoder4 runs one 16-CTA cluster per row and needs all of them co-resident (test_f64_reference_gpu.check_decoder4)
        if decoder != 4 or e.code != ffi.WB_ERR_UNSUPPORTED or rows <= 4:
            raise
        pytest.skip(f"decoder4 does not cover {rows} rows: fewer than {rows} co-resident 16-CTA clusters fit on this GPU")
    assert sess.last_decoder() == decoder
    worst = check_against_f64(sess, w64, dims, sp, ids, rows_of(sess, ids), kv, ln_eps_mode=mode)
    h.report(f"eps {mode}: greedy decoder{decoder} d={d} {'fp16' if exact else 'fp32'} weights rows={rows} kv={kv}", worst,
               h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 3. device beam search
@pytest.mark.parametrize("mode", lne.MODES)
@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("d", [128, 384])
def test_device_beam_vs_float64(d, kv, mode):
    """4 windows x beam 5 = 20 rows, one decoder6 launch"""
    dims, _, wh, w64 = lne.make_model(d, d // 64, V, mode)
    sp = synth.special_tokens(dims)
    _, waves = h.windows(4, seed=2200 + d)
    sess = transcribe.Session(wh, max_windows=4, max_beams=5, max_text_len=4 + h.DEPTH + 1, kv_dtype=h.kv_code(kv))
    ids = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=5, max_depth=h.DEPTH)
    assert sess.last_decoder() == 6
    worst = check_against_f64(sess, w64, dims, sp, ids, rows_of(sess, ids), kv, ln_eps_mode=mode)
    h.report(f"eps {mode}: device beam decoder6 d={d} B=5 kv={kv}", worst, h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 4. scoring pass
@pytest.mark.parametrize("mode", lne.MODES)
@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_score_tokens_vs_float64(kv, mode):
    dims, _, wh, w64 = lne.make_model(384, 6, V, mode)
    Ts, waves = h.windows(4, seed=2300)
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    seqs = h.random_seqs(V, 2301)
    wins = [i % len(waves) for i in range(len(seqs))]
    worst = 0.0
    for seq, w, (lp, am) in zip(seqs, wins, sess.score_tokens(seqs, wins)):
        ref = h.forward_rows(w64, dims, [xa[w]], [seq], kv, ln_eps_mode=mode)[0] if len(seq) > 1 else None
        worst = max(worst, h.check_rows(lp, am, ref, seq, kv, f"{mode} kv={kv} T={Ts[w]} len={len(seq)}"))
    h.report(f"eps {mode}: score_tokens d=384 kv={kv}", worst, h.GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- 5. npy tree
def test_npy_tree_keeps_every_eps(tmp_path):
    """The per-LayerNorm eps survive save_npy_tree / wb_model_load_npy_tree: with the "inside" placement, encoder output,
    greedy ids and their log-probs equal those of the same tensors set one by one."""
    dims, w_np, direct, _ = lne.make_model(384, 6, V, "inside")
    npytree.save_npy_tree(tmp_path, dims, w_np)
    loaded = model.Whisper.from_npy_tree(tmp_path, ln_eps_outside=False)
    sp = synth.special_tokens(dims)
    _, waves = h.windows(4, seed=2400)
    out = []
    for wh in (direct, loaded):
        sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=4 + h.DEPTH + 1)
        ids = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=h.DEPTH)
        out.append((ids, [sess.get_encoder_output(r) for r in range(4)], [sess.last_logprobs(r) for r in range(4)],
                    sess.last_decoder()))
    assert out[0][0] == out[1][0] and out[0][3] == out[1][3]
    worst = 0.0
    for a, b in zip(out[0][1] + out[0][2], out[1][1] + out[1][2]):
        assert np.array_equal(a, b)
        worst = max(worst, float(np.abs(a - b).max(initial=0.0)))
    h.report(f"eps inside: npy tree vs the tensors set one by one (decoder{out[0][3]})", worst, 0.0)
