"""Every decoder kernel instance and the encoder at real widths against a float64 restatement of the same arithmetic
(oracle/ on float64 weights, oracle.model.as_dtype), step by step on continuous values.

The token-id tests elsewhere pass unless an error moves an argmax; the synthetic models decode one or two distinct tokens per
window, so a dropped key or a lost bias can hide there.  Here each persistent decoder instance is compared on the log-probs it
selects, and the encoder on its output, at the shapes where the instance's tiling has edges (these models give every LayerNorm
eps = 1e-5 in the default placement, so a wrong eps or placement is invisible here: test_layernorm_eps_gpu.py checks those on
the same models with a distinct eps per LayerNorm, in both placements, and test_layernorm_eps_cpu.py shows that it can fail):

  * models of real width with few layers (1 audio layer, 2 text layers): the kernels are instantiated on d, heads, rows, k
    and the K/V type, not on the layer count, so the float64 reference stays cheap;
  * the real vocabulary sizes where the 16-row vocabulary tile has a tail (51864 leaves 8 ids, 51865 leaves 9, 2051 leaves 3);
  * windows whose encoder lengths fall on the cross-attention split edges, T in {6, 64, 65, 750}, mixed within one batch
    (T = (min(n // 160, 1490) + 10 - 1) // 2 + 1 for n samples).

The float64 reference runs on the GPU's own encoder output, so the decoder checks do not include encoder error.  Greedy
decoders are read back with wb_session_last_topk after greedy runs to each checked depth s: s = 1 .. DEPTH at the shapes
above, and at depth the steps on either side of every key count where a decoder's self attention changes how it walks the
keys.  Step s is chosen from the logits at position p = s + 2, over n = s + 3 keys; for each edge E the deep cases check
n = E - 1, E, E + 1 and the last step the session allows (n = max_text_len - 1):

  * decoder4: up to 128 keys one register batch from the cp.async ring; from 129 keys the long path (key p read back from
    the cache, attn_cta in 128-key turns): E = 128, 256, 384 at max_text_len 448;
  * decoder6: 32 key slots x 4 keys, slot u from 32 u keys on; max_text_len 128 (the most it covers): E = 32, 64, 96;
  * decoder5: fp32 K/V attn_warp in 64-key turns, fp16 K/V attn_warp_ring in 32-key turns through 8 stages (a stage is
    first reused from 257 keys on): E = 64, 128, 256 for both at max_text_len 448, with 1, 9, 17 and 33 rows (row groups);
  * decoder3: attn_cta in 128-key turns: E = 128, 256 at max_text_len 448;
  * the default selection on both sides of decoder6's t_max <= 128 (d = 384, 9 rows: decoder6 at 128, decoder3 at 129).

The deep cases use V = 2051 (the vocabulary tails are covered at depth 10) and declare EOT to be an id the windows never emit,
so every row runs to the last checked step; harness.check_greedy asserts that it does.  The tolerances are
harness.py's GREEDY_LP_TOL, STEP_LP_TOL, LOGITS_REL_TOL and ENC_REL_TOL."""
import pytest

from harness import ENC_REL_TOL, GREEDY_LP_TOL, LOGITS_REL_TOL, SHALLOW_STEPS, STEP_LP_TOL, check_greedy, check_step_k7, \
    edge_steps, encoder_error, forward_decoder_448_error, make_model, report, use_decoder, windows
import wb200  # noqa: F401
from oracle import synth
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu


def default_decoder(d, rows, t_max):
    """The decoder the default selection picks for a greedy launch of fp16-exact weights that decoder4 does not take (more
    rows than co-resident 16-CTA clusters, or more than 8): decoder6 for d = 128 / 384, <= 24 rows and t_max <= 128, else
    decoder5 where d % 256 == 0, else decoder3."""
    if d in (128, 384) and rows <= 24 and t_max <= 128:
        return 6
    return 5 if d % 256 == 0 else 3


# ---------------------------------------------------------------- a. greedy, per step, top-1 against float64
def test_last_topk_argument_checks(monkeypatch):
    """wb_session_last_topk reads what the last launch wrote: it refuses a k or a row count that launch did not have."""
    use_decoder(monkeypatch, 0)
    dims, wh, _ = make_model(128, 2, 2051)
    sp = synth.special_tokens(dims)
    sess = transcribe.Session(wh, max_windows=2, max_beams=1, max_text_len=8)
    with pytest.raises(ffi.WbError) as e:
        sess.last_topk(1, 1)
    assert e.value.code == ffi.WB_ERR_STATE
    toks = sess.transcribe_windows(windows(2, seed=900)[1], sp, sp.is_special_bitmap(), beam_size=1, max_depth=3)
    ids, _ = sess.last_topk(2, 1)
    assert [int(i) for i in ids[:, 0]] == [t[-1] for t in toks]
    for n_rows, k in ((2, 2), (3, 1), (0, 1)):
        with pytest.raises(ffi.WbError) as e:
            sess.last_topk(n_rows, k)
        assert e.value.code == ffi.WB_ERR_INVALID_ARG


DEC4_CASES = [(d, rows, kv) for d in (128, 384) for rows in (1, 4, 5, 8) for kv in ("f32", "f16")]


def check_decoder4(d, V, rows, kv, seed, what, monkeypatch, **greedy_args):
    """check_greedy on decoder4, or, where decoder4 does not cover the rows, on the decoder the default selection picks for
    them at this max_text_len (default_decoder), followed by a skip."""
    dims, wh, _ = make_model(d, d // 64, V)
    use_decoder(monkeypatch, 4)
    try:
        worst = check_greedy(dims, wh, kv, rows, 4, seed, **greedy_args)
    except ffi.WbError as e:
        if e.code != ffi.WB_ERR_UNSUPPORTED or rows <= 4:
            raise
        # decoder4 runs one 16-CTA cluster per row and needs all of them co-resident; where the GPU holds fewer, the default
        # selection must send these rows on, and they must pass there
        steps = greedy_args.get("steps", SHALLOW_STEPS)
        fallback = default_decoder(d, rows, greedy_args.get("max_text_len") or 4 + max(steps) + 1)
        use_decoder(monkeypatch, 0)
        worst = check_greedy(dims, wh, kv, rows, fallback, seed, **greedy_args)
        report(f"decoder{fallback} (default for decoder4's rows) {what} d={d} rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])
        pytest.skip(f"decoder4 does not cover {rows} rows: fewer than {rows} co-resident 16-CTA clusters fit on this GPU "
                    f"(checked on decoder{fallback} instead)")
    report(f"decoder4 {what} d={d} rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("d,rows,kv", DEC4_CASES)
def test_decoder4_greedy_steps_vs_float64(d, rows, kv, monkeypatch):
    """decoder4.cu, dec4_kernel<d, RC, KVT>: RC = 4 for <= 4 rows, 8 for 5 to 8 rows."""
    check_decoder4(d, 2051 if d == 128 else 51864, rows, kv, 300 + rows, "", monkeypatch)


@pytest.mark.parametrize("d,rows,kv", DEC4_CASES)
def test_decoder4_deep_greedy_steps_vs_float64(d, rows, kv, monkeypatch):
    """decoder4 at max_text_len 448: the register batch up to 128 keys, the long path (key p read back from the cache after
    the cluster barrier, attn_cta over row * t_max addressing) from 129 keys on, across its 128-key turns."""
    check_decoder4(d, 2051, rows, kv, 1300 + rows, "deep", monkeypatch, steps=edge_steps((128, 256, 384), 448),
                   max_text_len=448, full_depth=True)


DEC6_CASES = [(d, rows, kv) for d in (128, 384) for rows in (1, 8, 9, 24) for kv in ("f32", "f16")]


@pytest.mark.parametrize("d,rows,kv", DEC6_CASES)
def test_decoder6_greedy_steps_vs_float64(d, rows, kv, monkeypatch):
    """decoder6.cu, dec6_kernel<d, NT8, KVT>: NT8 = 1 for <= 8 rows, 3 for 9 to 24 rows."""
    dims, wh, _ = make_model(d, d // 64, 2051 if d == 128 else 51864)
    use_decoder(monkeypatch, 6)
    worst = check_greedy(dims, wh, kv, rows, 6, seed=400 + rows)
    report(f"decoder6 d={d} rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("d,rows,kv", DEC6_CASES)
def test_decoder6_deep_greedy_steps_vs_float64(d, rows, kv, monkeypatch):
    """decoder6 at max_text_len 128, the most it covers: all four key slots of self_attn6_body (slot u from 32 u keys on)."""
    dims, wh, _ = make_model(d, d // 64, 2051)
    use_decoder(monkeypatch, 6)
    worst = check_greedy(dims, wh, kv, rows, 6, 1400 + rows, steps=edge_steps((32, 64, 96), 128), max_text_len=128,
                         full_depth=True)
    report(f"decoder6 deep d={d} rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


# (d, rows): nt8 = 1..4, row groups of 32 (33 rows = 32 + 1), the split d x d stage table (n_splits == 1 with d >= 512),
# the 3-slab MLP2 (d = 768) and large-v2's width and vocabulary tail (d = 1280, V = 51865)
DEC5_CASES = [(d, rows, kv) for d, rows in ((256, 1), (256, 9), (256, 33), (512, 17), (512, 32), (768, 9), (1280, 1))
              for kv in ("f32", "f16")]


@pytest.mark.parametrize("d,rows,kv", DEC5_CASES)
def test_decoder5_greedy_steps_vs_float64(d, rows, kv, monkeypatch):
    """decoder5.cu, dec5_kernel<NT8, KVT> with NT8 = ceil(rows / 8) per row group, chosen by the default selection."""
    dims, wh, _ = make_model(d, d // 64, 51865 if d == 1280 else 2051)
    use_decoder(monkeypatch, 0)
    worst = check_greedy(dims, wh, kv, rows, 5, seed=500 + rows)
    report(f"decoder5 d={d} rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


DEC5_DEEP_CASES = [(d, rows, kv) for d, rows in ((256, 1), (256, 9), (256, 33), (512, 17)) for kv in ("f32", "f16")]


@pytest.mark.parametrize("d,rows,kv", DEC5_DEEP_CASES)
def test_decoder5_deep_greedy_steps_vs_float64(d, rows, kv, monkeypatch):
    """decoder5 at max_text_len 448: fp32 K/V attn_warp (64-key turns), fp16 K/V attn_warp_ring (32-key turns, 8 stages,
    the first stage reused from 257 keys on); 33 rows run as row groups of 32 + 1 (cache rows offset by kv_row0)."""
    dims, wh, _ = make_model(d, d // 64, 2051)
    use_decoder(monkeypatch, 0)
    worst = check_greedy(dims, wh, kv, rows, 5, 1500 + rows, steps=edge_steps((64, 128, 256), 448), max_text_len=448,
                         full_depth=True)
    report(f"decoder5 deep d={d} rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


DEC3_CASES = [(d, exact, rows, kv) for d in (128, 192, 384) for exact in (True, False) for rows in (3, 6)
              for kv in ("f32", "f16")]


@pytest.mark.parametrize("d,exact,rows,kv", DEC3_CASES)
def test_decoder3_greedy_steps_vs_float64(d, exact, rows, kv, monkeypatch):
    """decoder3.cu, dec3_kernel<WT, RC, 2, KVT>: RC = 4 for <= 4 rows, 8 above; WT = __half (fp16-exact weights) or float."""
    dims, wh, _ = make_model(d, d // 64, 51864 if d == 384 else 2051, exact=exact)
    use_decoder(monkeypatch, 3)
    worst = check_greedy(dims, wh, kv, rows, 3, seed=600 + rows)
    report(f"decoder3 d={d} {'fp16' if exact else 'fp32'} weights rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


DEC3_DEEP_CASES = [(d, exact, rows, kv) for d in (128, 384) for exact in (True, False) for rows in (3, 6)
                   for kv in ("f32", "f16")]


@pytest.mark.parametrize("d,exact,rows,kv", DEC3_DEEP_CASES)
def test_decoder3_deep_greedy_steps_vs_float64(d, exact, rows, kv, monkeypatch):
    """decoder3 at max_text_len 448: attn_cta over 128-key turns."""
    dims, wh, _ = make_model(d, d // 64, 2051, exact=exact)
    use_decoder(monkeypatch, 3)
    worst = check_greedy(dims, wh, kv, rows, 3, 1600 + rows, steps=edge_steps((128, 256), 448), max_text_len=448,
                         full_depth=True)
    report(f"decoder3 deep d={d} {'fp16' if exact else 'fp32'} weights rows={rows} kv={kv}", worst, GREEDY_LP_TOL[kv])


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("max_text_len,decoder", [(128, 6), (129, 3)])
def test_default_selection_at_t_max_edge_vs_float64(max_text_len, decoder, kv, monkeypatch):
    """9 rows of a d = 384 model (more than decoder4 ever takes) with the default selection: decoder6 up to t_max = 128;
    above, decoder5 needs d % 256 == 0, so decoder3 runs them."""
    assert default_decoder(384, 9, max_text_len) == decoder
    dims, wh, _ = make_model(384, 6, 2051)
    use_decoder(monkeypatch, 0)
    worst = check_greedy(dims, wh, kv, 9, decoder, 1700, steps=edge_steps((32, 64, 96, 128), max_text_len),
                         max_text_len=max_text_len, full_depth=True)
    report(f"default selection max_text_len={max_text_len} decoder{decoder} d=384 rows=9 kv={kv}", worst, GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- b. wb_session_step, k = 7, with beams
STEP_CASES = [(3, 384, True, kv) for kv in ("f32", "f16")] + [(3, 192, False, kv) for kv in ("f32", "f16")] + \
             [(5, 256, True, kv) for kv in ("f32", "f16")]


@pytest.mark.parametrize("decoder,d,exact,kv", STEP_CASES)
def test_session_step_k7_beams_vs_float64(decoder, d, exact, kv, monkeypatch):
    """wb_session_step with k = 7 (decoder3's dec3_kernel<WT, 4|8, 8, KVT>, decoder5) on two windows: fanned out from one
    parent per window, then continued from different parents so the ancestry table is exercised; all 7 (id, log-prob) pairs
    against float64 oracle.model.CachedDecoder rows reordered the same way."""
    dims, wh, w64 = make_model(d, d // 64, 51864 if d == 384 else 2051, exact=exact)
    use_decoder(monkeypatch, 3 if decoder == 3 else 0)
    worst = check_step_k7(dims, wh, w64, decoder, kv)
    report(f"step k=7 decoder{decoder} d={d} {'fp16' if exact else 'fp32'} weights kv={kv}", worst, STEP_LP_TOL[kv])


# ---------------------------------------------------------------- c. full logits at the maximum text length
@pytest.mark.parametrize("decoder,d", [(3, 384), (5, 256)])
def test_forward_decoder_448_positions_vs_float64(decoder, d, monkeypatch):
    """Stateless forward_decoder (position by position through the cached step, full logits) at seq_len = n_text_ctx = 448:
    self-attention over up to 448 keys.  Forcing the decoder makes any other choice an error."""
    use_decoder(monkeypatch, decoder)
    dims, wh, w64 = make_model(d, d // 64, 2051)
    worst = forward_decoder_448_error(dims, wh, w64)
    report(f"forward_decoder 448 positions decoder{decoder} d={d}", worst, LOGITS_REL_TOL)
    assert worst < LOGITS_REL_TOL


# ---------------------------------------------------------------- d. encoder at real widths, ragged windows
@pytest.mark.parametrize("exact", [True, False], ids=["tensor-core", "fp32"])
@pytest.mark.parametrize("d,H", [(384, 6), (512, 8), (768, 12), (1024, 16), (1280, 20)])
def test_encoder_ragged_windows_vs_float64(d, H, exact):
    """Encoder output of 4 windows with T = 6, 64, 65, 750 packed back to back in one batch, against the float64 encoder
    of each window's padded mel.  fp16-exact weights: wgmma GEMMs (gemm_f16.cu, N = 3d and 4d) and enc_attn_tc.cu;
    otherwise gemm.cu and the fp32 attention."""
    dims, wh, w64 = make_model(d, H, 2051, exact=exact, n_text_layer=1)
    Ts, waves = windows(4, seed=800 + d, order=(6, 64, 65, 750))
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8)
    sess.encode_waveforms(waves)
    worst = encoder_error(sess, w64, dims, Ts, ENC_REL_TOL)
    report(f"encoder d={d} {'tensor-core' if exact else 'fp32'}", worst, ENC_REL_TOL)
