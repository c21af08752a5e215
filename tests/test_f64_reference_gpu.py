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
so every row runs to the last checked step; check_greedy asserts that it does.

Tolerances are absolute on log-probs (|log-prob| ~ 7.6 for V = 2051, ~10.9 for V = 51864) and separate for the fp32 and the
fp16 K/V cache: at an fp16 rounding boundary a float64 value can round to the neighbour of the one the GPU's float32 value
rounds to.  Each constant states the worst error measured on one H100 80GB HBM3 and the margin over it."""
import functools
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest
import torch

import wb200  # noqa: F401
from oracle import model as o_model, synth, transcribe as o_tr
from whisper_burn_b200 import ffi, model, transcribe
from whisper_burn_b200.synth import WhisperDims

pytestmark = pytest.mark.gpu

# greedy top-1 log-prob vs float64 on the GPU's own path (all greedy decoders).  Worst measured: f32 5.0e-6 (decoder5,
# d = 1280), 4x margin; f16 1.7e-4 (decoder6, d = 384, 8 rows), 3x margin.  Dropping the 8 tail ids of V = 51864 from the
# softmax moves a log-prob by ~1.5e-4, 7x the f32 tolerance.
GREEDY_LP_TOL = {"f32": 2e-5, "f16": 5e-4}
# wb_session_step, all 7 candidates.  Worst measured: f32 1.2e-6 (decoder3, d = 384), 8x margin; f16 7.8e-5 (decoder3,
# d = 384), 4x margin
STEP_LP_TOL = {"f32": 1e-5, "f16": 3e-4}
# full logits of the stateless forward_decoder at 448 positions, each position relative to its logits' scale (the suite's
# decoder bar).  Worst measured 6.7e-6 (decoder5, d = 256), 3x margin
LOGITS_REL_TOL = 2e-5
# encoder output, relative to its scale (the suite's encoder bar).  Worst measured 6.7e-6 (tensor-core, d = 1280), 3x margin
ENC_REL_TOL = 2e-5

DEPTH = 10                                       # greedy steps per window: 2 with the special-token mask, 8 without
SHALLOW_STEPS = tuple(range(1, DEPTH + 1))
N_OF_T = {6: 400, 64: 18720, 65: 19040, 750: 480000}   # waveform samples giving each encoder length
T_ORDER = (750, 6, 65, 64)


def rel_to_scale(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def kv_code(kv):
    return ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32


def report(what, worst, tol):
    print(f"\n[f64] {what}: worst {worst:.3e} (tolerance {tol:.0e})")


@functools.lru_cache(maxsize=2)
def _weights(d, H, V, n_text_layer, exact):
    dims = WhisperDims(80, 1500, d, H, 1, V, 448, d, H, n_text_layer)
    _, w_np, _ = synth.make_weights(dims, seed=d + V)
    if not exact:   # no longer fp16-representable: the fp32 encoder (gemm.cu) and decoder3<float>
        w_np = {k: (v * np.float32(1.0001) if v.ndim else v) for k, v in w_np.items()}
    return dims, w_np, o_model.as_dtype(synth.to_torch(w_np))


def _greedy_ref_rows(model_key, sp, xa, tokens, kv, steps):
    """In a worker process: the float64 log-prob rows of the greedy steps `steps` along `tokens` (greedy_path_log_probs on
    the weights _weights(*model_key) and the window's encoder output xa [T, d])."""
    dims, _, w64 = _weights(*model_key)
    ref = o_tr.greedy_path_log_probs(w64, dims, sp, torch.from_numpy(xa)[None], tokens, opts=o_model.OracleOptions(kv_dtype=kv))
    return {s: ref[s - 1].numpy() for s in steps}


@functools.lru_cache(maxsize=1)
def _ref_pool():
    """Worker processes for the float64 reference: scoring one row is a few hundred small sequential float64 steps, so rows
    run side by side, one torch thread each."""
    return ProcessPoolExecutor(max(1, min(8, (os.cpu_count() or 2) - 1)), mp_context=multiprocessing.get_context("spawn"),
                               initializer=torch.set_num_threads, initargs=(1,))


def make_model(d, H, V, exact=True, n_text_layer=2):
    """(dims, GPU model, float64 weights).  A fresh model.Whisper per call: its stateless forward session reads
    WB200_DECODER when it is created."""
    dims, w_np, w64 = _weights(d, H, V, n_text_layer, exact)
    wh = model.Whisper(dims, w_np)
    assert wh.weights_fp16_exact == exact
    return dims, wh, w64


def windows(n, seed, order=T_ORDER):
    Ts = [order[i % len(order)] for i in range(n)]
    return Ts, [synth.waveform(N_OF_T[T], seed=seed + i) for i, T in enumerate(Ts)]


def encoder_outputs64(sess, Ts):
    out = []
    for r, T in enumerate(Ts):
        xa = sess.get_encoder_output(r)
        assert xa.shape[0] == T
        out.append(torch.from_numpy(xa).double()[None])
    return out


def use_decoder(monkeypatch, n):
    if n:
        monkeypatch.setenv("WB200_DECODER", str(n))
    else:
        monkeypatch.delenv("WB200_DECODER", raising=False)


def edge_steps(edges, max_text_len):
    """The greedy steps whose self attention runs over E - 1, E and E + 1 keys for every edge E, and the last step a session
    of max_text_len allows (step s attends over n = s + 3 keys: the 4-id prompt and s - 1 generated ids)."""
    last = max_text_len - 4
    return tuple(sorted({s for e in edges for s in (e - 4, e - 3, e - 2) if s <= last} | {last}))


def default_decoder(d, rows, t_max):
    """The decoder the default selection picks for a greedy launch of fp16-exact weights that decoder4 does not take (more
    rows than co-resident 16-CTA clusters, or more than 8): decoder6 for d = 128 / 384, <= 24 rows and t_max <= 128, else
    decoder5 where d % 256 == 0, else decoder3."""
    if d in (128, 384) and rows <= 24 and t_max <= 128:
        return 6
    return 5 if d % 256 == 0 else 3


# ---------------------------------------------------------------- a. greedy, per step, top-1 against float64
def check_greedy(dims, wh, kv, n_rows, decoder, seed, steps=SHALLOW_STEPS, max_text_len=None, full_depth=False, tol=None,
                 ref_rows=None):
    """Greedy-decodes n_rows windows once to the deepest step of `steps` and once to each step s of `steps`, and checks the
    top-1 (id, log-prob) of every row at every step s against float64 on the GPU's own path.  max_text_len defaults to the
    deepest step plus the prompt and one.  full_depth: EOT is declared to be a special id past the named ones that no row
    emits (the largest one not emitted by an earlier full-depth launch that a row stopped in), and every row must reach the
    deepest step.  tol defaults to GREEDY_LP_TOL[kv].  ref_rows(sp, xa, paths, kv, steps) -> per row {s: float64 log-prob
    row} computes the reference in this process (xa: the rows' float64 encoder outputs [1, T, d], steps: per row); by
    default worker processes rebuild the model with _weights.  Returns the worst |log-prob error|."""
    depth = max(steps)
    sp = synth.special_tokens(dims)
    bitmap = sp.is_special_bitmap()
    Ts, waves = windows(n_rows, seed)
    sess = transcribe.Session(wh, max_windows=n_rows, max_beams=1, max_text_len=max_text_len or 4 + depth + 1,
                              kv_dtype=kv_code(kv))
    full = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=depth) if not full_depth else None
    eot = sp.n_vocab
    while full is None or (full_depth and any(len(t) < 4 + depth for t in full)):
        eot = max(set(range(sp.first_special, eot)) - {i for t in full or [] for i in t})
        sp = o_tr.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, eot, sp.first_special, sp.n_vocab)
        full = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=depth)
    assert sess.last_decoder() == decoder
    if full_depth:
        assert sess.last_steps() == depth and [len(t) for t in full] == [4 + depth] * n_rows
    xa = encoder_outputs64(sess, Ts)
    row_steps = [[s for s in steps if 4 + s <= len(full[r])] for r in range(n_rows)]
    if ref_rows is None:
        key = (dims.n_text_state, dims.n_text_head, dims.n_vocab, dims.n_text_layer, wh.weights_fp16_exact)
        refs = [_ref_pool().submit(_greedy_ref_rows, key, sp, xa[r][0].numpy(), full[r], kv, row_steps[r]) for r in range(n_rows)]
    got = [dict() for _ in range(n_rows)]      # step -> (id, log-prob) of every row that produced a token at that step
    for s in steps:
        toks = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=s)
        assert sess.last_decoder() == decoder
        ids, lps = sess.last_topk(n_rows, 1)
        for r in range(n_rows):
            assert toks[r] == full[r][:len(toks[r])], f"row {r}: the depth-{s} launch is not a prefix of the depth-{depth} one"
            if len(toks[r]) == 4 + s:
                assert int(ids[r, 0]) == toks[r][-1]
                got[r][s] = float(lps[r, 0])
    tol = tol or GREEDY_LP_TOL[kv]
    worst = 0.0
    local = ref_rows(sp, xa, full, kv, row_steps) if ref_rows is not None else None
    for r in range(n_rows):
        ref = local[r] if local is not None else refs[r].result()
        assert sorted(got[r]) == sorted(ref)
        for s, lp in got[r].items():
            tok = full[r][4 + s - 1]
            err = abs(lp - ref[s][tok])
            worst = max(worst, err)
            assert err < tol, f"row {r} (T = {Ts[r]}) step {s}: log-prob {lp} vs float64 {ref[s][tok]}"
            gap = ref[s].max() - ref[s][tok]       # the GPU id is the float64 argmax up to a near-tie
            assert gap < tol, f"row {r} step {s}: id {tok} is {gap} below the float64 argmax {int(ref[s].argmax())}"
    return worst


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


def check_step_k7(dims, wh, w64, decoder, kv, sess=None, tol=None, out=None):
    """The steps of test_session_step_k7_beams_vs_float64 on `sess` (default: a fresh session of 2 windows, 5 beams,
    max_text_len 16), each checked against float64 within tol (default STEP_LP_TOL[kv]).  out, a list, receives every
    step's (ids, log-probs).  Returns the worst |log-prob error|."""
    sp = synth.special_tokens(dims)
    bitmap = sp.is_special_bitmap()
    K = 7
    Ts, waves = windows(2, seed=700, order=(65, 6))
    if sess is None:
        sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=16, kv_dtype=kv_code(kv))
    sess.encode_waveforms(waves)
    xa = encoder_outputs64(sess, Ts)
    opts = o_model.OracleOptions(kv_dtype=kv)
    prompt = sp.prompt()
    sess.begin(prompt)
    ref = [o_model.CachedDecoder(w64, dims, xa[w], opts) for w in range(2)]
    for dec in ref:
        for t in prompt[:-1]:
            dec.step(torch.tensor([t], dtype=torch.int64))
    rows = [(0, 0), (1, 0)]          # GPU row -> (window, row of that window's float64 decoder)
    maskout = torch.from_numpy(sp.maskout())
    tol = tol or STEP_LP_TOL[kv]
    worst = 0.0

    def step(parents, tokens, masked):
        nonlocal rows, worst
        win = [rows[p][0] for p in parents]
        ids, lps = sess.step(win, parents, tokens, masked, bitmap, K)
        assert sess.last_decoder() == decoder
        if out is not None:
            out.append((ids, lps))
        new_rows = []
        for w in range(2):
            mine = [i for i in range(len(parents)) if win[i] == w]
            ref[w].reorder([rows[parents[i]][1] for i in mine])
            logits = ref[w].step(torch.tensor([tokens[i] for i in mine], dtype=torch.int64))
            if masked:
                logits = logits + maskout
            lp = o_model.log_softmax_last(logits).numpy()
            for j, i in enumerate(mine):
                want = np.sort(lp[j])[::-1][:K]
                have = lp[j][ids[i]]
                err = float(np.abs(lps[i] - have).max())
                worst = max(worst, err)
                assert err < tol, f"row {i}: log-probs {lps[i]} vs float64 {have}"
                # ids differ from float64's order only where float64's own neighbours lie within the tolerance
                assert np.abs(have - want).max() < tol, f"row {i}: ids {ids[i]} vs float64 order {np.argsort(-lp[j])[:K]}"
        for i in range(len(parents)):
            w = win[i]
            new_rows.append((w, sum(1 for q in range(i) if win[q] == w)))
        rows = new_rows
        return ids

    ids = step([0, 1], [prompt[-1]] * 2, True)                                  # 2 rows: RC = 4
    ids = step([0, 0, 0, 1, 1, 1], [int(ids[0, j]) for j in range(3)] + [int(ids[1, j]) for j in range(3)], True)   # fan out: 6
    ids = step([2, 0, 1, 5, 3], [int(ids[2, 1]), int(ids[0, 0]), int(ids[1, 6]), int(ids[5, 0]), int(ids[3, 2])], False)
    ids = step([4, 0, 2], [int(ids[4, 3]), int(ids[0, 0]), int(ids[2, 5])], False)   # back to 3 rows from other parents
    step([1, 0, 2, 2, 1], [int(ids[1, 0]), int(ids[0, 1]), int(ids[2, 0]), int(ids[2, 4]), int(ids[1, 2])], False)
    return worst


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


def forward_decoder_448_error(dims, wh, w64):
    """The worst relative-to-scale error of forward_decoder's logits at every one of n_text_ctx positions."""
    d = dims.n_text_state
    rng = np.random.default_rng(d)
    xa = rng.standard_normal((1, 65, d)).astype(np.float32)
    toks = rng.integers(0, dims.n_vocab, size=(1, dims.n_text_ctx)).astype(np.int64)
    got = wh.forward_decoder(toks, xa)
    want = o_model.forward_decoder(w64, dims, torch.from_numpy(toks), torch.from_numpy(xa).double()).numpy()
    return max(rel_to_scale(got[0, p], want[0, p]) for p in range(dims.n_text_ctx))


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
    worst = 0.0
    for w, T in enumerate(Ts):
        got = sess.get_encoder_output(w)
        assert got.shape == (T, d)
        mel = torch.from_numpy(sess.get_mel(w)).double()[None]
        want = o_model.forward_encoder(w64, dims, mel)[0].numpy()
        e = rel_to_scale(got, want)
        worst = max(worst, e)
        assert e < ENC_REL_TOL, f"window {w} (T = {T}): {e}"
    report(f"encoder d={d} {'tensor-core' if exact else 'fp32'}", worst, ENC_REL_TOL)
