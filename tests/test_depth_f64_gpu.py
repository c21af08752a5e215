"""Every decoder instance, the encoder and the scorer against float64 at the real models' layer counts.

test_f64_reference_gpu.py checks every kernel instance on models of real width with 1 audio layer and 2 text layers.  The
kernels run a lot of code per layer that cannot go visibly wrong there: decoder4 streams layer l + 1's Wqkv during layer l and
layer 0's at the last layer, with stage barriers of phase parity l & 1 (with L = 2 "the next layer" and "layer 0 of the next
position" are one index modulo 2, and every position flips each parity an even number of times); decoder6's producer warp
lines up its TMA weight ring from one position to the next by the number of weight slabs per position, which grows with L;
decoder5 chains its stage table into the next layer and folds a layer's MLP2 partial sums in the next LayerNorm stage; the
encoder caches its tensor-map plans per GEMM site (2 + 4 l + ...) and the scorer keeps 6 plans per layer.  Here the same
checks run on models of 3, 4, 6, 12, 24 and 32 layers (L = 3 breaks the even parity every real depth shares):

  * deep decoder models have 1 audio layer, deep encoder models 1 text layer; one float64 model is held at a time (harness.deep_weights);
  * greedy decoders, per step, top-1 against float64 (harness.check_greedy), at the rows that pick each
    instance's tile (decoder4 RC = 4 / 8, decoder6 NT8 = 1 / 3, decoder5 row groups) and, for one deep case per decoder, at
    every self-attention key-count edge up to max_text_len;
  * wb_session_step (k = 7, beams) and the stateless forward_decoder at 448 positions;
  * the encoder on both paths over ragged windows T = 6, 64, 65, 750 and one native T = 1500 window; the fp32 path stops at
    12 layers (its float64 reference on fp32 weights is a second model of the same size for every width);
  * score_tokens at 12, 24 and 32 layers, and one call of more than SCORE_GROUP_ROWS = 4096 rows (two groups and more);
  * one long-lived Session per decoder family taking a sequence of calls whose rows, decoder, search and kind change from
    call to call, each checked against float64 and bit for bit against the same call on a fresh Session.

The float64 reference of a greedy or beam path is one teacher-forced oracle.model.forward_decoder over the whole path
(harness.forward_rows, rows on windows of one length batched): the same arithmetic as the cached decoder, with the weights
read once per path rather than once per step, which is what makes 24 and 32 float64 layers affordable in this process.  The
error grows with depth, so harness.py's DEEP_* constants replace the float64 suite's here, each with the worst error
measured on one H100 and its margin.
test_depth_f64_cpu.py shows that a layer-indexing mistake moves what is compared here by far more than these tolerances."""
import dataclasses
import resource
import time

import numpy as np
import pytest

import harness as h
import wb200  # noqa: F401
from oracle import synth
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu

SCORE_GROUP_ROWS = 4096     # score.cu: rows of one scoring pass


@pytest.fixture(scope="module", autouse=True)
def _peak_memory():
    t0 = time.time()
    yield
    peak = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    print(f"\n[f64] depth file: {time.time() - t0:.0f} s, peak host memory {peak:.1f} GB")


def ref_rows_of(w64, dims):
    return lambda sp, xa, paths, kv, row_steps: h.forward_rows(w64, dims, xa, paths, kv, sp=sp, steps=row_steps)


# ---------------------------------------------------------------- a. greedy decoders, per step, top-1 against float64
def case_id(c):
    dec, d, L, V, rows, kv, deep, exact = c
    return f"dec{dec}-d{d}-L{L}-V{V}-rows{rows}-{kv}" + ("-deep" if deep else "") + ("" if exact else "-fp32w")


KVS = ("f32", "f16")
# (decoder, d, L, V, rows, kv, deep, fp16-exact weights); deep: every key-count edge up to the decoder's max_text_len
GREEDY_CASES = sorted(
    [(4, 384, L, 51864, rows, kv, False, True) for L in (3, 4) for rows in (1, 5) for kv in KVS]
    + [(4, 384, 4, 2051, 5, kv, True, True) for kv in KVS]
    + [(6, 384, L, 51864, rows, kv, False, True) for L in (3, 4) for rows in (8, 9, 24) for kv in KVS]
    + [(6, 384, 4, 2051, 9, kv, True, True) for kv in KVS]
    + [(3, 384, 4, 51864, rows, kv, False, exact) for exact in (True, False) for rows in (3, 6) for kv in KVS]
    + [(5, d, L, V, rows, kv, False, True) for d, L, V, rows in
       ((512, 6, 2051, 9), (512, 6, 2051, 33), (768, 12, 2051, 1), (768, 12, 2051, 9), (1024, 24, 51864, 1),
        (1024, 24, 51864, 9), (1280, 32, 51865, 1), (1280, 32, 51865, 9), (1280, 4, 51865, 1), (1280, 4, 51865, 33))
       for kv in KVS]
    + [(5, 512, 6, 2051, 9, kv, True, True) for kv in KVS],
    key=lambda c: (c[1], c[2], c[3], not c[7]))     # cases of one model in a row
DEEP_EDGES = {4: ((128, 256, 384), 448), 6: ((32, 64, 96), 128), 5: ((64, 128, 256), 448)}


@pytest.mark.parametrize("case", GREEDY_CASES, ids=case_id)
def test_greedy_steps_vs_float64(case, monkeypatch):
    """decoder4 (RC = 4, 8), decoder6 (NT8 = 1, 3), decoder5 (1, 9 and 33 rows: one row group and 32 + 1) and decoder3
    (fp16 and fp32 weights), each forced with WB200_DECODER, at 3 to 32 layers."""
    dec, d, L, V, rows, kv, deep, exact = case
    dims, wh, w64 = h.make_deep_model(d, V, n_text_layer=L, exact=exact)
    h.use_decoder(monkeypatch, dec)
    args = dict(tol=h.DEEP_GREEDY_LP_TOL[kv], ref_rows=ref_rows_of(w64, dims))
    if deep:
        edges, t_max = DEEP_EDGES[dec]
        args.update(steps=h.edge_steps(edges, t_max), max_text_len=t_max, full_depth=True)
    try:
        worst = h.check_greedy(dims, wh, kv, rows, dec, 3000 + 10 * L + rows, **args)
    except ffi.WbError as e:
        # decoder4 runs one 16-CTA cluster per row and needs all of them co-resident (test_f64_reference_gpu.check_decoder4)
        if dec != 4 or e.code != ffi.WB_ERR_UNSUPPORTED or rows <= 4:
            raise
        pytest.skip(f"decoder4 does not cover {rows} rows: fewer than {rows} co-resident 16-CTA clusters fit on this GPU")
    h.report(case_id(case), worst, h.DEEP_GREEDY_LP_TOL[kv])


# ---------------------------------------------------------------- b. wb_session_step and forward_decoder
@pytest.mark.parametrize("kv", KVS)
@pytest.mark.parametrize("decoder,d,L,V", [(3, 384, 4, 51864), (5, 512, 6, 2051)])
def test_session_step_k7_beams_vs_float64(decoder, d, L, V, kv, monkeypatch):
    """test_f64_reference_gpu.test_session_step_k7_beams_vs_float64 (rows fanned out and continued from other parents) on
    decoder3 at 384 / 4 layers and decoder5 at 512 / 6."""
    dims, wh, w64 = h.make_deep_model(d, V, n_text_layer=L)
    h.use_decoder(monkeypatch, decoder)
    worst = h.check_step_k7(dims, wh, w64, decoder, kv, tol=h.DEEP_STEP_LP_TOL[kv])
    h.report(f"step k=7 decoder{decoder} d={d} L={L} kv={kv}", worst, h.DEEP_STEP_LP_TOL[kv])


@pytest.mark.parametrize("decoder,d,L", [(3, 384, 4), (5, 512, 6)])
def test_forward_decoder_448_positions_vs_float64(decoder, d, L, monkeypatch):
    h.use_decoder(monkeypatch, decoder)
    dims, wh, w64 = h.make_deep_model(d, 2051, n_text_layer=L)
    worst = h.forward_decoder_448_error(dims, wh, w64)
    h.report(f"forward_decoder 448 positions decoder{decoder} d={d} L={L}", worst, h.DEEP_LOGITS_REL_TOL)
    assert worst < h.DEEP_LOGITS_REL_TOL


# ---------------------------------------------------------------- c. encoder
ENC_DEPTHS = ((384, 4), (512, 6), (768, 12), (1024, 24), (1280, 32))


@pytest.mark.parametrize("d,L,exact", [(d, L, exact) for d, L in ENC_DEPTHS for exact in (True, False) if exact or L <= 12],
                         ids=lambda v: str(v) if not isinstance(v, bool) else ("tensor-core" if v else "fp32"))
def test_deep_encoder_vs_float64(d, L, exact):
    """Windows of T = 6, 64, 65, 750 in one batch (and at 384 / 4 one native T = 1500 window) through L encoder layers:
    wgmma GEMMs and enc_attn_tc.cu on fp16-exact weights, gemm.cu and the fp32 attention otherwise."""
    dims, wh, w64 = h.make_deep_model(d, 2051, n_audio_layer=L, exact=exact)
    Ts, waves = h.windows(4, seed=900 + L, order=(6, 64, 65, 750))
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8)
    sess.encode_waveforms(waves)
    worst = h.encoder_error(sess, w64, dims, Ts, h.DEEP_ENC_REL_TOL)
    h.report(f"encoder d={d} L={L} {'tensor-core' if exact else 'fp32'}", worst, h.DEEP_ENC_REL_TOL)
    if d == 384:
        sess = transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=8, windows="native")
        sess.encode_waveforms([synth.waveform(480000, seed=901)])
        worst = h.encoder_error(sess, w64, dataclasses.replace(dims, n_audio_ctx=2 * dims.n_audio_ctx), [1500], h.DEEP_ENC_REL_TOL)
        h.report(f"encoder native T=1500 d={d} L={L} {'tensor-core' if exact else 'fp32'}", worst, h.DEEP_ENC_REL_TOL)


# ---------------------------------------------------------------- d. scorer
def check_masked(sess, w64, dims, sp, xa, kv, tol):
    seqs = h.masked_seqs(sp, 9)
    wins = [r % len(xa) for r in range(len(seqs))]
    out = sess.score_tokens(seqs, wins, apply_special_mask=True, is_special=h.is_special_of(sp))
    rows = h.forward_rows(w64, dims, [xa[w] for w in wins], seqs, kv, sp=sp, steps=[range(1, len(s) - 3) for s in seqs])
    worst = 0.0
    for seq, (lp, _), ref in zip(seqs, out, rows):
        assert np.isneginf(lp[4]) and np.isneginf(lp[5]) and np.all(np.isfinite(lp[6:]))
        want = np.array([ref[j - 3][seq[j]] for j in range(6, len(seq))])
        err = float(np.abs(lp[6:].astype(np.float64) - want).max())
        worst = max(worst, err)
        assert err < tol, f"masked rows: {err}"
    return worst


@pytest.mark.parametrize("kv", KVS)
@pytest.mark.parametrize("d,L,V", [(768, 12, 2051), (1024, 24, 51864), (1280, 32, 51865)])
def test_score_deep_vs_float64(d, L, V, kv):
    """The harness.LENGTHS sequences (around the 64-row tiles up to n_text_ctx) on windows of T = 6, 64,
    65, 750, and the masked rows of the beam rule, through 12, 24 and 32 layers."""
    dims, wh, w64 = h.make_deep_model(d, V, n_text_layer=L)
    sp = synth.special_tokens(dims)
    Ts, waves = h.windows(4, seed=11 * L)
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    seqs = h.random_seqs(V, L)
    wins = [i % 4 for i in range(len(seqs))]
    out = sess.score_tokens(seqs, wins)
    tol = h.DEEP_SCORE_LP_TOL[kv]
    worst = 0.0
    for (lp, am), seq, w in zip(out, seqs, wins):
        ref = h.forward_rows(w64, dims, [xa[w]], [seq], kv)[0] if len(seq) > 1 else None
        worst = max(worst, h.check_rows(lp, am, ref, seq, kv, f"d={d} L={L} kv={kv} T={Ts[w]} len={len(seq)}", tol=tol))
    worst = max(worst, check_masked(sess, w64, dims, sp, xa, kv, tol))
    h.report(f"score_tokens d={d} L={L} kv={kv}", worst, tol)


@pytest.mark.parametrize("kv", KVS)
def test_score_groups_vs_float64(kv):
    """One call of more than SCORE_GROUP_ROWS rows at 384 / 4 layers: ten length-448 sequences among short ones (length 1
    included) run as two groups; each sequence against float64 and bit for bit against itself scored alone; and a call of
    length-1 sequences only (a group without rows)."""
    dims, wh, w64 = h.make_deep_model(384, 2051, n_text_layer=4)
    Ts, waves = h.windows(4, seed=13)
    sess = transcribe.Session(wh, max_windows=4, max_beams=1, max_text_len=8, kv_dtype=h.kv_code(kv))
    sess.encode_waveforms(waves)
    xa = h.encoder_outputs64(sess, Ts)
    long = h.random_seqs(dims.n_vocab, 17, lengths=(448,) * 10)
    short = h.random_seqs(dims.n_vocab, 18, lengths=(1, 2, 65, 1, 130, 1, 7, 64, 1, 300, 1))
    seqs = [s for pair in zip(long, short) for s in pair] + short[10:]
    wins = [(3 * i) % 4 for i in range(len(seqs))]
    assert sum(len(s) - 1 for s in seqs) > SCORE_GROUP_ROWS
    out = sess.score_tokens(seqs, wins)
    tol = h.DEEP_SCORE_LP_TOL[kv]
    worst = 0.0
    for i, ((lp, am), seq, w) in enumerate(zip(out, seqs, wins)):
        ref = h.forward_rows(w64, dims, [xa[w]], [seq], kv)[0] if len(seq) > 1 else None
        worst = max(worst, h.check_rows(lp, am, ref, seq, kv, f"sequence {i} len={len(seq)} T={Ts[w]}", tol=tol))
        alone = sess.score_tokens([seq], [w])[0]
        assert np.array_equal(alone[0], lp) and np.array_equal(alone[1], am), f"sequence {i}: not the bits it scores alone"
    ones = sess.score_tokens([[5], [7], [2050]], [0, 3, 1])
    assert all(np.array_equal(lp, [0.0]) and np.array_equal(am, [-1]) for lp, am in ones)
    h.report(f"score_tokens {len(seqs)} sequences, {sum(len(s) - 1 for s in seqs)} rows d=384 L=4 kv={kv}", worst, tol)


# ---------------------------------------------------------------- e. one long-lived Session, calls that change
def decode_call(rows, beam, seed):
    return ("decode", rows, beam, seed)


# per family model: (d, L, V, session rows, beams, max_text_len, calls); each call's expected decoder follows it
HISTORY = {
    "d384-L4": (384, 4, 2051, 24, 5, 40, [
        (decode_call(1, 1, 40), 4), (("score", 41), None), (decode_call(9, 1, 42), 6), (decode_call(2, 5, 43), 6),
        (("step",), 3), (decode_call(3, 1, 44), 4), (("score", 45), None), (decode_call(24, 1, 46), 6),
        (decode_call(3, 5, 47), 6), (decode_call(1, 1, 40), 4)]),
    "d512-L6": (512, 6, 2051, 33, 5, 40, [
        (decode_call(1, 1, 50), 5), (("score", 51), None), (decode_call(33, 1, 52), 5), (("step",), 5),
        (decode_call(2, 5, 53), 5), (decode_call(9, 1, 54), 5), (("score", 55), None), (decode_call(1, 1, 50), 5)]),
}


def run_call(sess, call, decoder, dims, wh, w64, kv):
    """Runs one call on sess and checks it against float64; returns (its outputs, compared bit for bit across sessions,
    the worst |log-prob error|)."""
    sp = synth.special_tokens(dims)
    tol = h.DEEP_GREEDY_LP_TOL[kv]
    if call[0] == "step":
        out = []
        worst = h.check_step_k7(dims, wh, w64, decoder, kv, sess=sess, tol=h.DEEP_STEP_LP_TOL[kv], out=out)
        return out, worst
    if call[0] == "score":
        Ts, waves = h.windows(3, seed=call[1])
        sess.encode_waveforms(waves)
        xa = h.encoder_outputs64(sess, Ts)
        seqs = h.random_seqs(dims.n_vocab, call[1], lengths=(2, 65, 448, 1, 130))
        wins = [i % 3 for i in range(len(seqs))]
        out = sess.score_tokens(seqs, wins)
        worst = max(h.check_rows(lp, am, h.forward_rows(w64, dims, [xa[w]], [seq], kv)[0] if len(seq) > 1 else None, seq, kv, f"{call}",
                               tol=h.DEEP_SCORE_LP_TOL[kv]) for (lp, am), seq, w in zip(out, seqs, wins))
        return out, worst
    _, rows, beam, seed = call
    Ts, waves = h.windows(rows, seed)
    toks = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=beam, max_depth=h.DEPTH)
    assert sess.last_decoder() == decoder, (call, sess.last_decoder())
    lps = [sess.last_logprobs(r) for r in range(rows)]
    xa = h.encoder_outputs64(sess, Ts)
    refs = h.forward_rows(w64, dims, xa, toks, kv, sp=sp, steps=[range(1, len(t) - 3) for t in toks])
    worst = 0.0
    for r, (t, lp, ref) in enumerate(zip(toks, lps, refs)):
        for s in range(1, len(t) - 3):
            err = abs(float(lp[3 + s]) - ref[s][t[3 + s]])
            worst = max(worst, err)
            assert err < tol, f"{call} row {r} step {s}: log-prob {lp[3 + s]} vs float64 {ref[s][t[3 + s]]}"
            if beam == 1:
                assert ref[s].max() - ref[s][t[3 + s]] < tol, f"{call} row {r} step {s}: not the float64 arg-max"
    return (toks, lps), worst


def same_bits(a, b):
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same_bits(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("kv", KVS)
@pytest.mark.parametrize("family", list(HISTORY))
def test_long_lived_session_vs_fresh(family, kv):
    """One Session takes greedy launches of changing rows (and so decoders), device or host beam searches, host steps and
    scoring calls in between; each call is checked against float64 and against the same call on a fresh Session.  The fresh
    result is itself taken twice: a call that two fresh sessions do not repeat bit for bit is reported and left to the
    float64 check."""
    d, L, V, n_win, n_beam, t_max, calls = HISTORY[family]
    dims, wh, w64 = h.make_deep_model(d, V, n_text_layer=L)

    def session():
        return transcribe.Session(wh, max_windows=n_win, max_beams=n_beam, max_text_len=t_max, kv_dtype=h.kv_code(kv))

    long_lived = session()
    unrepeatable = []
    worst = 0.0
    for i, (call, decoder) in enumerate(calls):
        got, err = run_call(long_lived, call, decoder, dims, wh, w64, kv)
        worst = max(worst, err)
        fresh = [run_call(session(), call, decoder, dims, wh, w64, kv)[0] for _ in range(2)]
        if not same_bits(fresh[0], fresh[1]):
            unrepeatable.append(call)
            continue
        assert same_bits(got, fresh[0]), f"call {i} {call}: the long-lived session's result differs from a fresh session's"
    if unrepeatable:
        print(f"\n[f64] {family} kv={kv}: not bit-repeatable on fresh sessions (checked against float64 only): {unrepeatable}")
    h.report(f"long-lived session {family} kv={kv}, {len(calls)} calls", worst, h.DEEP_SCORE_LP_TOL[kv])
