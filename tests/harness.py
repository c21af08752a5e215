"""What the test modules share: synthetic models, float64 reference rows, tolerances, inputs and the checks more than one
module runs.  Test modules import shared code from here (and from layernorm_eps.py, the oracle_*.py restatements, oracle/
and the package), never from one another.

pytest rewrites assert only in test modules, so every assert here carries its own message.

Synthetic models (synth.make_weights):
  * the float64 suite's models of real width with 1 audio layer and 2 text layers (shallow_weights, make_model): seed
    d + V, the last two float64 models kept (LRU);
  * the depth suite's models of real layer counts (deep_weights, make_deep_model): seed d + V + 100 n_audio_layer +
    n_text_layer, one model held at a time;
  * the named seed-0 models (named_model).
exact=False scales every tensor by 1.0001: no longer fp16-representable, so the library runs the fp32 encoder (gemm.cu) and
decoder3<float>.

Float64 reference rows, two ways (each caller keeps the one it uses; the two differ in the last bits):
  * path_rows: along a decoded path by the cached decoder (oracle.transcribe.greedy_path_log_probs);
  * forward_rows: whole sequences by full recompute (oracle.model.forward_decoder), batched by window length.

Tolerances are absolute on log-probs (|log-prob| ~ 7.6 for V = 2051, ~10.9 for V = 51864) and separate for the fp32 and the
fp16 K/V cache: at an fp16 rounding boundary a float64 value can round to the neighbour of the one the GPU's float32 value
rounds to.  Each constant states the worst error measured on one H100 80GB HBM3 and the margin over it."""
import collections
import functools
import gc
import json
import math
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np
import torch

import oracle_logprobs as olp
import wb200  # noqa: F401
from oracle import audio as o_audio, model as o_model, synth, transcribe as o_tr
from whisper_burn_b200 import ffi, model, transcribe
from whisper_burn_b200.synth import WhisperDims

G = Path(__file__).resolve().parent / "golden"

# ---------------------------------------------------------------- tolerances of the float64 suite (1 audio, 2 text layers)
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

# ---------------------------------------------------------------- tolerances of the depth suite (3 to 32 layers)
# Worst errors measured on one H100 80GB HBM3 (700 W power limit) at 3 to 32 layers; each constant keeps a 3x margin or
# more.  The error grows with depth and width: none of these fit the float64 suite's constants with that margin.
# greedy top-1 log-prob (and the log-probs of decoded greedy and beam paths).  Worst: f32 9.8e-6 (decoder5, d = 1280,
# L = 32, 9 rows), 3.0x; f16 4.5e-4 (the same case), 3.3x
DEEP_GREEDY_LP_TOL = {"f32": 3e-5, "f16": 1.5e-3}
# wb_session_step, all 7 candidates.  Worst: f32 2.1e-6 (decoder3, d = 384, L = 4), 4.7x (the float64 suite's
# constant); f16 2.9e-4 (decoder5, d = 512, L = 6), 3.4x
DEEP_STEP_LP_TOL = {"f32": STEP_LP_TOL["f32"], "f16": 1e-3}
# score_tokens.  Worst: f32 1.8e-5 (d = 1280, L = 32), 3.4x; f16 7.0e-4 (d = 1024, L = 24), 3.6x
DEEP_SCORE_LP_TOL = {"f32": 6e-5, "f16": 2.5e-3}
# forward_decoder logits at 448 positions, relative to scale.  Worst 1.35e-5 (decoder5, d = 512, L = 6), 3.7x
DEEP_LOGITS_REL_TOL = 5e-5
# encoder output, relative to scale.  Worst 2.0e-5 (tensor-core, d = 1280, L = 32), 3.5x
DEEP_ENC_REL_TOL = 7e-5


# GPU log-probs against the float32 oracle's at real shapes (fixtures of tests/golden): fp32 rounding through 12 to 32
# layers on log-probs of magnitude ~10
REAL_LP_TOL = 2e-4


# ---------------------------------------------------------------- small helpers
def is_special_of(sp):
    return (np.arange(sp.n_vocab) >= sp.first_special).astype(np.uint8)


def kv_code(kv):
    return ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32


def rel_to_scale(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def report(what, worst, tol):
    print(f"\n[f64] {what}: worst {worst:.3e} (tolerance {tol:.0e})")


def use_decoder(monkeypatch, n):
    if n:
        monkeypatch.setenv("WB200_DECODER", str(n))
    else:
        monkeypatch.delenv("WB200_DECODER", raising=False)


@functools.lru_cache(maxsize=None)
def golden(name):
    """tests/golden/<name>.json, read once (callers must not change it)"""
    return json.loads((G / f"{name}.json").read_text())


# ---------------------------------------------------------------- inputs
N_OF_T = {6: 400, 64: 18720, 65: 19040, 750: 480000}   # waveform samples giving each encoder length
T_ORDER = (750, 6, 65, 64)                             # T = (min(n // 160, 1490) + 10 - 1) // 2 + 1 for n samples


def windows(n, seed, order=T_ORDER):
    Ts = [order[i % len(order)] for i in range(n)]
    return Ts, [synth.waveform(N_OF_T[T], seed=seed + i) for i, T in enumerate(Ts)]


def pool_waves(gold, n):
    """n windows of chunk 0 cycling through gold["pool"] (tokens_beam.json: T = 750, 6, 314, 65, 750, 314)"""
    chunk = synth.chunk_waveform(0)
    return [chunk[off:off + m] for off, m in (gold["pool"][i % len(gold["pool"])] for i in range(n))]


def real_windows(name, kv, chunks=None):
    """(waves, records) of the windows of tests/golden/tokens_real.json's model `name` in chunks (default: all of them), with
    the records of K/V type kv"""
    g = golden("tokens_real")[name]["chunks"]
    waves, recs = [], []
    for c in range(len(g)) if chunks is None else chunks:
        chunk = synth.chunk_waveform(c)
        for (s, e), r in zip(g[c]["bounds"], g[c][kv]):
            waves.append(chunk[s:e])
            recs.append(r)
    return waves, recs


def check_ids_where_separated(got, recs, tol=1e-4):
    """ids identical up to the first step whose oracle top-1/top-2 log-prob gap ("margins") is below tol (there fp32
    rounding decides; 24 windows x 100 steps of the synthetic tiny.en model contain 4 such steps, smallest gap 3e-6)."""
    for i, (g, r) in enumerate(zip(got, recs)):
        want = r["tokens"]
        n = next((4 + s for s, v in enumerate(r.get("margins", [])) if v < tol), len(want))
        assert g[:n] == want[:n], f"window {i}: first difference at {next(j for j in range(n) if g[j] != want[j])} (compared {n} ids)"
        if n == len(want):
            assert g == want, f"window {i}: {g} vs {want}"


def encoder_outputs64(sess, Ts):
    out = []
    for r, T in enumerate(Ts):
        xa = sess.get_encoder_output(r)
        assert xa.shape[0] == T, f"window {r}: {xa.shape[0]} encoder positions, not {T}"
        out.append(torch.from_numpy(xa).double()[None])
    return out


# ---------------------------------------------------------------- synthetic models
def synthetic(dims_or_name, seed, exact=True, f64=True):
    """(dims, float32 numpy weights, torch weights, float64 weights or None without f64) of synth.make_weights"""
    dims, w_np, w_t = synth.make_weights(dims_or_name, seed=seed)
    if not exact:
        w_np = {k: (v * np.float32(1.0001) if v.ndim else v) for k, v in w_np.items()}
        w_t = synth.to_torch(w_np)
    return dims, w_np, w_t, o_model.as_dtype(w_t) if f64 else None


@functools.lru_cache(maxsize=2)
def shallow_weights(d, H, V, n_text_layer, exact):
    """synthetic() of the float64 suite's model: 1 audio layer, seed d + V"""
    return synthetic(WhisperDims(80, 1500, d, H, 1, V, 448, d, H, n_text_layer), d + V, exact)


_held = {}


def deep_weights(d, V, n_audio_layer, n_text_layer, exact=True):
    """synthetic() of the depth suite's model (d // 64 heads), one model at a time: a float64 d = 1280, 32-layer decoder is
    ~7 GB, so the previous model is dropped before the next is made (an lru_cache would make the new one first)."""
    key = (d, V, n_audio_layer, n_text_layer, exact)
    if key not in _held:
        _held.clear()
        gc.collect()
        dims = WhisperDims(80, 1500, d, d // 64, n_audio_layer, V, 448, d, d // 64, n_text_layer)
        _held[key] = synthetic(dims, d + V + 100 * n_audio_layer + n_text_layer, exact)
    return _held[key]


def whisper(dims, w_np, exact=True, ln_eps_outside=True):
    """A fresh model.Whisper per call: its stateless forward session reads WB200_DECODER when it is created."""
    wh = model.Whisper(dims, w_np, ln_eps_outside=ln_eps_outside)
    assert wh.weights_fp16_exact == exact, f"weights_fp16_exact is {wh.weights_fp16_exact}, not {exact}"
    return wh


def make_model(d, H, V, exact=True, n_text_layer=2):
    """(dims, GPU model, float64 weights) of shallow_weights"""
    dims, w_np, _, w64 = shallow_weights(d, H, V, n_text_layer, exact)
    return dims, whisper(dims, w_np, exact), w64


def make_deep_model(d, V, n_audio_layer=1, n_text_layer=1, exact=True):
    """(dims, GPU model, float64 weights) of deep_weights: a deep decoder (n_audio_layer = 1) or a deep encoder
    (n_text_layer = 1)"""
    dims, w_np, _, w64 = deep_weights(d, V, n_audio_layer, n_text_layer, exact)
    return dims, whisper(dims, w_np, exact), w64


Named = collections.namedtuple("Named", "dims sp wh w_np w_t w64")


def named_model(name, f64=False):
    """The seed-0 synthetic model `name` with its special tokens and a fresh model.Whisper; float64 weights with f64."""
    dims, w_np, w_t, w64 = synthetic(name, 0, f64=f64)
    return Named(dims, synth.special_tokens(dims), model.Whisper(dims, w_np), w_np, w_t, w64)


# ---------------------------------------------------------------- float64 reference rows
def path_rows(w64, dims, sp, xa, ids, kv="f32", n_prompt=4, ln_eps_mode="outside", unmask=False):
    """The float64 log-softmax rows [len(ids) - n_prompt, V] the search evaluated along the decoded path ids (prompt first),
    by the cached decoder (greedy_path_log_probs): row j picked ids[n_prompt + j], with the beam rule's special-token mask
    of sp, or none with unmask (the greedy loop).  xa: the window's [1, T, d]."""
    opts = o_model.OracleOptions(ln_eps_mode=ln_eps_mode, kv_dtype=kv)
    return o_tr.greedy_path_log_probs(w64, dims, olp.unmasked(sp) if unmask else sp, xa, ids, n_prompt=n_prompt,
                                      opts=opts).numpy()


def along(rows, ids, n_prompt=4):
    """The log-prob of every generated id of ids in the path_rows row that picked it."""
    return np.array([float(rows[j - n_prompt][ids[j]]) for j in range(n_prompt, len(ids))])


def forward_rows(w64, dims, xa, seqs, kv="f32", ln_eps_mode="outside", sp=None, steps=None):
    """Float64 log-softmax rows of whole sequences by one teacher-forced oracle.model.forward_decoder per window length: the
    same arithmetic as the cached decoder, with the weights read once per batch rather than once per step.  xa: per
    sequence its window's [1, T, d]; sequences on windows of one length run as one batch, padded at the end (which the
    causal mask keeps from earlier positions).

    Without steps: per sequence the rows of every position, [len, V] (row j scores seqs[r][j + 1]).
    With steps: seqs are decoded paths (prompt of 4 ids first, the last id not fed) and per path the result is {s: row}
    for the steps s of steps[r], the row that picked seqs[r][3 + s], with sp's special-token mask where the beam rule
    applies it."""
    opts = o_model.OracleOptions(ln_eps_mode=ln_eps_mode, kv_dtype=kv)
    fed = seqs if steps is None else [p[:-1] for p in seqs]
    maskout = torch.from_numpy(sp.maskout()).double() if steps is not None else None
    by_T = {}
    for r, x in enumerate(xa):
        by_T.setdefault(x.shape[1], []).append(r)
    out = [None] * len(seqs)
    for rs in by_T.values():
        n = max(len(fed[r]) for r in rs)
        toks = torch.tensor([fed[r] + [0] * (n - len(fed[r])) for r in rs], dtype=torch.int64)
        logits = o_model.forward_decoder(w64, dims, toks, torch.cat([xa[r] for r in rs]), opts)
        for i, r in enumerate(rs):
            if steps is None:
                out[r] = o_model.log_softmax_last(logits[i:i + 1])[0].numpy()
                continue
            rows = {}
            for s in steps[r]:
                row = logits[i, s + 2]
                if o_tr.masks_specials(s + 3):
                    row = row + maskout
                rows[s] = o_model.log_softmax_last(row).numpy()
            out[r] = rows
    return out


def greedy_ref_rows(model_key, sp, xa, tokens, kv, steps):
    """In a worker process: the float64 log-prob rows of the greedy steps `steps` along `tokens` (path_rows on the weights
    shallow_weights(*model_key) and the window's encoder output xa [T, d])."""
    dims, _, _, w64 = shallow_weights(*model_key)
    ref = path_rows(w64, dims, sp, torch.from_numpy(xa)[None], tokens, kv)
    return {s: ref[s - 1] for s in steps}


@functools.lru_cache(maxsize=1)
def ref_pool():
    """Worker processes for the float64 reference: scoring one row is a few hundred small sequential float64 steps, so rows
    run side by side, one torch thread each."""
    return ProcessPoolExecutor(max(1, min(8, (os.cpu_count() or 2) - 1)), mp_context=multiprocessing.get_context("spawn"),
                               initializer=torch.set_num_threads, initargs=(1,))


# ---------------------------------------------------------------- the oracle alone: checks that can fail
MARGIN = 10   # a mistake a GPU check must notice moves what it compares by at least MARGIN times its tolerance


def check_moves(moved, tol, what, tag):
    """moved: change -> how far it moves the quantity; every one at least MARGIN * tol"""
    short = {k: v for k, v in moved.items() if v < MARGIN * tol}
    least = min(moved, key=moved.get)
    print(f"\n[{tag}] {what}: smallest move {moved[least]:.2e} ({least}), {moved[least] / tol:.0f}x the tolerance {tol:.0e}")
    assert not short, f"{what}: moved less than {MARGIN}x {tol:.0e}: {short}"


def window_mel(dims, T=65):
    """the float64 padded mel of the window of T encoder positions (waveform seed T)"""
    mel = o_tr.pad_mel(o_audio.prep_audio(torch.from_numpy(synth.waveform(N_OF_T[T], seed=T))[None]), dims.n_audio_ctx)
    return mel.double()


def greedy_path(w64, dims, sp, xa, opts):
    """the oracle's greedy ids (beam-rule mask) from the prompt, DEPTH steps or to EOT"""
    dec = o_model.CachedDecoder(w64, dims, xa, opts)
    toks = list(sp.prompt())
    for t in toks[:-1]:
        dec.step(torch.tensor([t], dtype=torch.int64))
    maskout = torch.from_numpy(sp.maskout())
    while len(toks) < 4 + DEPTH and toks[-1] != sp.eot:
        logits = dec.step(torch.tensor([toks[-1]], dtype=torch.int64))
        if o_tr.masks_specials(len(toks)):
            logits = logits + maskout
        toks.append(int(logits.argmax()))
    return toks


# ---------------------------------------------------------------- encoder against float64
def encoder_error(sess, w64, dims, Ts, tol, opts=o_model.DEFAULT_OPTS):
    """The worst relative-to-scale error of the session's encoder output of every window (T encoder positions each) against
    the float64 encoder of its padded mel, each within tol."""
    worst = 0.0
    for w, T in enumerate(Ts):
        got = sess.get_encoder_output(w)
        assert got.shape == (T, dims.n_audio_state), f"window {w}: encoder output of shape {got.shape}"
        mel = torch.from_numpy(sess.get_mel(w)).double()[None]
        e = rel_to_scale(got, o_model.forward_encoder(w64, dims, mel, opts)[0].numpy())
        worst = max(worst, e)
        assert e < tol, f"window {w} (T = {T}): {e}"
    return worst


# ---------------------------------------------------------------- greedy, per step, top-1 against float64
def edge_steps(edges, max_text_len):
    """The greedy steps whose self attention runs over E - 1, E and E + 1 keys for every edge E, and the last step a session
    of max_text_len allows (step s attends over n = s + 3 keys: the 4-id prompt and s - 1 generated ids)."""
    last = max_text_len - 4
    return tuple(sorted({s for e in edges for s in (e - 4, e - 3, e - 2) if s <= last} | {last}))


def check_greedy(dims, wh, kv, n_rows, decoder, seed, steps=SHALLOW_STEPS, max_text_len=None, full_depth=False, tol=None,
                 ref_rows=None, inputs=None, mode="reference"):
    """Greedy-decodes n_rows windows once to the deepest step of `steps` and once to each step s of `steps`, and checks the
    top-1 (id, log-prob) of every row at every step s against float64 on the GPU's own path.  max_text_len defaults to the
    deepest step plus the prompt and one.  full_depth: EOT is declared to be a special id past the named ones that no row
    emits (the largest one not emitted by an earlier full-depth launch that a row stopped in), and every row must reach the
    deepest step.  tol defaults to GREEDY_LP_TOL[kv].  ref_rows(sp, xa, paths, kv, steps) -> per row {s: float64 log-prob
    row} computes the reference in this process (xa: the rows' float64 encoder outputs [1, T, d], steps: per row); by
    default worker processes rebuild the model with shallow_weights.  inputs: (Ts, waves) in place of windows(n_rows, seed),
    for a session of windowing `mode`.  Returns the worst |log-prob error|."""
    depth = max(steps)
    sp = synth.special_tokens(dims)
    bitmap = sp.is_special_bitmap()
    Ts, waves = inputs or windows(n_rows, seed)
    sess = transcribe.Session(wh, max_windows=n_rows, max_beams=1, max_text_len=max_text_len or 4 + depth + 1,
                              kv_dtype=kv_code(kv), windows=mode)
    full = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=depth) if not full_depth else None
    eot = sp.n_vocab
    while full is None or (full_depth and any(len(t) < 4 + depth for t in full)):
        eot = max(set(range(sp.first_special, eot)) - {i for t in full or [] for i in t})
        sp = o_tr.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, eot, sp.first_special, sp.n_vocab)
        full = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=depth)
    assert sess.last_decoder() == decoder, f"decoder{sess.last_decoder()} ran, not decoder{decoder}"
    if full_depth:
        assert sess.last_steps() == depth and [len(t) for t in full] == [4 + depth] * n_rows, \
            f"{sess.last_steps()} steps, lengths {[len(t) for t in full]}: not every row reached step {depth}"
    xa = encoder_outputs64(sess, Ts)
    row_steps = [[s for s in steps if 4 + s <= len(full[r])] for r in range(n_rows)]
    if ref_rows is None:
        key = (dims.n_text_state, dims.n_text_head, dims.n_vocab, dims.n_text_layer, wh.weights_fp16_exact)
        refs = [ref_pool().submit(greedy_ref_rows, key, sp, xa[r][0].numpy(), full[r], kv, row_steps[r]) for r in range(n_rows)]
    got = [dict() for _ in range(n_rows)]      # step -> (id, log-prob) of every row that produced a token at that step
    for s in steps:
        toks = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=s)
        assert sess.last_decoder() == decoder, f"step {s}: decoder{sess.last_decoder()} ran, not decoder{decoder}"
        ids, lps = sess.last_topk(n_rows, 1)
        for r in range(n_rows):
            assert toks[r] == full[r][:len(toks[r])], f"row {r}: the depth-{s} launch is not a prefix of the depth-{depth} one"
            if len(toks[r]) == 4 + s:
                assert int(ids[r, 0]) == toks[r][-1], f"row {r} step {s}: last_topk id {int(ids[r, 0])} vs {toks[r][-1]}"
                got[r][s] = float(lps[r, 0])
    tol = tol or GREEDY_LP_TOL[kv]
    worst = 0.0
    local = ref_rows(sp, xa, full, kv, row_steps) if ref_rows is not None else None
    for r in range(n_rows):
        ref = local[r] if local is not None else refs[r].result()
        assert sorted(got[r]) == sorted(ref), f"row {r}: steps {sorted(got[r])} vs float64 steps {sorted(ref)}"
        for s, lp in got[r].items():
            tok = full[r][4 + s - 1]
            err = abs(lp - ref[s][tok])
            worst = max(worst, err)
            assert err < tol, f"row {r} (T = {Ts[r]}) step {s}: log-prob {lp} vs float64 {ref[s][tok]}"
            gap = ref[s].max() - ref[s][tok]       # the GPU id is the float64 argmax up to a near-tie
            assert gap < tol, f"row {r} step {s}: id {tok} is {gap} below the float64 argmax {int(ref[s].argmax())}"
    return worst


# ---------------------------------------------------------------- wb_session_step, k = 7, with beams
def check_step_k7(dims, wh, w64, decoder, kv, sess=None, tol=None, out=None):
    """wb_session_step with k = 7 on two windows: fanned out from one parent per window, then continued from different
    parents so the ancestry table is exercised; all 7 (id, log-prob) pairs against float64 oracle.model.CachedDecoder rows
    reordered the same way, on `sess` (default: a fresh session of 2 windows, 5 beams, max_text_len 16), each within tol
    (default STEP_LP_TOL[kv]).  out, a list, receives every step's (ids, log-probs).  Returns the worst |log-prob error|."""
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
        assert sess.last_decoder() == decoder, f"decoder{sess.last_decoder()} ran, not decoder{decoder}"
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


# ---------------------------------------------------------------- full logits at the maximum text length
def forward_decoder_448_error(dims, wh, w64):
    """The worst relative-to-scale error of forward_decoder's logits at every one of n_text_ctx positions."""
    d = dims.n_text_state
    rng = np.random.default_rng(d)
    xa = rng.standard_normal((1, 65, d)).astype(np.float32)
    toks = rng.integers(0, dims.n_vocab, size=(1, dims.n_text_ctx)).astype(np.int64)
    got = wh.forward_decoder(toks, xa)
    want = o_model.forward_decoder(w64, dims, torch.from_numpy(toks), torch.from_numpy(xa).double()).numpy()
    return max(rel_to_scale(got[0, p], want[0, p]) for p in range(dims.n_text_ctx))


# ---------------------------------------------------------------- scoring: sequences and their rows against float64
GAP = 1e-4         # arg-max compared where the reference's top-1 / top-2 gap is at least this
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 448)   # around the scorer's 64-row tiles up to n_text_ctx


def random_seqs(V, seed, lengths=LENGTHS):
    rng = np.random.default_rng(seed)
    return [[int(t) for t in rng.integers(0, V, size=n)] for n in lengths]


def masked_seqs(sp, seed):
    """prompt + ids with special ids at j = 4, 5 (masked: -inf), 6 and 9 (not masked)"""
    rng = np.random.default_rng(seed)
    specials = list(range(sp.first_special, sp.n_vocab))
    seqs = []
    for r in range(4):
        body = [int(t) for t in rng.integers(0, sp.first_special, size=20 + 7 * r)]
        body[0], body[1], body[2], body[5] = specials[r], specials[r + 1], specials[r + 2], specials[r + 3]
        seqs.append(list(sp.prompt()) + body)
    return seqs


def check_rows(lp, am, ref, seq, kv, what, tol=None):
    """lp / argmax of one sequence against its float64 rows, within tol (default GREEDY_LP_TOL[kv]; a tol given compares
    arg-maxes only where the float64 top-1 / top-2 gap is at least 2 tol as well); returns the worst |error|"""
    assert lp[0] == 0.0 and am[0] == -1, f"{what}: position 0 is ({lp[0]}, {am[0]}), not (0, -1)"
    if len(seq) == 1:
        return 0.0
    want = np.array([ref[j - 1][seq[j]] for j in range(1, len(seq))])
    err = float(np.abs(lp[1:].astype(np.float64) - want).max())
    assert err < (tol or GREEDY_LP_TOL[kv]), f"{what}: worst log-prob error {err}"
    gap = GAP if tol is None else max(GAP, 2 * tol)
    for j in range(1, len(seq)):
        top2 = np.sort(ref[j - 1])[-2:]
        if top2[1] - top2[0] >= gap:
            assert am[j] == int(ref[j - 1].argmax()), f"{what} position {j}: arg-max {am[j]} vs {int(ref[j - 1].argmax())}"
    return err


# ---------------------------------------------------------------- per-token log-probs of a transcription
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


def check_against_f64(sess, w64, dims, sp, ids, lps, kv, unmask=False, skip_nan=False, ln_eps_mode="outside"):
    """Every row's log-probs lps[r] past the prompt against float64 teacher forcing of its ids (path_rows) on the session's
    encoder output, within GREEDY_LP_TOL[kv]; returns the worst |error|."""
    worst = 0.0
    for r, t in enumerate(ids):
        xa = torch.from_numpy(sess.get_encoder_output(r)).double()[None]
        ref = along(path_rows(w64, dims, sp, xa, t, kv, ln_eps_mode=ln_eps_mode, unmask=unmask), t)
        got = lps[r][4:].astype(np.float64)
        ok = ~np.isnan(got) if skip_nan else np.ones(len(got), bool)
        err = np.abs(got[ok] - ref[ok]).max(initial=0.0)
        worst = max(worst, float(err))
        assert err < GREEDY_LP_TOL[kv], f"row {r}: log-probs {got} vs float64 {ref}"
    return worst


# ---------------------------------------------------------------- the greedy loop's cases (WB_SEARCH_GREEDY_LOOP)
LOOP_GAP_TOL = 1e-4
LOOP_EOT_ID = 500   # declared EOT of the synthetic models: an ordinary id whose logit is sometimes within ln 2 of the arg-max
# (decoder, model, windows, max_text_len, rules that end some window): decoder6 takes t_max <= 128 and 8+ rows here;
# decoder5 needs d % 256 == 0 (test-c, whose logits never put id 500 within ln 2 of the arg-max on these windows)
_ALL_RULES = {"eot", "repeat", "context"}
LOOP_CASES = [(4, "test-a", 4, 448, _ALL_RULES), (6, "test-a", 9, 128, _ALL_RULES), (5, "test-c", 4, 448, {"repeat", "context"}),
              (3, "test-a", 4, 448, _ALL_RULES)]


@functools.lru_cache(maxsize=None)
def loop_model(name):
    """named_model(name), one per process: the greedy-loop tests and their oracle caches share it"""
    return named_model(name)


def loop_window(i):
    return synth.waveform(16000 * (3 + 4 * (i % 4)) + 1600 * (i // 4), seed=100 + i)


def loop_session(name, n, t_max, kv, search="greedy_loop"):
    return transcribe.Session(loop_model(name).wh, max_windows=n, max_beams=1, max_text_len=t_max, kv_dtype=kv_code(kv),
                              search=search)


def same_up_to_ties(got, want, tr):
    """got == want, or identical up to the first step whose EOT-test or top-1/top-2 gap is below LOOP_GAP_TOL."""
    if got == want:
        return True
    for s, (e, t) in enumerate(zip(tr["eot_gap"], tr["top_gap"])):
        if abs(e) < LOOP_GAP_TOL or t < LOOP_GAP_TOL:
            return got[:4 + s] == want[:4 + s]
    return False
