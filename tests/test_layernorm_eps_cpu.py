"""The float64 oracle alone: the per-LayerNorm-eps models of tests/layernorm_eps.py make test_layernorm_eps_gpu.py able to
fail.  For each placement and every width the GPU tests use, each of these changes to the model moves the quantity a GPU test
compares by at least MARGIN times the tolerance it is compared with:

  * the other placement;
  * any one LayerNorm's eps reset to 1e-5 (a hard-coded or default eps);
  * any two LayerNorms' eps swapped within the encoder or within the decoder (a kernel reading another LayerNorm's eps).

The quantities: the encoder output (relative to its scale) against harness.ENC_REL_TOL; the teacher-forced log-probs of the
oracle's own DEPTH-step greedy path, and the log-probs of every position of the scoring test's sequences, against the fp32
K/V harness.GREEDY_LP_TOL.  The decoder quantities are computed on one fixed encoder output, as the GPU tests check the decoders on the
GPU's own.  With the fp16 K/V tolerance (25 times larger) only the placement is claimed."""
import itertools

import numpy as np
import pytest

import harness as h
import layernorm_eps as lne
from harness import check_moves, greedy_path, random_seqs, window_mel
from oracle import model as o_model, synth

V = 2051
T = 65


def changes(eps, keys, mode):
    """(what, eps dict, placement) of every change the GPU tests must notice, among the LayerNorms `keys`"""
    out = [("the other placement", eps, "inside" if mode == "outside" else "outside")]
    out += [(f"{k} = 1e-5", {**eps, k: 1e-5}, mode) for k in keys]
    out += [(f"{a} <-> {b}", {**eps, a: eps[b], b: eps[a]}, mode) for a, b in itertools.combinations(keys, 2)]
    return out


def check(moved, tol, what):
    check_moves(moved, tol, what, "eps")


@pytest.mark.parametrize("mode", lne.MODES)
@pytest.mark.parametrize("d,H", [(384, 6), (768, 12)])
def test_encoder_output_moves(d, H, mode):
    dims, w_np, w64 = lne.weights(d, H, V, n_text_layer=1)
    mel = window_mel(dims)
    base = o_model.forward_encoder(w64, dims, mel, o_model.OracleOptions(ln_eps_mode=mode))[0].numpy()
    assert base.shape[0] == T
    eps = lne.scheme(w_np)
    moved = {}
    for what, e, m in changes(eps, lne.eps_keys(w_np)[0], mode):
        _, w = lne.with_eps(w_np, w64, e)
        got = o_model.forward_encoder(w, dims, mel, o_model.OracleOptions(ln_eps_mode=m))[0].numpy()
        moved[what] = h.rel_to_scale(got, base)
    check(moved, h.ENC_REL_TOL, f"encoder d={d} {mode}")


def path_log_probs(w64, dims, sp, xa, toks, mode):
    return h.along(h.path_rows(w64, dims, sp, xa, toks, ln_eps_mode=mode), toks)


def scored_log_probs(w64, dims, xa, seqs, mode):
    out = []
    for seq in seqs:
        rows = h.forward_rows(w64, dims, [xa], [seq], ln_eps_mode=mode)[0]
        out.append(rows[np.arange(len(seq) - 1), seq[1:]])
    return np.concatenate(out)


@pytest.mark.parametrize("mode", lne.MODES)
@pytest.mark.parametrize("d,H", [(128, 2), (256, 4), (384, 6)])
def test_decoder_log_probs_move(d, H, mode):
    """The greedy path at every decoder width, and at d = 384 the scoring pass's sequences, on one encoder output."""
    dims, w_np, w64 = lne.weights(d, H, V)
    sp = synth.special_tokens(dims)
    xa = o_model.forward_encoder(w64, dims, window_mel(dims), o_model.OracleOptions(ln_eps_mode=mode))
    toks = greedy_path(w64, dims, sp, xa, o_model.OracleOptions(ln_eps_mode=mode))
    assert len(toks) == 4 + h.DEPTH, toks
    base = path_log_probs(w64, dims, sp, xa, toks, mode)
    seqs = [s for s in random_seqs(V, d) if len(s) > 1] if d == 384 else []
    base_scored = scored_log_probs(w64, dims, xa, seqs, mode) if seqs else None
    moved, moved_scored = {}, {}
    for what, e, m in changes(lne.scheme(w_np), lne.eps_keys(w_np)[1], mode):
        _, w = lne.with_eps(w_np, w64, e)
        moved[what] = float(np.abs(path_log_probs(w, dims, sp, xa, toks, m) - base).max())
        if seqs:
            moved_scored[what] = float(np.abs(scored_log_probs(w, dims, xa, seqs, m) - base_scored).max())
    flip = "the other placement"
    for tol in h.GREEDY_LP_TOL.values():
        check({flip: moved[flip]}, tol, f"greedy path d={d} {mode}, placement")
    check(moved, h.GREEDY_LP_TOL["f32"], f"greedy path d={d} {mode}")
    if seqs:
        for tol in h.GREEDY_LP_TOL.values():
            check({flip: moved_scored[flip]}, tol, f"scored sequences d={d} {mode}, placement")
        check(moved_scored, h.GREEDY_LP_TOL["f32"], f"scored sequences d={d} {mode}")
