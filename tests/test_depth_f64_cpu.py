"""The float64 oracle alone: the deep models of test_depth_f64_gpu.py make its checks able to fail.  On the same models at 3,
4 and 6 layers, each of these layer-indexing mistakes moves the quantity a GPU test compares by at least MARGIN times the
tolerance it is compared with:

  * layer l + 1's Wqkv (query, key, value weights and biases) used in layer l, for every l < L - 1 (a weight stream one
    layer ahead);
  * layer 0's Wqkv used in layer l + 1, for every l + 1 >= 1 (the wrap to the next position's layer 0 taken too early);
  * one middle layer's MLP bias left out (mlp1 or mlp2, the partial sums the next LayerNorm stage folds);
  * two layers' LayerNorm parameters (weight and bias) swapped, for every pair of layers and every LayerNorm of a block.

The quantities: the teacher-forced log-probs of the oracle's own DEPTH-step greedy path on one fixed encoder output against
the fp32 K/V harness.DEEP_GREEDY_LP_TOL, and the encoder output (relative to its scale) against harness.DEEP_ENC_REL_TOL.
Against the fp16 K/V tolerance (50 times larger) nothing is claimed: a left-out MLP bias moves the log-probs by less."""
import itertools

import numpy as np
import pytest
import torch

import harness as h
from harness import check_moves, greedy_path, window_mel
from oracle import model as o_model, synth

V = 2051
QKV = ("query/weight", "query/bias", "key/weight", "value/weight", "value/bias")


def moved_block(w, src, dst, names):
    """a copy of w with block dst's entries `names` taken from block src"""
    w = dict(w)
    for n in names:
        w[f"{dst}/{n}"] = w[f"{src}/{n}"]
    return w


def swapped(w, a, b, names):
    """a copy of w with blocks a and b's entries `names` exchanged"""
    w = dict(w)
    for n in names:
        w[f"{a}/{n}"], w[f"{b}/{n}"] = w[f"{b}/{n}"], w[f"{a}/{n}"]
    return w


def changes(w, prefix, L, lns):
    """(what, weights) of every mistake of the module docstring in the blocks `prefix`/block_*"""
    b = [f"{prefix}/block_{i}" for i in range(L)]
    qkv = [f"attn/{n}" for n in QKV]
    out = [(f"layer {l + 1}'s Wqkv in layer {l}", moved_block(w, b[l + 1], b[l], qkv)) for l in range(L - 1)]
    out += [(f"layer 0's Wqkv in layer {l}", moved_block(w, b[0], b[l], qkv)) for l in range(1, L)]
    for n in ("mlp1", "mlp2"):
        key = f"{b[L // 2]}/mlp/{n}/bias"
        out.append((f"no {key}", {**w, key: torch.zeros_like(w[key])}))
    for ln, (i, j) in itertools.product(lns, itertools.combinations(range(L), 2)):
        out.append((f"{ln} of layers {i} <-> {j}", swapped(w, b[i], b[j], (f"{ln}/weight", f"{ln}/bias"))))
    return out


def check(moved, tol, what):
    check_moves(moved, tol, what, "depth")


def path_log_probs(w64, dims, sp, xa, toks):
    rows = h.forward_rows(w64, dims, [xa], [toks], sp=sp, steps=[range(1, len(toks) - 3)])[0]
    return np.array([rows[s][toks[3 + s]] for s in rows])


@pytest.mark.parametrize("d,L", [(384, 3), (384, 4), (512, 6)])
def test_decoder_log_probs_move(d, L):
    dims, _, _, w64 = h.deep_weights(d, V, 1, L)
    sp = synth.special_tokens(dims)
    xa = o_model.forward_encoder(w64, dims, window_mel(dims))
    toks = greedy_path(w64, dims, sp, xa, o_model.DEFAULT_OPTS)
    assert len(toks) == 4 + h.DEPTH, toks
    base = path_log_probs(w64, dims, sp, xa, toks)
    moved = {what: float(np.abs(path_log_probs(w, dims, sp, xa, toks) - base).max())
             for what, w in changes(w64, "decoder", L, ("attn_ln", "cross_attn_ln", "mlp_ln"))}
    check(moved, h.DEEP_GREEDY_LP_TOL["f32"], f"greedy path d={d} L={L}")


@pytest.mark.parametrize("d,L", [(384, 4), (512, 6)])
def test_encoder_output_moves(d, L):
    dims, _, _, w64 = h.deep_weights(d, V, L, 1)
    mel = window_mel(dims)
    base = o_model.forward_encoder(w64, dims, mel)[0].numpy()
    moved = {what: h.rel_to_scale(o_model.forward_encoder(w, dims, mel)[0].numpy(), base)
             for what, w in changes(w64, "encoder", L, ("attn_ln", "mlp_ln"))}
    check(moved, h.DEEP_ENC_REL_TOL, f"encoder d={d} L={L}")
