"""The per-LayerNorm-eps models of test_layernorm_eps_cpu.py and test_layernorm_eps_gpu.py.

synth.make_weights_np gives every LayerNorm eps = 1e-5, so a kernel that reads another LayerNorm's eps, hard-codes 1e-5 or
falls back to a default computes the same bits as a correct one.  These are the real-width models of the float64 tests
(harness.shallow_weights) with every LayerNorm given its own eps, a power of two (the same number in float32 and
float64), in the order of the sorted /eps keys:

  * decoder: 2^-11, 2^-4, 2^-9, 2^-8, 2^-3, 2^-6, 2^-5 (block_0/attn_ln, block_0/cross_attn_ln, block_0/mlp_ln,
    block_1/..., decoder/ln; the first four with one text layer): 2^-11 ... 2^-5 in order, except that the cross-attention
    LayerNorms get 2^-4 and 2^-3, where 2^-10 and 2^-7 moved the d = 128 greedy log-probs too little
    (test_layernorm_eps_cpu.py);
  * encoder: 2^-8, 2^-6, 2^-4 (block_0/attn_ln, block_0/mlp_ln, ln_post).

Both placements are run: "outside" (x - mean) / (sqrt(var) + eps), the default, and "inside" (x - mean) / sqrt(var + eps)."""
import functools

import numpy as np
import torch

import harness as h

MODES = ("outside", "inside")
DEC_EPS = tuple(2.0 ** e for e in (-11, -4, -9, -8, -3, -6, -5))
ENC_EPS = (2.0 ** -8, 2.0 ** -6, 2.0 ** -4)


def eps_keys(w):
    """(encoder /eps keys, decoder /eps keys), each sorted"""
    keys = sorted(k for k in w if k.endswith("/eps"))
    return [k for k in keys if k.startswith("encoder/")], [k for k in keys if k.startswith("decoder/")]


def scheme(w):
    """/eps key -> the eps this module gives that LayerNorm"""
    enc, dec = eps_keys(w)
    assert len(enc) == len(ENC_EPS) and len(dec) <= len(DEC_EPS), (enc, dec)
    return {**dict(zip(enc, ENC_EPS)), **dict(zip(dec, DEC_EPS))}


def with_eps(w_np, w64, eps):
    """Copies of the float32 and float64 weight dicts with the /eps entries of `eps` replaced (the inputs are cached and
    shared with other tests: never changed in place)."""
    w_np = dict(w_np)
    w64 = dict(w64)
    for k, v in eps.items():
        w_np[k] = np.float32(v)
        w64[k] = torch.tensor(float(np.float32(v)), dtype=torch.float64)
    return w_np, w64


@functools.lru_cache(maxsize=4)
def weights(d, H, V, n_text_layer=2, exact=True):
    """(dims, float32 weights, float64 weights) of harness.shallow_weights with the per-LayerNorm eps of this module"""
    dims, w_np, _, w64 = h.shallow_weights(d, H, V, n_text_layer, exact)
    return (dims, *with_eps(w_np, w64, scheme(w_np)))


def make_model(d, H, V, mode, exact=True, n_text_layer=2):
    """(dims, float32 weights, GPU model in placement `mode`, float64 weights) of weights()"""
    dims, w_np, w64 = weights(d, H, V, n_text_layer, exact)
    return dims, w_np, h.whisper(dims, w_np, exact, ln_eps_outside=mode == "outside"), w64
