"""Oracle restatement of the Whisper model graph (reference: src/model/mod.rs).

TEST INFRASTRUCTURE (see oracle/__init__.py).  PyTorch-CPU fp32, or float64 when the weights and inputs are float64
(``as_dtype``): the same graph with the rounding of the GPU's fp32 arithmetic removed.  Weights are a flat dict
keyed by the reference's own npy-tree paths (src/model/load.rs:19-310, python/dump.py:
130-213), e.g. ``encoder/block_0/attn/query/weight`` with Linear weights in burn layout
``[d_in, d_out]`` (dump.py:141-145) and Conv1d weights ``[out, in, k]`` (load.rs:145-161).

Two decoders are provided:
  * ``forward_decoder``   -- the reference's stateless full recompute (mod.rs:131-157);
                             this is the contract and the "reference-cost" CPU baseline.
  * ``CachedDecoder``     -- the same arithmetic for the last position only with K/V kept
                             between steps; used to generate long golden sequences fast
                             and to show the cache does not change tokens.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F


@dataclass(frozen=True)
class WhisperDims:
    """WhisperConfig / AudioEncoderConfig / TextDecoderConfig (mod.rs:16-39,73-80,164-171)."""
    n_mels: int = 80
    n_audio_ctx: int = 1500
    n_audio_state: int = 384
    n_audio_head: int = 6
    n_audio_layer: int = 4
    n_vocab: int = 51864
    n_text_ctx: int = 448
    n_text_state: int = 384
    n_text_head: int = 6
    n_text_layer: int = 4


# OpenAI model sizes (not in the reference; they come from the checkpoint, dump.py:215-216)
MODEL_DIMS = {
    "tiny.en": WhisperDims(80, 1500, 384, 6, 4, 51864, 448, 384, 6, 4),
    "base.en": WhisperDims(80, 1500, 512, 8, 6, 51864, 448, 512, 8, 6),
    "small.en": WhisperDims(80, 1500, 768, 12, 12, 51864, 448, 768, 12, 12),
    "medium": WhisperDims(80, 1500, 1024, 16, 24, 51865, 448, 1024, 16, 24),
    "large-v2": WhisperDims(80, 1500, 1280, 20, 32, 51865, 448, 1280, 20, 32),
    # small shapes for seconds-scale tests (same structure, head dim 64 / 32)
    "test-a": WhisperDims(80, 1500, 128, 2, 2, 1024, 448, 128, 2, 2),
    "test-b": WhisperDims(80, 1500, 192, 3, 3, 2051, 448, 192, 3, 3),
}


@dataclass
class OracleOptions:
    # burn 0.9 LayerNorm: (x-mean)/(sqrt(var)+eps)  ["outside"]; later burn: /sqrt(var+eps) ["inside"]
    ln_eps_mode: str = "outside"
    # K/V storage rounding at the cache boundary: "f32" (reference) or "f16" (fp16 KV-cache mode)
    kv_dtype: str = "f32"


DEFAULT_OPTS = OracleOptions()


def _f32(x: float) -> float:
    return float(np.float32(x))


def as_dtype(w: dict, dtype: torch.dtype = torch.float64) -> dict:
    """The weights in another float type (float64: the oracle then runs every op in float64).  The scalar constants stay the
    fp32 values the GPU multiplies by (_f32)."""
    return {k: v.to(dtype) for k, v in w.items()}


# ---------------------------------------------------------------- third-party (burn) ops
def linear(x: torch.Tensor, w: dict, path: str) -> torch.Tensor:
    """burn nn::Linear: x @ W[d_in,d_out] (+ b)."""
    y = torch.matmul(x, w[path + "/weight"])
    b = w.get(path + "/bias")
    return y if b is None else y + b


def layer_norm(x: torch.Tensor, w: dict, path: str, opts: OracleOptions = DEFAULT_OPTS) -> torch.Tensor:
    """burn nn::LayerNorm (biased variance over the last dim; eps from the record, load.rs:71)."""
    eps = _f32(float(w[path + "/eps"]))
    mean = x.mean(dim=-1, keepdim=True)
    var = torch.pow(x - mean, 2.0).mean(dim=-1, keepdim=True)
    if opts.ln_eps_mode == "outside":
        xn = (x - mean) / (torch.sqrt(var) + eps)
    else:
        xn = (x - mean) / torch.sqrt(var + eps)
    return xn * w[path + "/weight"] + w[path + "/bias"]


def gelu(x: torch.Tensor) -> torch.Tensor:
    """burn activation::gelu, erf form: x * (erf(x / sqrt2) + 1) / 2."""
    return (x * (torch.erf(x / _f32(math.sqrt(2.0))) + 1.0)) / 2.0


def softmax_last(x: torch.Tensor) -> torch.Tensor:
    """burn activation::softmax: exp(x - max) / sum."""
    x = x - x.max(dim=-1, keepdim=True).values
    e = torch.exp(x)
    return e / e.sum(dim=-1, keepdim=True)


def log_softmax_last(x: torch.Tensor) -> torch.Tensor:
    """burn activation::log_softmax: (x - max) - log(sum(exp(x - max)))."""
    x = x - x.max(dim=-1, keepdim=True).values
    return x - torch.log(torch.exp(x).sum(dim=-1, keepdim=True))


# ---------------------------------------------------------------- mod.rs
def attn_decoder_mask(n: int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """mod.rs:535-544: zeros with strict upper triangle = -inf."""
    return torch.triu(torch.full((n, n), float("-inf"), dtype=dtype), diagonal=1)


def qkv_attention(q, k, v, mask, n_head: int, kv_f16: bool = False) -> torch.Tensor:
    """mod.rs:493-533.  kv_f16 (not in the reference): the scaled keys and the values are rounded to fp16
    at the point where the CUDA path stores them in its fp16 K/V cache."""
    n_batch, n_qctx, n_state = q.shape
    n_ctx = k.shape[1]
    scale = _f32((n_state / n_head) ** -0.25)
    n_hstate = n_state // n_head
    q = q.reshape(n_batch, n_qctx, n_head, n_hstate).transpose(1, 2) * scale
    k = k.reshape(n_batch, n_ctx, n_head, n_hstate).transpose(1, 2).transpose(2, 3) * scale
    v = v.reshape(n_batch, n_ctx, n_head, n_hstate).transpose(1, 2)
    if kv_f16:
        k = k.to(torch.float16).to(k.dtype)
        v = v.to(torch.float16).to(v.dtype)
    qk = torch.matmul(q, k)
    if mask is not None:
        qk = qk + mask[0:n_qctx, 0:n_ctx]
    w = softmax_last(qk)
    return torch.matmul(w, v).transpose(1, 2).flatten(2, 3)


def _round_kv(t: torch.Tensor, opts: OracleOptions) -> torch.Tensor:
    return t   # rounding happens inside qkv_attention (after the key scaling), see kv_f16


def _f16(opts: OracleOptions) -> bool:
    return opts.kv_dtype == "f16"


def self_attention(x, w, path, mask, n_head, opts=DEFAULT_OPTS):
    """MultiHeadSelfAttention::forward mod.rs:428-436 (key has no bias, mod.rs:402-404)."""
    q = linear(x, w, path + "/query")
    k = _round_kv(linear(x, w, path + "/key"), opts)
    v = _round_kv(linear(x, w, path + "/value"), opts)
    return linear(qkv_attention(q, k, v, mask, n_head, _f16(opts)), w, path + "/out")


def cross_attention(x, xa, w, path, n_head, opts=DEFAULT_OPTS):
    """MultiHeadCrossAttention::forward mod.rs:482-490 (k, v re-projected from xa every call)."""
    q = linear(x, w, path + "/query")
    k = _round_kv(linear(xa, w, path + "/key"), opts)
    v = _round_kv(linear(xa, w, path + "/value"), opts)
    return linear(qkv_attention(q, k, v, None, n_head, _f16(opts)), w, path + "/out")


def mlp(x, w, path):
    """MLP::forward mod.rs:376-382."""
    return linear(gelu(linear(x, w, path + "/mlp1")), w, path + "/mlp2")


def forward_encoder(w: dict, dims: WhisperDims, mel: torch.Tensor, opts=DEFAULT_OPTS,
                    kv_opts_apply: bool = False) -> torch.Tensor:
    """AudioEncoder::forward mod.rs:228-260.  mel [B,80,Tm] -> [B,T,d], T = (Tm-1)//2 + 1."""
    _, n_mels, n_ctx = mel.shape
    assert n_mels == dims.n_mels, f"Audio mel spectrum size must be {dims.n_mels}."
    assert n_ctx <= dims.n_audio_ctx, f"Audio length {n_ctx} cannot exceed {dims.n_audio_ctx}."
    enc_opts = opts if kv_opts_apply else OracleOptions(ln_eps_mode=opts.ln_eps_mode, kv_dtype="f32")
    x = gelu(F.conv1d(mel, w["encoder/conv1/weight"], w["encoder/conv1/bias"], padding=1))
    x = gelu(F.conv1d(x, w["encoder/conv2/weight"], w["encoder/conv2/bias"], stride=2, padding=1))
    x = x.transpose(1, 2)
    k = x.shape[1]
    x = x + w["encoder/positional_embedding"][0:k].unsqueeze(0)
    for i in range(dims.n_audio_layer):
        p = f"encoder/block_{i}"
        x = x + self_attention(layer_norm(x, w, p + "/attn_ln", opts), w, p + "/attn", None,
                               dims.n_audio_head, enc_opts)           # mod.rs:300
        x = x + mlp(layer_norm(x, w, p + "/mlp_ln", opts), w, p + "/mlp")  # mod.rs:301
    return layer_norm(x, w, "encoder/ln_post", opts)


def forward_decoder(w: dict, dims: WhisperDims, tokens: torch.Tensor, xa: torch.Tensor,
                    opts=DEFAULT_OPTS) -> torch.Tensor:
    """TextDecoder::forward mod.rs:131-157.  tokens [nb,t] int64, xa [nb,T,d] -> logits [nb,t,V]."""
    n_batch, seq_len = tokens.shape
    assert seq_len <= dims.n_text_ctx, f"Token sequence length {seq_len} must not exceed {dims.n_text_ctx}."
    x = F.embedding(tokens, w["decoder/token_embedding/weight"]) \
        + w["decoder/positional_embedding"][0:seq_len].unsqueeze(0)
    mask = attn_decoder_mask(dims.n_text_ctx, x.dtype)
    for i in range(dims.n_text_layer):
        p = f"decoder/block_{i}"
        x = x + self_attention(layer_norm(x, w, p + "/attn_ln", opts), w, p + "/attn", mask,
                               dims.n_text_head, opts)                                   # mod.rs:346
        x = x + cross_attention(layer_norm(x, w, p + "/cross_attn_ln", opts), xa, w, p + "/cross_attn",
                                dims.n_text_head, opts)                                  # mod.rs:347
        x = x + mlp(layer_norm(x, w, p + "/mlp_ln", opts), w, p + "/mlp")             # mod.rs:348
    x = layer_norm(x, w, "decoder/ln", opts)
    return torch.matmul(x, w["decoder/token_embedding/weight"].transpose(0, 1).unsqueeze(0))


class CachedDecoder:
    """Last-position-only decoder with persistent K/V (same per-op arithmetic as mod.rs, F8 of
    SURVEY.md removed).  One instance per encoder output ``xa`` [1,T,d]; rows are beams."""

    def __init__(self, w: dict, dims: WhisperDims, xa: torch.Tensor, opts=DEFAULT_OPTS):
        assert xa.shape[0] == 1
        self.w, self.dims, self.opts = w, dims, opts
        self.cross = []
        for i in range(dims.n_text_layer):
            p = f"decoder/block_{i}/cross_attn"
            self.cross.append((_round_kv(linear(xa, w, p + "/key"), opts),
                               _round_kv(linear(xa, w, p + "/value"), opts)))
        self.k = [None] * dims.n_text_layer   # each [nb, t, d]
        self.v = [None] * dims.n_text_layer
        self.t = 0

    def reorder(self, parents: list[int]) -> None:
        idx = torch.tensor(parents, dtype=torch.int64)
        for i in range(self.dims.n_text_layer):
            if self.k[i] is not None:
                self.k[i] = self.k[i][idx]
                self.v[i] = self.v[i][idx]

    def step(self, tokens: torch.Tensor) -> torch.Tensor:
        """tokens [nb] int64 at position self.t -> logits [nb, V] for that position."""
        w, dims, opts = self.w, self.dims, self.opts
        nb = tokens.shape[0]
        x = F.embedding(tokens, w["decoder/token_embedding/weight"]).unsqueeze(1) \
            + w["decoder/positional_embedding"][self.t:self.t + 1].unsqueeze(0)
        for i in range(dims.n_text_layer):
            p = f"decoder/block_{i}"
            h = layer_norm(x, w, p + "/attn_ln", opts)
            q = linear(h, w, p + "/attn/query")
            kn = _round_kv(linear(h, w, p + "/attn/key"), opts)
            vn = _round_kv(linear(h, w, p + "/attn/value"), opts)
            self.k[i] = kn if self.k[i] is None else torch.cat([self.k[i], kn], dim=1)
            self.v[i] = vn if self.v[i] is None else torch.cat([self.v[i], vn], dim=1)
            x = x + linear(qkv_attention(q, self.k[i], self.v[i], None, dims.n_text_head, _f16(opts)), w, p + "/attn/out")
            h = layer_norm(x, w, p + "/cross_attn_ln", opts)
            q = linear(h, w, p + "/cross_attn/query")
            ck, cv = self.cross[i]
            x = x + linear(qkv_attention(q, ck.expand(nb, -1, -1), cv.expand(nb, -1, -1), None,
                                         dims.n_text_head, _f16(opts)), w, p + "/cross_attn/out")
            x = x + mlp(layer_norm(x, w, p + "/mlp_ln", opts), w, p + "/mlp")
        x = layer_norm(x, w, "decoder/ln", opts)
        self.t += 1
        return torch.matmul(x[:, 0, :], w["decoder/token_embedding/weight"].transpose(0, 1))
