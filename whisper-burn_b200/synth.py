"""Seeded synthetic inputs shared by the tests, smoke() and bench.py (SURVEY.md section 8d).

Input GENERATION only (pure numpy, no arithmetic of the hot path; the oracle re-exports it as
oracle.synth).  There are no Whisper weights, tokenizer.json or
16 kHz audio on disk, so everything is generated with numpy's PCG64 ``default_rng`` (stable
across numpy versions and machines):

  * waveforms: noise + 3 sinusoids (220 Hz, 1 kHz, 3.5 kHz) + seeded tone bursts, clipped.
  * weights:   real Whisper shapes, unit-gain Linear/Conv init so that the residual branches
               (and therefore the audio, through cross-attention) dominate the token embedding;
               with the reference's own N(0,1) embedding init (mod.rs:84-93) the tied-embedding
               logits are trivially self-predicting and parity checks would be vacuous.
               Every value is rounded to an fp16-representable f32, as OpenAI's released
               checkpoints are (they are stored in fp16; python/dump.py writes them out as f32).
  * tokenizer stand-in: 6 special ids >= eot (startofprev = eot + 5) and ``is_special(id) <=> id >= eot``.
"""
from __future__ import annotations

import math

from dataclasses import dataclass
from typing import List

import numpy as np

from .model import WhisperConfig as WhisperDims

# OpenAI model sizes (not in the reference; they come from the checkpoint, python/dump.py:215-216)
MODEL_DIMS = {
    "tiny.en": WhisperDims(80, 1500, 384, 6, 4, 51864, 448, 384, 6, 4),
    "base.en": WhisperDims(80, 1500, 512, 8, 6, 51864, 448, 512, 8, 6),
    "small.en": WhisperDims(80, 1500, 768, 12, 12, 51864, 448, 768, 12, 12),
    "medium": WhisperDims(80, 1500, 1024, 16, 24, 51865, 448, 1024, 16, 24),
    "large-v2": WhisperDims(80, 1500, 1280, 20, 32, 51865, 448, 1280, 20, 32),
    # small shapes for seconds-scale tests (same structure, head dim 64)
    "test-a": WhisperDims(80, 1500, 128, 2, 2, 1024, 448, 128, 2, 2),
    "test-b": WhisperDims(80, 1500, 192, 3, 3, 2051, 448, 192, 3, 3),
    "test-c": WhisperDims(80, 1500, 256, 4, 2, 2051, 448, 256, 4, 3),
    "test-e": WhisperDims(80, 1500, 768, 12, 1, 2051, 448, 768, 12, 2),   # d = 768 (small.en width): MLP2 runs as 3 K-slabs of 1024 in decoder5.cu
    "test-d": WhisperDims(80, 1500, 512, 8, 1, 2051, 448, 512, 8, 2),    # 8 heads: 17+ rows give >= 132 (row, head) units -> unsplit cross attention in decoder5.cu    # d % 256 == 0: the batched tensor-core decoder (decoder5.cu)
}


@dataclass(frozen=True)
class SpecialTokens:
    """Stand-in for what mels_to_text asks the tokenizer (src/transcribe.rs:179-185, 243-251)."""
    sot: int
    lang: int
    transcribe: int
    notimestamps: int
    eot: int
    first_special: int   # is_special(id) <=> id >= first_special (stand-in for src/token.rs:41-47)
    n_vocab: int
    startofprev: int = -1   # <|startofprev|> (token.rs:280-294), the first id of a previous-text prompt; -1: unknown

    def is_special(self, tok: int) -> bool:
        return tok >= self.first_special

    def is_special_bitmap(self) -> np.ndarray:
        return (np.arange(self.n_vocab) >= self.first_special).astype(np.uint8)

    def maskout(self) -> np.ndarray:
        """special_tokens_maskout (transcribe.rs:243-251): -inf on special ids, 0 elsewhere."""
        m = np.zeros(self.n_vocab, dtype=np.float32)
        m[self.first_special:] = -np.inf
        return m

    def prompt(self) -> List[int]:
        """transcribe.rs:203 (the prev-token prompt is shadowed by Vec::new(), :195-201)."""
        return [self.sot, self.lang, self.transcribe, self.notimestamps]


def waveform(n_samples: int, seed: int = 1234, kind: str = "mix") -> np.ndarray:
    rng = np.random.default_rng(seed)
    t = np.arange(n_samples, dtype=np.float64) / 16000.0
    if kind == "mix":
        # stationary floor (noise + 3 tones) + seeded 40-250 ms tone bursts ("syllables") so the
        # encoder output varies along time and cross-attention has something to select
        x = 0.02 * rng.standard_normal(n_samples)
        for f in (220.0, 1000.0, 3500.0):
            x += 0.05 * np.sin(2.0 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
        pos = 0
        while pos < n_samples:
            seg = min(int(rng.uniform(0.04, 0.25) * 16000), n_samples - pos)
            if rng.uniform() < 0.8:
                f0 = math.exp(rng.uniform(math.log(80.0), math.log(7000.0)))
                f1 = f0 * math.exp(rng.uniform(-0.3, 0.3))
                tt = np.arange(seg, dtype=np.float64) / 16000.0
                ph = 2.0 * np.pi * (f0 * tt + 0.5 * (f1 - f0) / max(seg / 16000.0, 1e-3) * tt * tt)
                env = np.sin(np.pi * np.arange(seg) / seg) ** 2
                x[pos:pos + seg] += rng.uniform(0.1, 0.5) * env * np.sin(ph)
            pos += seg
    elif kind == "noise":
        x = 0.3 * rng.standard_normal(n_samples)
    elif kind == "chirp":
        f0, f1 = 50.0, 7500.0
        dur = max(n_samples / 16000.0, 1e-3)
        x = 0.5 * np.sin(2.0 * np.pi * (f0 * t + 0.5 * (f1 - f0) / dur * t * t))
    elif kind == "click":
        x = np.zeros(n_samples)
        x[n_samples // 3] = 0.9
        x[(2 * n_samples) // 3] = -0.7
    elif kind == "silence":
        x = np.zeros(n_samples)
    else:
        raise ValueError(kind)
    return np.clip(x, -1.0, 1.0).astype(np.float32)


def chunk_waveform(chunk_id: int, n_samples: int = 480000) -> np.ndarray:
    """One synthetic '30 s chunk' (SURVEY.md 8d): seed 1234 + chunk_id."""
    return waveform(n_samples, seed=1234 + chunk_id, kind="mix")


def special_tokens(dims: WhisperDims) -> SpecialTokens:
    v = dims.n_vocab
    eot = 50256 if v == 51864 else (50257 if v == 51865 else v - 16)
    return SpecialTokens(sot=eot + 1, lang=eot + 2, transcribe=eot + 3, notimestamps=eot + 4,
                         eot=eot, first_special=eot, n_vocab=v, startofprev=eot + 5)


def _fp16_exact(a: np.ndarray) -> np.ndarray:
    return a.astype(np.float16).astype(np.float32)


def make_weights_np(dims: WhisperDims, seed: int = 0) -> dict:
    """Flat dict of float32 numpy arrays keyed by the reference's npy-tree paths."""
    rng = np.random.default_rng(seed)
    d, L_e, L_d = dims.n_audio_state, dims.n_audio_layer, dims.n_text_layer
    w: dict = {}

    def normal(shape, std):
        return _fp16_exact((rng.standard_normal(shape, dtype=np.float32) * np.float32(std)))

    def lin(path, d_in, d_out, bias=True, gain=1.0):
        w[path + "/weight"] = normal((d_in, d_out), gain / math.sqrt(d_in))   # burn layout [d_in, d_out]
        if bias:
            w[path + "/bias"] = normal((d_out,), 0.01)

    def ln(path, n):
        w[path + "/weight"] = _fp16_exact(1.0 + 0.02 * rng.standard_normal(n, dtype=np.float32))
        w[path + "/bias"] = normal((n,), 0.02)
        w[path + "/eps"] = np.float32(1e-5)

    def attn(path, n, gain_out):
        lin(path + "/query", n, n, gain=2.0)           # sharper softmax: tokens depend on the audio
        lin(path + "/key", n, n, bias=False, gain=2.0)
        lin(path + "/value", n, n)
        lin(path + "/out", n, n, gain=gain_out)

    def block(path, n, cross, gain_out):
        attn(path + "/attn", n, gain_out)
        ln(path + "/attn_ln", n)
        if cross:
            attn(path + "/cross_attn", n, gain_out)
            ln(path + "/cross_attn_ln", n)
        lin(path + "/mlp/mlp1", n, 4 * n)
        lin(path + "/mlp/mlp2", 4 * n, n, gain=gain_out)
        ln(path + "/mlp_ln", n)

    w["encoder/conv1/weight"] = normal((d, dims.n_mels, 3), 1.0 / math.sqrt(3 * dims.n_mels))
    w["encoder/conv1/bias"] = normal((d,), 0.01)
    w["encoder/conv2/weight"] = normal((d, d, 3), 1.0 / math.sqrt(3 * d))
    w["encoder/conv2/bias"] = normal((d,), 0.01)
    w["encoder/positional_embedding"] = normal((dims.n_audio_ctx, d), 0.1)
    for i in range(L_e):
        block(f"encoder/block_{i}", d, False, 1.0 / math.sqrt(2 * L_e))
    ln("encoder/ln_post", d)

    dt = dims.n_text_state
    w["decoder/token_embedding/weight"] = normal((dims.n_vocab, dt), 0.02)
    w["decoder/positional_embedding"] = normal((dims.n_text_ctx, dt), 0.01)
    for i in range(L_d):
        block(f"decoder/block_{i}", dt, True, 1.0 / math.sqrt(2 * L_d))
    ln("decoder/ln", dt)
    return w


def make_weights(model_name_or_dims, seed: int = 0):
    dims = MODEL_DIMS[model_name_or_dims] if isinstance(model_name_or_dims, str) else model_name_or_dims
    return dims, make_weights_np(dims, seed)
