"""Float64 restatement of the library's conversion to 16 kHz mono (whisper_b200.h wb_resample), for the resample tests.  It
sits beside the oracle package; the reference has no resampler (its README converts with sox first).

    x[i] = (x[i,0] + .. + x[i,C-1]) / C                                  f64, channel order
    g = gcd(sr, 16000), up = 16000 / g, down = sr / g                    supported when sr >= 1 and max(up, down) <= 1024
    m = max(up, down), half = 10 m
    h[j] = up * w[j] / sum(w),  w[j] = sinc((j - half) / m) * kaiser(2 half + 1, 5.0)[j]     (h = [1], half = 0 for up = down = 1)
    y[k] = sum_i h[half + k down - i up] x[i]   over 0 <= half + k down - i up <= 2 half, 0 <= i < n;   k < ceil(n up / down)

This is scipy.signal.resample_poly(x, up, down) with its defaults.  The sum runs per phase: outputs k with the same k mod up
share the phase p = (half + k down) mod up and read taps p, p + up, p + 2 up, .. at input frames base_k, base_k - 1, ..
(base_k = (half + k down - p) / up), so each phase is a few vector multiply-adds over all its outputs.
"""
from __future__ import annotations

import math

import numpy as np

MAX_FACTOR = 1024


def ratio(sample_rate: int):
    """(up, down) of sample_rate -> 16 kHz, or None for an unsupported rate."""
    if sample_rate < 1:
        return None
    g = math.gcd(sample_rate, 16000)
    up, down = 16000 // g, sample_rate // g
    return (up, down) if max(up, down) <= MAX_FACTOR else None


def resampled_length(n_frames: int, sample_rate: int) -> int:
    r = ratio(sample_rate)
    if r is None or n_frames < 0:
        return -1
    up, down = r
    return -(-n_frames * up // down)


def taps(up: int, down: int):
    """(h, half): resample_poly's filter scaled by up."""
    if up == 1 and down == 1:
        return np.ones(1), 0
    m = max(up, down)
    half = 10 * m
    j = np.arange(2 * half + 1, dtype=np.float64)
    w = np.sinc((j - half) / m) * np.i0(5.0 * np.sqrt(np.maximum(0.0, 1.0 - ((j - half) / half) ** 2))) / np.i0(5.0)
    return up * w / w.sum(), half


def downmix(waveform: np.ndarray) -> np.ndarray:
    """f64 mean of the channels of [n_frames] or [n_frames, channels], summed in channel order."""
    x = np.asarray(waveform)
    if x.ndim == 1:
        return x.astype(np.float64)
    s = x[:, 0].astype(np.float64)
    for c in range(1, x.shape[1]):
        s = s + x[:, c].astype(np.float64)
    return s / x.shape[1]


def resample(waveform: np.ndarray, sample_rate: int) -> np.ndarray:
    """y in float64: the exact value the library rounds once to float32."""
    up, down = ratio(sample_rate)
    x = downmix(waveform)
    n = len(x)
    n_out = resampled_length(n, sample_rate)
    h, half = taps(up, down)
    y = np.zeros(n_out)
    pad = half // up + 2                                      # every frame an output reads lies in [-pad, n + pad)
    xp = np.concatenate([np.zeros(pad), x, np.zeros(pad)])   # zeros outside the input
    for r in range(min(up, n_out)):
        k = np.arange(r, n_out, up, dtype=np.int64)
        p = (half + r * down) % up                            # the same for every k = r mod up
        base = (half + k * down - p) // up
        for t in range((2 * half - p) // up + 1):
            y[k] += h[p + t * up] * xp[base - t + pad]
    return y
