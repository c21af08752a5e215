"""Mirror of the reference's ``audio`` module (src/audio.rs) over the C ABI."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import ffi


def max_waveform_samples(n_frame_max: int) -> int:
    """audio::max_waveform_samples (audio.rs:12-17)."""
    return int(ffi.lib().wb_max_waveform_samples(n_frame_max))


def prep_audio(waveform: np.ndarray, sample_rate: float = 16000.0, device: int = 0) -> np.ndarray:
    """audio::prep_audio (audio.rs:34-56): [n_batch, n_samples] f32 -> [n_batch, 80, n_samples/160].
    Raises WbError(WB_ERR_INVALID_ARG) where the reference panics (n_samples < 400, audio.rs:292)."""
    if sample_rate != 16000.0:
        raise ffi.WbError(ffi.WB_ERR_UNSUPPORTED, "only 16 kHz input is supported (the reference asserts it, transcribe/main.rs:41)")
    w = np.ascontiguousarray(waveform, dtype=np.float32)
    if w.ndim != 2:
        raise ffi.WbError(ffi.WB_ERR_INVALID_ARG, "prep_audio expects [n_batch, n_samples]")
    n_batch, n = w.shape
    out = np.empty((n_batch, 80, max(n // 160, 0)), dtype=np.float32)
    nf = C.c_int64(0)
    ffi.check(ffi.lib().wb_prep_audio(device, ffi.fptr(w), n_batch, n, ffi.fptr(out), C.byref(nf)))
    return out


def resampled_length(n_frames: int, sample_rate: int) -> int:
    """Samples wb_resample makes of n_frames at sample_rate: ceil(n_frames * up / down), -1 for an unsupported rate."""
    return int(ffi.lib().wb_resampled_length(n_frames, sample_rate))


def _frames(waveform: np.ndarray) -> np.ndarray:
    """A waveform as C-contiguous f32 [n_frames, channels]: 1-D is mono, 2-D [n_frames, channels] interleaved (what
    wav.load_audio_waveform(strict=False) returns)."""
    w = np.ascontiguousarray(waveform, dtype=np.float32)
    if w.ndim == 1:
        w = w[:, None]
    if w.ndim != 2:
        raise ffi.WbError(ffi.WB_ERR_INVALID_ARG, "a waveform is 1-D (mono) or 2-D [n_frames, channels]")
    return w


def resample(waveform: np.ndarray, sample_rate: int, device: int = 0) -> np.ndarray:
    """16 kHz mono f32 of a waveform at sample_rate (wb_resample): the channels' mean, then scipy.signal.resample_poly(x, up,
    down) with up / down = 16000 / sample_rate in lowest terms, computed in f64 on the GPU.  WbError(WB_ERR_UNSUPPORTED) when
    up or down exceeds 1024."""
    w = _frames(waveform)
    n = resampled_length(w.shape[0], sample_rate)
    out = np.empty(max(n, 0), dtype=np.float32)
    n_out = C.c_int64(0)
    ffi.check(ffi.lib().wb_resample(device, ffi.fptr(w), w.shape[0], w.shape[1], sample_rate, ffi.fptr(out), len(out), C.byref(n_out)))
    return out
