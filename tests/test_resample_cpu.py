"""CPU tests of the conversion to 16 kHz mono (wb_resample, wb_resampled_length, wb_waveforms_to_tokens_resampled):

  1. the float64 oracle (tests/oracle_resample.py) is scipy.signal.resample_poly with its defaults, on unit-scale noise at
     every common rate and at lengths around the filter's edges, and on the reference's own 22 050 Hz audio.wav;
  2. audio.resampled_length is the length resample_poly returns, and -1 for an unsupported rate;
  3. argument errors are WB_ERR_INVALID_ARG / WB_ERR_UNSUPPORTED before the device is touched, so they come back as such
     on a machine without a GPU (where a computing call fails with WB_ERR_CUDA)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import scipy.signal

import oracle_resample as o_rs
import wb200  # noqa: F401
from whisper_burn_b200 import audio, ffi, wav

RATES = (8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000, 96000, 192000)
FIXTURE = Path(__file__).resolve().parent / "golden" / "reference_audio_22050.wav"


def lengths(sample_rate):
    """1, 2, the filter's half-length in input frames +- 1, 399, 4001 and 7.64 s (the fixture's duration)"""
    up, down = o_rs.ratio(sample_rate)
    half = o_rs.taps(up, down)[1]
    return sorted({1, 2, max(half // up - 1, 1), half // up + 1, 399, 4001, int(7.64 * sample_rate)})


@pytest.mark.parametrize("sample_rate", RATES)
def test_oracle_is_resample_poly(sample_rate):
    rng = np.random.default_rng(sample_rate)
    up, down = o_rs.ratio(sample_rate)
    for n in lengths(sample_rate):
        x = rng.standard_normal(n)
        want = scipy.signal.resample_poly(x, up, down)
        got = o_rs.resample(x, sample_rate)
        assert len(got) == len(want), (sample_rate, n)
        assert np.abs(got - want).max() <= 1e-12, (sample_rate, n)
        assert audio.resampled_length(n, sample_rate) == len(want) == o_rs.resampled_length(n, sample_rate)


def test_oracle_on_the_reference_audio_file():
    x, sr = wav.load_audio_waveform(str(FIXTURE), strict=False)
    assert sr == 22050 and x.ndim == 1 and len(x) == 168511   # 7.64 s, mono int16
    want = scipy.signal.resample_poly(x.astype(np.float64), 320, 441)
    got = o_rs.resample(x, sr)
    assert len(got) == len(want) == audio.resampled_length(len(x), sr) == 122276
    assert np.abs(got - want).max() <= 1e-12


def test_ratios_and_unsupported_rates():
    assert o_rs.ratio(44100) == (160, 441) and o_rs.ratio(11025) == (640, 441) and o_rs.ratio(48000) == (1, 3)
    assert o_rs.ratio(16000) == (1, 1) and o_rs.ratio(8000) == (2, 1) and o_rs.ratio(192000) == (1, 12)
    for sr in (16001, 0, -1):
        assert audio.resampled_length(1000, sr) == -1, sr
    assert audio.resampled_length(-1, 16000) == -1
    assert audio.resampled_length(0, 44100) == 0
    assert audio.resampled_length(12345, 16000) == 12345


def test_argument_errors_come_before_the_device():
    """Each case fails with its own code, not WB_ERR_CUDA, with or without a GPU."""
    lib = ffi.lib()
    x = np.zeros(8000, dtype=np.float32)
    out = np.zeros(16000, dtype=np.float32)
    n = C.c_int64(0)

    def resample(inp, frames, channels, rate, dst, cap):
        return lib.wb_resample(0, inp, frames, channels, rate, dst, cap, C.byref(n))

    assert resample(ffi.fptr(x), 8000, 0, 8000, ffi.fptr(out), len(out)) == ffi.WB_ERR_INVALID_ARG          # channels 0
    assert resample(ffi.fptr(x), 0, 1, 8000, ffi.fptr(out), len(out)) == ffi.WB_ERR_INVALID_ARG             # n_frames 0
    assert resample(ffi.fptr(x), 8000, 1, 16001, ffi.fptr(out), len(out)) == ffi.WB_ERR_UNSUPPORTED         # 16001 Hz
    assert resample(None, 8000, 1, 8000, ffi.fptr(out), len(out)) == ffi.WB_ERR_INVALID_ARG                 # null input
    assert resample(ffi.fptr(x), 8000, 1, 8000, None, len(out)) == ffi.WB_ERR_INVALID_ARG                  # null output
    assert resample(ffi.fptr(x), 8000, 1, 8000, ffi.fptr(out), 15999) == ffi.WB_ERR_INVALID_ARG             # capacity
    with pytest.raises(ffi.WbError) as e:
        audio.resample(np.zeros((100, 0), np.float32), 44100)
    assert e.value.code == ffi.WB_ERR_INVALID_ARG
    with pytest.raises(ffi.WbError) as e:
        audio.resample(np.zeros(100, np.float32), 16001)
    assert e.value.code == ffi.WB_ERR_UNSUPPORTED
    # the decode entry point without a session
    ptrs = (ffi._F * 1)(ffi.fptr(x))
    one = np.ones(1, dtype=np.int64)
    toks = np.zeros(64, dtype=np.int64)
    ids = ffi.SpecialIds(0, 1, 2, 3, 4)
    st = lib.wb_waveforms_to_tokens_resampled(None, ptrs, ffi.i64ptr(one * 8000), ffi.i64ptr(one), ffi.i64ptr(one * 8000), 1, 1, 4,
                                              C.byref(ids), None, ffi.i64ptr(toks), 64, ffi.i64ptr(one))
    assert st == ffi.WB_ERR_INVALID_ARG
