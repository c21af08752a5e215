"""Native windowing, host side: the frame limit, window length and window bounds of both window modes, in the library
(wb_window_samples + wb_window_bounds) and in the oracle (its n_audio_ctx doubled, see tests/golden/make_golden_native.py),
against each other and against hand-worked numbers.  No GPU needed."""
import dataclasses

import pytest
import torch

import wb200  # noqa: F401
from oracle import audio as o_audio, model as o_model, transcribe as o_tr
from whisper_burn_b200 import audio, ffi, transcribe

WHISPER = o_model.MODEL_DIMS["tiny.en"]   # n_audio_ctx = 1500, as every Whisper checkpoint


@pytest.fixture(scope="module", autouse=True)
def built():
    if not ffi.library_path().exists():
        import __graft_entry__ as ge
        ge.build()


def oracle_dims(mode):
    return dataclasses.replace(WHISPER, n_audio_ctx=2 * WHISPER.n_audio_ctx) if mode == "native" else WHISPER


def oracle_window(n_samples, mode):
    """(Tm, T) of one window of n_samples through the oracle: prep_audio's frame count, pad_mel's clip + 10 zero frames,
    conv2's stride."""
    F = n_samples // 160
    Tm = o_tr.pad_mel(torch.zeros(1, 80, F), oracle_dims(mode).n_audio_ctx).shape[2]
    return Tm, (Tm - 1) // 2 + 1


# n_samples -> {mode: (Tm, T of a window that long, [start, end) of every window of waveform_to_tokens)}.  The window
# stepping is the reference's (transcribe.rs:114-138): (n - 1) // shift + 1 windows, so a waveform exactly one window long
# still gets a second, overlap-only window.
HAND = {
    400: {"reference": (12, 6, [(0, 400)]), "native": (12, 6, [(0, 400)])},
    238559: {"reference": (1500, 750, [(0, 238559), (190559, 238559)]), "native": (1500, 750, [(0, 238559)])},
    478559: {"reference": (1500, 750, [(0, 238559), (190559, 429118), (381118, 478559)]),
             "native": (3000, 1500, [(0, 478559), (430559, 478559)])},
    478560: {"reference": (1500, 750, [(0, 238559), (190559, 429118), (381118, 478560)]),
             "native": (3000, 1500, [(0, 478559), (430559, 478560)])},
    480000: {"reference": (1500, 750, [(0, 238559), (190559, 429118), (381118, 480000)]),
             "native": (3000, 1500, [(0, 478559), (430559, 480000)])},
    1120000: {"reference": (1500, 750, [(i * 190559, min(i * 190559 + 238559, 1120000)) for i in range(6)]),
              "native": (3000, 1500, [(0, 478559), (430559, 909118), (861118, 1120000)])},
}


def test_window_samples_hand_worked():
    assert transcribe.window_samples(1500, "reference") == 238559
    assert transcribe.window_samples(1500, "native") == 478559
    assert o_tr.audio.max_waveform_samples(2990) == 478559
    assert o_tr.window_bounds(480000, 16000, 478559)[1] == (430559, 480000)   # shift 478 559 - 48 000 = 430 559


@pytest.mark.parametrize("mode", ["reference", "native"])
@pytest.mark.parametrize("n_samples", sorted(HAND))
def test_window_table_library_oracle_and_hand(n_samples, mode):
    Tm, T, bounds = HAND[n_samples][mode]
    assert oracle_window(n_samples, mode) == (Tm, T)
    window_len = transcribe.window_samples(WHISPER.n_audio_ctx, mode)
    assert window_len == o_audio.max_waveform_samples(oracle_dims(mode).n_audio_ctx - o_tr.PADDING)
    got = transcribe.window_bounds(n_samples, 16000, window_len)
    assert got == o_tr.window_bounds(n_samples, 16000, window_len) == bounds
    # every window after the first: the worked second window of 480 000 samples is F = 309, Tm = 319, T = 160
    if (n_samples, mode) == (480000, "native"):
        s, e = got[1]
        assert oracle_window(e - s, mode) == (319, 160)


def test_reference_mode_is_the_reference_window():
    for n_audio_ctx in (11, 64, 1500, 3000):
        assert transcribe.window_samples(n_audio_ctx, "reference") == audio.max_waveform_samples(n_audio_ctx - 10)
        assert transcribe.window_samples(n_audio_ctx, "native") == audio.max_waveform_samples(2 * n_audio_ctx - 10)


def test_window_samples_rejects_bad_arguments():
    lib = ffi.lib()
    assert lib.wb_window_samples(1500, 2) == -1
    assert lib.wb_window_samples(1500, -1) == -1
    assert lib.wb_window_samples(10, ffi.WB_WINDOWS_REFERENCE) == -1
    with pytest.raises(ValueError):
        transcribe.window_samples(10, "native")
    with pytest.raises(KeyError):
        transcribe.window_samples(1500, "30s")
