"""GPU tests (-m gpu) of the conversion to 16 kHz mono and of wb_waveforms_to_tokens_resampled:

  1. the kernel (audio.resample) against the float64 oracle (tests/oracle_resample.py) at every common rate, with 1, 2 and 6
     channels, at lengths around the filter's edges, on one 10-minute 48 kHz stereo input and on the reference's audio.wav:
     every sample within one float32 ulp of the exact value (+ 1e-12);
  2. 16 kHz mono passes through bit-unchanged, 16 kHz stereo is fl32((a + b) / 2);
  3. waveforms_to_tokens_resampled on mixed rates and channel counts gives the ids, log-prob bits and n-best lists of
     waveforms_to_tokens on the converted audio, under the host beam search, the device beam search, beam_size 1, the greedy
     loop and the previous-text prompt, with several batches per call;
  4. 16 kHz mono through the new entry point is the old path;
  5. rejected calls (unsupported rate, no channels, a last window under 400 samples) leave the session's results as they were."""
from pathlib import Path

import numpy as np
import pytest

import harness as h
import oracle_resample as o_rs
import wb200  # noqa: F401
from oracle import synth
from whisper_burn_b200 import audio, ffi, transcribe, wav

pytestmark = pytest.mark.gpu
RATES = (8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000, 96000, 192000)
FIXTURE = Path(__file__).resolve().parent / "golden" / "reference_audio_22050.wav"
DEPTH = 12


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def check_samples(got, want64, what):
    assert got.dtype == np.float32 and len(got) == len(want64), what
    ulp = np.spacing(np.abs(want64).astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want64)
    bad = np.flatnonzero(err > ulp + 1e-12)
    assert len(bad) == 0, f"{what}: {len(bad)} samples off, first at {bad[:5]}: {got[bad[:5]]} vs {want64[bad[:5]]}"


def lengths(sample_rate):
    up, down = o_rs.ratio(sample_rate)
    half = o_rs.taps(up, down)[1]
    return sorted({1, 2, max(half // up - 1, 1), half // up + 1, 399, 4001, int(7.64 * sample_rate)})


@pytest.mark.parametrize("sample_rate", RATES)
def test_kernel_matches_the_oracle(sample_rate):
    rng = np.random.default_rng(sample_rate)
    for channels in (1, 2, 6):
        for n in lengths(sample_rate):
            x = rng.standard_normal((n, channels)).astype(np.float32)
            if channels == 1 and n % 2:
                x = x[:, 0]   # 1-D mono as well as [n, 1]
            check_samples(audio.resample(x, sample_rate), o_rs.resample(x, sample_rate), f"{sample_rate} Hz, C={channels}, n={n}")


def test_ten_minutes_of_48k_stereo_and_the_reference_file():
    rng = np.random.default_rng(48)
    x = (0.3 * rng.standard_normal((48000 * 600, 2))).astype(np.float32)
    check_samples(audio.resample(x, 48000), o_rs.resample(x, 48000), "10 min 48 kHz stereo")
    f, sr = wav.load_audio_waveform(str(FIXTURE), strict=False)
    assert sr == 22050
    check_samples(audio.resample(f, sr), o_rs.resample(f, sr), "reference audio.wav")


def test_16k_is_a_copy_and_a_channel_mean():
    rng = np.random.default_rng(16)
    x = rng.standard_normal(50001).astype(np.float32)
    assert np.array_equal(bits(audio.resample(x, 16000)), bits(x))
    ab = rng.standard_normal((50001, 2)).astype(np.float32)
    want = ((ab[:, 0].astype(np.float64) + ab[:, 1].astype(np.float64)) / 2).astype(np.float32)
    assert np.array_equal(bits(audio.resample(ab, 16000)), bits(want))


@pytest.fixture(scope="module")
def tiny():
    return h.named_model("tiny.en")


def channels(n, c, seed):
    """n frames of c channels: synthetic speech-like signals, one per channel"""
    return np.stack([synth.waveform(n, seed=seed + i) for i in range(c)], axis=1) if c > 1 else synth.waveform(n, seed=seed)


def mixed_inputs():
    """(waveforms, rates): the reference's 22.05 kHz audio.wav, 29.5 s of 44.1 kHz stereo (3 windows), 48 kHz with 6 channels
    and 8 kHz mono"""
    f, sr = wav.load_audio_waveform(str(FIXTURE), strict=False)
    return [f, channels(1300000, 2, 31), channels(150000, 6, 41), channels(60000, 1, 51)], [sr, 44100, 48000, 8000]


def results(sess, ids, n_windows, nbest):
    return (ids, [bits(sess.last_logprobs(i)) for i in range(len(ids))],
            [sess.last_nbest(i) for i in range(n_windows)] if nbest else None)


def same(a, b, what):
    assert a[0] == b[0], f"{what}: ids"
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        assert np.array_equal(x, y), f"{what}: log-probs of waveform {i}"
    if a[2] is not None:
        assert len(a[2]) == len(b[2]), what
        for w, (la, lb) in enumerate(zip(a[2], b[2])):
            assert len(la) == len(lb), f"{what}: n-best size of window {w}"
            for (ia, pa, sa, fa), (ib, pb, sb, fb) in zip(la, lb):
                assert ia == ib and np.array_equal(bits(pa), bits(pb)) and sa == sb and fa == fb, f"{what}: n-best of window {w}"


# (search rule, beam_size, max_windows, previous-text prompt): beam 5 over 5 windows is 25 rows, past the device search's 24
RUNS = [("beam", 5, 5, False), ("beam", 3, 4, False), ("beam", 1, 4, False), ("greedy_loop", 1, 4, False), ("beam", 3, 2, True)]


@pytest.mark.parametrize("search,beam_size,max_windows,prev", RUNS)
def test_pipeline_is_the_16k_path_on_the_converted_audio(tiny, search, beam_size, max_windows, prev):
    dims, sp, wh, *_ = tiny
    waves, rates = mixed_inputs()
    conv = [audio.resample(x, r) for x, r in zip(waves, rates)]
    n_windows = sum(len(transcribe.window_bounds(len(c), 16000, 238559)) for c in conv)
    assert n_windows == 6 and n_windows > max_windows
    sess = transcribe.Session(wh, max_windows=max_windows, max_beams=beam_size, max_text_len=10 + DEPTH + 1, search=search)
    if prev:
        sess.set_prev_prompt(sp.startofprev)
    bm = None if search == "greedy_loop" else sp.is_special_bitmap()
    nbest = search == "beam"
    got = results(sess, sess.waveforms_to_tokens_resampled(waves, rates, sp, bm, beam_size=beam_size, max_depth=DEPTH), n_windows, nbest)
    want = results(sess, sess.waveforms_to_tokens(conv, sp, bm, beam_size=beam_size, max_depth=DEPTH), n_windows, nbest)
    assert all(len(t) > 4 for t in want[0])
    same(got, want, f"{search} B={beam_size} max_windows={max_windows} prev={prev}")


@pytest.mark.parametrize("search,beam_size", [("beam", 3), ("greedy_loop", 1)])
def test_16k_mono_through_the_new_entry_point_is_the_old_path(tiny, search, beam_size):
    dims, sp, wh, *_ = tiny
    waves = [synth.waveform(n, seed=60 + i) for i, n in enumerate((400000, 48000, 130000))]
    sess = transcribe.Session(wh, max_windows=3, max_beams=beam_size, max_text_len=4 + DEPTH + 1, search=search)
    bm = None if search == "greedy_loop" else sp.is_special_bitmap()
    nbest = search == "beam"
    want = results(sess, sess.waveforms_to_tokens(waves, sp, bm, beam_size=beam_size, max_depth=DEPTH), 5, nbest)
    got = results(sess, sess.waveforms_to_tokens_resampled(waves, [16000] * 3, sp, bm, beam_size=beam_size, max_depth=DEPTH), 5, nbest)
    same(got, want, f"16 kHz {search}")


def test_rejected_calls_leave_the_last_results(tiny):
    dims, sp, wh, *_ = tiny
    bm = sp.is_special_bitmap()
    sess = transcribe.Session(wh, max_windows=2, max_beams=3, max_text_len=4 + DEPTH + 1)
    f, sr = wav.load_audio_waveform(str(FIXTURE), strict=False)

    def state():
        return ([bits(sess.get_encoder_output(w)) for w in range(2)], [bits(sess.last_logprobs(i)) for i in range(2)],
                sess.last_timings_ms(), sess.last_nbest(0))

    sess.waveforms_to_tokens_resampled([f, channels(120000, 2, 7)], [sr, 44100], sp, bm, beam_size=3, max_depth=DEPTH)
    want = state()
    n_short = 572577   # 48 kHz frames -> 190 859 samples: two windows, the second of 300 samples
    assert audio.resampled_length(n_short, 48000) == 238559 - 48000 + 300
    cases = {
        "unsupported rate": ([f, f], [sr, 16001], ffi.WB_ERR_UNSUPPORTED),
        "no channels": ([f, np.zeros((50000, 0), np.float32)], [sr, 44100], ffi.WB_ERR_INVALID_ARG),
        "last window under 400 samples": ([f, channels(n_short, 1, 8)], [sr, 48000], ffi.WB_ERR_INVALID_ARG),
        "beam_size above max_beams": ([f, f], [sr, sr], ffi.WB_ERR_INVALID_ARG),
    }
    for what, (waves, rates, code) in cases.items():
        b = 4 if what.startswith("beam_size") else 3
        with pytest.raises(ffi.WbError) as e:
            sess.waveforms_to_tokens_resampled(waves, rates, sp, bm, beam_size=b, max_depth=DEPTH)
        assert e.value.code == code, f"{what}: {e.value}"
        got = state()
        for w in range(2):
            assert np.array_equal(got[0][w], want[0][w]), f"{what}: encoder output of window {w}"
            assert np.array_equal(got[1][w], want[1][w]), f"{what}: log-probs of waveform {w}"
        assert got[2] == want[2], f"{what}: timings"
        assert len(got[3]) == len(want[3]) and all(a[0] == b[0] and a[2] == b[2] for a, b in zip(got[3], want[3])), f"{what}: n-best"
