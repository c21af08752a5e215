"""GPU tests (-m gpu) of the five transcribe entry points of the C ABI on the synthetic test-a model:

  1. wb_transcribe_windows, wb_transcribe_windows_dev (the windows in one CUDA tensor at offsets) and
     wb_transcribe_windows_prev with empty previous lists give identical ids and bit-identical log-probs, for beam_size 1,
     beam_size 3 (the device search) and the greedy loop; wb_waveform_to_tokens equals wb_waveforms_to_tokens of that one
     waveform, ids and log-probs;
  2. a call rejected for an argument error leaves the session as the last successful call left it: the encoded windows,
     wb_session_last_logprobs and wb_session_last_timings."""
import numpy as np
import pytest
import torch

import harness as h
import wb200  # noqa: F401
from oracle import synth
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu
DEPTH = 12
# (search rule, beam_size)
SEARCHES = [("beam", 1), ("beam", 3), ("greedy_loop", 1)]


@pytest.fixture(scope="module")
def tiny():
    return h.named_model("test-a")


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def on_device(waves):
    """(device tensor, offsets, lens) of the windows concatenated in one CUDA tensor, each at a 16-byte aligned offset"""
    lens = [len(w) for w in waves]
    offsets = list(np.cumsum([0] + [(n + 3) // 4 * 4 for n in lens[:-1]]))
    flat = np.zeros(offsets[-1] + lens[-1], dtype=np.float32)
    for w, o in zip(waves, offsets):
        flat[o:o + len(w)] = w
    return torch.from_numpy(flat).cuda(), offsets, lens


@pytest.mark.parametrize("search,beam_size", SEARCHES)
def test_window_entry_points_agree(tiny, search, beam_size):
    dims, sp, wh, *_ = tiny
    waves = [synth.waveform(n, seed=70 + i) for i, n in enumerate((48000, 40000, 56000))]
    sess = transcribe.Session(wh, max_windows=3, max_beams=3, max_text_len=4 + DEPTH + 1, search=search)
    bm = None if search == "greedy_loop" else sp.is_special_bitmap()
    dev, offsets, lens = on_device(waves)
    runs = {
        "host": lambda: sess.transcribe_windows(waves, sp, bm, beam_size=beam_size, max_depth=DEPTH),
        "dev": lambda: sess.transcribe_windows_dev(dev.data_ptr(), offsets, lens, sp, bm, beam_size=beam_size, max_depth=DEPTH),
        "prev": lambda: sess.transcribe_windows_prev(waves, [[]] * 3, sp, bm, beam_size=beam_size, max_depth=DEPTH),
    }
    got = {}
    for name, run in runs.items():
        ids = run()
        if beam_size > 1:
            assert sess.last_decoder() == 6, name
        got[name] = (ids, [bits(sess.last_logprobs(r)) for r in range(3)])
    ids, lps = got["host"]
    assert all(len(t) > 4 for t in ids)
    for name in ("dev", "prev"):
        assert got[name][0] == ids, name
        for r in range(3):
            assert np.array_equal(got[name][1][r], lps[r]), f"{name} window {r}"


@pytest.mark.parametrize("search,beam_size", SEARCHES)
def test_waveform_is_the_one_waveform_batch(tiny, search, beam_size):
    dims, sp, wh, *_ = tiny
    wave = synth.waveform(400000, seed=9)   # 3 windows of the reference windowing
    sess = transcribe.Session(wh, max_windows=3, max_beams=3, max_text_len=4 + DEPTH + 1, search=search)
    bm = None if search == "greedy_loop" else sp.is_special_bitmap()
    one = sess.waveform_to_tokens(wave, sp, bm, beam_size=beam_size, max_depth=DEPTH)
    lp_one = bits(sess.last_logprobs(0))
    batch = sess.waveforms_to_tokens([wave], sp, bm, beam_size=beam_size, max_depth=DEPTH)
    assert batch[0] == one
    assert np.array_equal(bits(sess.last_logprobs(0)), lp_one)


def test_rejected_calls_leave_the_last_results(tiny):
    dims, sp, wh, *_ = tiny
    V = dims.n_vocab
    good = [synth.waveform(n, seed=80 + i) for i, n in enumerate((48000, 40000))]
    other = [synth.waveform(n, seed=90 + i) for i, n in enumerate((44000, 52000))]
    dev, offsets, lens = on_device(other)
    sess = transcribe.Session(wh, max_windows=2, max_beams=3, max_text_len=4 + DEPTH + 1)
    bm = sp.is_special_bitmap()

    def state():
        return ([bits(sess.get_encoder_output(w)) for w in range(2)], [bits(sess.last_logprobs(w)) for w in range(2)],
                sess.last_timings_ms())

    sess.transcribe_windows(good, sp, bm, beam_size=3, max_depth=DEPTH)
    want = state()
    bad_sp = synth.SpecialTokens(sot=V, lang=sp.lang, transcribe=sp.transcribe, notimestamps=sp.notimestamps, eot=sp.eot,
                                 first_special=sp.first_special, n_vocab=sp.n_vocab, startofprev=sp.startofprev)
    # each argument error as (special tokens, beam_size, max_depth, previous ids)
    errors = {"beam_size above max_beams": (sp, 4, DEPTH, [[]] * 2), "special id >= n_vocab": (bad_sp, 1, DEPTH, [[]] * 2),
              "negative max_depth": (sp, 1, -1, [[]] * 2)}
    calls = {
        "windows": lambda s, b, d, p: sess.transcribe_windows(other, s, bm, beam_size=b, max_depth=d),
        "windows_dev": lambda s, b, d, p: sess.transcribe_windows_dev(dev.data_ptr(), offsets, lens, s, bm, beam_size=b,
                                                                      max_depth=d),
        "windows_prev": lambda s, b, d, p: sess.transcribe_windows_prev(other, p, s, bm, beam_size=b, max_depth=d),
        "waveform": lambda s, b, d, p: sess.waveform_to_tokens(other[0], s, bm, beam_size=b, max_depth=d),
        "waveforms": lambda s, b, d, p: sess.waveforms_to_tokens(other, s, bm, beam_size=b, max_depth=d),
    }
    cases = [(c, e) + args for c in calls for e, args in errors.items()]
    cases.append(("windows_prev", "previous id out of range", sp, 1, DEPTH, [[1, V], []]))
    cases.append(("windows_prev", "greedy loop with previous ids", sp, 1, DEPTH, [[1, 2], []]))
    cases.append(("waveforms", "greedy loop with the previous-text prompt", sp, 1, DEPTH, None))
    cases.append(("waveform", "greedy loop with the previous-text prompt", sp, 1, DEPTH, None))

    for call, error, s, b, d, p in cases:
        loop = error.startswith("greedy loop")
        if loop:
            ffi.check(ffi.lib().wb_session_set_search(sess._h, ffi.WB_SEARCH_GREEDY_LOOP))
            if p is None:
                sess.set_prev_prompt(sp.startofprev)
        try:
            with pytest.raises(ffi.WbError) as e:
                calls[call](s, b, d, p)
            assert e.value.code == ffi.WB_ERR_INVALID_ARG, f"{call}: {error}: {e.value}"
        finally:
            if loop:
                ffi.check(ffi.lib().wb_session_set_search(sess._h, ffi.WB_SEARCH_BEAM))
                sess.set_prev_prompt(-1)
        got = state()
        for w in range(2):
            assert np.array_equal(got[0][w], want[0][w]), f"{call}: {error}: encoder output of window {w}"
            assert np.array_equal(got[1][w], want[1][w]), f"{call}: {error}: log-probs of window {w}"
        assert got[2] == want[2], f"{call}: {error}: timings"
