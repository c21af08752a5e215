"""GPU tests (-m gpu) of the on-device beam search: with fp16-exact weights, d = 128 / 384 and n_windows * beam_size <= 24,
transcribe_windows runs prefill and the whole width-B search in one decoder6 launch.  It must give the oracle's ids
(tests/golden/tokens_beam.json, make_golden_beam.py), and the same ids as the host search driven through decoder3."""
import pytest
import torch

import harness as h
import wb200  # noqa: F401
from harness import is_special_of, kv_code, pool_waves
from oracle import audio as o_audio, model as o_model, synth, transcribe as o_tr
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    return h.golden("tokens_beam")


@pytest.fixture(scope="module")
def small():
    return h.named_model("test-a")


@pytest.fixture(scope="module")
def tiny():
    return h.named_model("tiny.en")


def decode(wh, waves, sp, b, depth, kv, host=False, monkeypatch=None, max_text_len=None):
    if host:
        monkeypatch.setenv("WB200_DECODER", "3")   # the host search on the FMA decoder: a second reference
    try:
        sess = transcribe.Session(wh, max_windows=len(waves), max_beams=7, max_text_len=max_text_len or 4 + depth + 1,
                                  kv_dtype=kv_code(kv))
    finally:
        if host:
            monkeypatch.delenv("WB200_DECODER", raising=False)
    got = sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=b, max_depth=depth)
    return got, sess


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("b", [2, 3, 4, 5, 6, 7])
def test_device_beam_test_a_vs_oracle_and_host(small, gold, monkeypatch, b, kv):
    """test-a (d = 128): 1 .. 24 // B windows of mixed lengths in one launch each"""
    _, sp, wh, *_ = small
    depth = gold["depth_test_a"]
    want = gold["test_a"][kv][str(b)]
    n_max = 24 // b
    for n in range(1, n_max + 1):
        waves = pool_waves(gold, n)
        got, sess = decode(wh, waves, sp, b, depth, kv)
        assert sess.last_decoder() == 6, n
        assert got == [want[i % len(gold["pool"])] for i in range(n)], n
    host, hs = decode(wh, waves, sp, b, depth, kv, host=True, monkeypatch=monkeypatch)
    assert hs.last_decoder() == 3
    assert host == got
    assert hs.last_steps() == sess.last_steps() == depth


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_device_beam_tiny_en_vs_oracle_and_host(tiny, gold, monkeypatch, kv):
    """tiny.en (d = 384): the three reference windows of chunk 0, beam 5, depth 30"""
    _, sp, wh, *_ = tiny
    te = h.golden("tokens_tiny_en")
    chunk = synth.chunk_waveform(0)
    waves = [chunk[s:e] for s, e in te["bounds"]]
    got, sess = decode(wh, waves, sp, 5, gold["depth_tiny_en"], kv)
    assert sess.last_decoder() == 6
    assert got == gold["tiny_en"][kv]["5"]
    host, hs = decode(wh, waves, sp, 5, gold["depth_tiny_en"], kv, host=True, monkeypatch=monkeypatch)
    assert hs.last_decoder() == 3 and host == got and hs.last_steps() == sess.last_steps()


DEEP = 124   # 4 + 124 = 128, the longest text decoder6 holds: the last step attends over 127 keys


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("b", [2, 5, 7])
def test_device_beam_test_a_deep_vs_oracle_and_host(small, gold, monkeypatch, b, kv):
    """test-a at max_depth 124 (max_text_len 128): self attention through all four of decoder6's 32-key slots, the keys read
    through the ancestry tables, beam sequences copied to 128 ids.  EOT is declared to be the last vocabulary id, which
    these searches never emit, so every window runs all 124 steps.  The same ids as the live oracle and as the host search
    on decoder3, and the same number of steps."""
    dims, sp, wh, _, w_t, _ = small
    sp2 = o_tr.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, sp.n_vocab - 1, sp.first_special, sp.n_vocab)
    waves = pool_waves(gold, min(len(gold["pool"]), 24 // b))
    got, sess = decode(wh, waves, sp2, b, DEEP, kv, max_text_len=4 + DEEP)
    assert sess.last_decoder() == 6 and sess.last_steps() == DEEP
    host, hs = decode(wh, waves, sp2, b, DEEP, kv, host=True, monkeypatch=monkeypatch, max_text_len=4 + DEEP)
    assert hs.last_decoder() == 3 and hs.last_steps() == DEEP
    assert host == got
    opts = o_model.OracleOptions(kv_dtype=kv)
    for i, wave in enumerate(waves):
        want = o_tr.mels_to_tokens(w_t, dims, sp2, o_audio.prep_audio(torch.from_numpy(wave)[None]), beam_size=b,
                                   max_depth=DEEP, opts=opts)
        assert len(want) == 4 + DEEP and got[i] == want, f"window {i}"


def test_device_beam_live_oracle(small):
    """one case against the oracle computed here (the golden file is the oracle's output too)"""
    dims, sp, wh, _, w_t, _ = small
    wave = synth.chunk_waveform(0)[120000:120000 + 98882]
    got, sess = decode(wh, [wave], sp, 4, 8, "f16")
    want = o_tr.mels_to_tokens(w_t, dims, sp, o_audio.prep_audio(torch.from_numpy(wave)[None]), beam_size=4, max_depth=8,
                               opts=o_model.OracleOptions(kv_dtype="f16"))
    assert sess.last_decoder() == 6 and got[0] == want


def test_device_beam_early_stop(small, gold, monkeypatch):
    """EOT declared to be a token the search emits: one window's search ends early (its sequence ends in EOT) while the other
    continues; the launch stops when both are done, after as many steps as the host search takes."""
    dims, sp, wh, *_ = small
    ta = h.golden("tokens_test_a")
    eot = gold["eot"]
    sp2 = o_tr.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, eot, sp.first_special, sp.n_vocab)
    chunk = synth.chunk_waveform(0)
    waves = [chunk[:238559], chunk[:98882]]
    got, sess = decode(wh, waves, sp2, 5, 30, "f32")
    assert sess.last_decoder() == 6
    assert got[0] == ta["eot_case_beam5"]["tokens"] and got[1] == gold["eot_window1"]
    short, long_ = sorted(got, key=len)
    assert short[-1] == eot and len(short) < len(long_)
    host, hs = decode(wh, waves, sp2, 5, 30, "f32", host=True, monkeypatch=monkeypatch)
    assert host == got and hs.last_steps() == sess.last_steps() <= 30


def test_device_beam_is_one_launch(small, gold, monkeypatch):
    """The whole search is one launch: the library launches as many kernels at depth 30 as at depth 5; the host search
    launches more per depth."""
    _, sp, wh, *_ = small
    waves = pool_waves(gold, 2)

    def launches(sess, depth):
        ffi.lib().wb_kernel_launch_count_reset()
        sess.transcribe_windows(waves, sp, is_special_of(sp), beam_size=5, max_depth=depth)
        return ffi.lib().wb_kernel_launch_count()

    sess = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=4 + 30 + 1)
    launches(sess, 5)                                   # packs the decoder6 weights once
    n5, n30 = launches(sess, 5), launches(sess, 30)
    assert sess.last_decoder() == 6 and sess.last_steps() == 30
    assert n30 == n5
    monkeypatch.setenv("WB200_DECODER", "3")
    hs = transcribe.Session(wh, max_windows=2, max_beams=5, max_text_len=4 + 30 + 1)
    monkeypatch.delenv("WB200_DECODER")
    assert launches(hs, 30) > launches(hs, 5)


def test_device_beam_coverage_edge(small, gold):
    """24 rows (4 windows x B = 6) are one decoder6 launch; 25 rows (5 windows x B = 5) fall back to the host search, with
    the same ids"""
    _, sp, wh, *_ = small
    depth = gold["depth_test_a"]
    got, sess = decode(wh, pool_waves(gold, 4), sp, 6, depth, "f32")
    assert sess.last_decoder() == 6
    assert got == gold["test_a"]["f32"]["6"][:4]
    got, sess = decode(wh, pool_waves(gold, 5), sp, 5, depth, "f32")
    assert sess.last_decoder() == 3
    assert got == gold["test_a"]["f32"]["5"][:5]
