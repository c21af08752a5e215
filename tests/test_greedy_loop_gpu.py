"""GPU tests of the greedy loop (WB_SEARCH_GREEDY_LOOP, src/transcribe.rs:314-380): token ids identical to the oracle loop
(tests/oracle_greedy_loop.py) on every persistent decoder, on tiny.en at its real shape against a committed fixture, through
waveform_to_tokens, and the contract of the search rule.

Each decoder case runs a batch twice, with max_depth = max_text_len - 4 and with max_depth 3, and with a declared EOT id (500)
whose logit comes within ln 2 of the arg-max at some steps of the d = 128 synthetic model: across the two runs the EOT test,
the repetition cut and the context stop each end some window, which the test asserts from the oracle's record.  Where the oracle's
EOT-test gap or top-1 / top-2 logit gap falls below 1e-4 at a step, ids are compared up to that step (the decoders' logits
differ from the oracle's in the last bits)."""
import dataclasses

import pytest
import torch

import oracle_greedy_loop as loop
import wb200  # noqa: F401
from harness import LOOP_CASES, LOOP_EOT_ID, golden, loop_model, loop_session as session, loop_window as window, \
    same_up_to_ties
from oracle import audio as o_audio, synth
from whisper_burn_b200 import ffi, transcribe

pytestmark = pytest.mark.gpu

_ORACLE = {}


def oracle(name, i, sp, max_depth, kv):
    key = (name, i, sp.eot, max_depth, kv)
    if key not in _ORACLE:
        dims, _, _, _, w_t, _ = loop_model(name)
        mel = o_audio.prep_audio(torch.from_numpy(window(i))[None])
        tr = {}
        toks = loop.mels_to_tokens_greedy_loop(w_t, dims, sp, mel, max_depth, loop.model.OracleOptions(kv_dtype=kv), trace=tr)
        _ORACLE[key] = (toks, tr)
    return _ORACLE[key]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("dec,name,n,t_max,rules", LOOP_CASES)
def test_each_decoder_matches_the_oracle_loop(monkeypatch, dec, name, n, t_max, rules, kv):
    dims = loop_model(name).dims
    sp = dataclasses.replace(synth.special_tokens(dims), eot=LOOP_EOT_ID)
    monkeypatch.setenv("WB200_DECODER", str(dec))
    s = session(name, n, t_max, kv)
    monkeypatch.delenv("WB200_DECODER")
    waves = [window(i) for i in range(n)]
    stops = set()
    for max_depth in (t_max - 4, 3):
        got = s.transcribe_windows(waves, sp, None, beam_size=1, max_depth=max_depth)
        assert s.last_decoder() == dec
        for i in range(n):
            want, tr = oracle(name, i, sp, max_depth, kv)
            stops.add(tr["stop"])
            assert same_up_to_ties(got[i], want, tr), f"window {i} depth {max_depth}:\n got {got[i]}\nwant {want}"
            assert got[i][-1] == LOOP_EOT_ID and len(got[i]) <= 4 + max_depth + 1
    assert stops == rules, stops
    s.close()


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_tiny_en_real_shape_against_fixture(kv):
    g = golden("tokens_greedy_loop")
    dims = loop_model("tiny.en").dims
    sp = synth.special_tokens(dims)
    assert g["eot"] == sp.eot
    chunk = synth.chunk_waveform(g["chunk"])
    waves = [chunk[s:e] for s, e in g["bounds"]]
    s = session("tiny.en", len(waves), dims.n_text_ctx, kv)
    got = s.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=g["max_depth"])
    for i, rec in enumerate(g[kv]):
        assert same_up_to_ties(got[i], rec["tokens"], rec), f"window {i}:\n got {got[i]}\nwant {rec['tokens']}"
    s.close()


def test_waveform_to_tokens_in_loop_mode():
    dims, _, _, _, w_t, _ = loop_model("test-a")
    sp = dataclasses.replace(synth.special_tokens(dims), eot=LOOP_EOT_ID)
    wave = synth.waveform(16000 * 35, seed=77)   # 3 reference windows
    want = loop.waveform_to_tokens(w_t, dims, sp, wave, beam_size=1, max_depth=60, search="greedy_loop")
    s = session("test-a", 2, 65, "f32")
    got = s.waveform_to_tokens(wave, sp, None, beam_size=1, max_depth=60)
    assert got == want
    s.close()


def test_search_rule_contract():
    dims, _, wh, *_ = loop_model("test-a")
    sp = synth.special_tokens(dims)
    s = session("test-a", 1, 20, "f32")
    with pytest.raises(ffi.WbError) as e:
        s.transcribe_windows([window(0)], sp, None, beam_size=2, max_depth=5)
    assert e.value.code == ffi.WB_ERR_INVALID_ARG
    assert ffi.lib().wb_session_set_search(s._h, 2) == ffi.WB_ERR_INVALID_ARG
    assert ffi.lib().wb_session_set_search(s._h, ffi.WB_SEARCH_BEAM) == ffi.WB_OK
    with pytest.raises(ffi.WbError) as e:   # the beam rule still needs is_special
        s.transcribe_windows([window(0)], sp, None, beam_size=1, max_depth=5)
    assert e.value.code == ffi.WB_ERR_INVALID_ARG
    s.close()
    with pytest.raises(ValueError):
        transcribe.Session(wh, max_windows=1, max_beams=1, max_text_len=20, search="greedy")
