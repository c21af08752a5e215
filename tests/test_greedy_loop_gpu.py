"""GPU tests of the greedy loop (WB_SEARCH_GREEDY_LOOP, src/transcribe.rs:314-380): token ids identical to the oracle loop
(tests/oracle_greedy_loop.py) on every persistent decoder, on tiny.en at its real shape against a committed fixture, through
waveform_to_tokens, and the contract of the search rule.

Each decoder case runs a batch twice, with max_depth = max_text_len - 4 and with max_depth 3, and with a declared EOT id (500)
whose logit comes within ln 2 of the arg-max at some steps of the d = 128 synthetic model: across the two runs the EOT test,
the repetition cut and the context stop each end some window, which the test asserts from the oracle's record.  Where the oracle's
EOT-test gap or top-1 / top-2 logit gap falls below 1e-4 at a step, ids are compared up to that step (the decoders' logits
differ from the oracle's in the last bits)."""
import dataclasses
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_greedy_loop as loop
import wb200  # noqa: F401
from oracle import audio as o_audio, synth
from whisper_burn_b200 import ffi, model, transcribe

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"
GAP_TOL = 1e-4
EOT_ID = 500   # declared EOT of the synthetic models: an ordinary id whose logit is sometimes within ln 2 of the arg-max

_MODELS, _ORACLE = {}, {}


def weights(name):
    if name not in _MODELS:
        dims, w_np, w_t = synth.make_weights(name, seed=0)
        _MODELS[name] = (dims, w_t, model.Whisper(dims, w_np))
    return _MODELS[name]


def window(i):
    return synth.waveform(16000 * (3 + 4 * (i % 4)) + 1600 * (i // 4), seed=100 + i)


def oracle(name, i, sp, max_depth, kv):
    key = (name, i, sp.eot, max_depth, kv)
    if key not in _ORACLE:
        dims, w_t, _ = weights(name)
        mel = o_audio.prep_audio(torch.from_numpy(window(i))[None])
        tr = {}
        toks = loop.mels_to_tokens_greedy_loop(w_t, dims, sp, mel, max_depth, loop.model.OracleOptions(kv_dtype=kv), trace=tr)
        _ORACLE[key] = (toks, tr)
    return _ORACLE[key]


def same_up_to_ties(got, want, tr):
    """got == want, or identical up to the first step whose EOT-test or top-1/top-2 gap is below GAP_TOL."""
    if got == want:
        return True
    for s, (e, t) in enumerate(zip(tr["eot_gap"], tr["top_gap"])):
        if abs(e) < GAP_TOL or t < GAP_TOL:
            return got[:4 + s] == want[:4 + s]
    return False


def session(name, n, t_max, kv, search="greedy_loop"):
    _, _, wh = weights(name)
    return transcribe.Session(wh, max_windows=n, max_beams=1, max_text_len=t_max,
                              kv_dtype=ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32, search=search)


# (decoder, model, windows, max_text_len, rules that end some window): decoder6 takes t_max <= 128 and 8+ rows here;
# decoder5 needs d % 256 == 0 (test-c, whose logits never put id 500 within ln 2 of the arg-max on these windows)
ALL = {"eot", "repeat", "context"}
CASES = [(4, "test-a", 4, 448, ALL), (6, "test-a", 9, 128, ALL), (5, "test-c", 4, 448, {"repeat", "context"}),
         (3, "test-a", 4, 448, ALL)]


@pytest.mark.parametrize("kv", ["f32", "f16"])
@pytest.mark.parametrize("dec,name,n,t_max,rules", CASES)
def test_each_decoder_matches_the_oracle_loop(monkeypatch, dec, name, n, t_max, rules, kv):
    dims, _, _ = weights(name)
    sp = dataclasses.replace(synth.special_tokens(dims), eot=EOT_ID)
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
            assert got[i][-1] == EOT_ID and len(got[i]) <= 4 + max_depth + 1
    assert stops == rules, stops
    s.close()


@pytest.mark.parametrize("kv", ["f32", "f16"])
def test_tiny_en_real_shape_against_fixture(kv):
    g = json.loads((G / "tokens_greedy_loop.json").read_text())
    dims, _, wh = weights("tiny.en")
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
    dims, w_t, _ = weights("test-a")
    sp = dataclasses.replace(synth.special_tokens(dims), eot=EOT_ID)
    wave = synth.waveform(16000 * 35, seed=77)   # 3 reference windows
    want = loop.waveform_to_tokens(w_t, dims, sp, wave, beam_size=1, max_depth=60, search="greedy_loop")
    s = session("test-a", 2, 65, "f32")
    got = s.waveform_to_tokens(wave, sp, None, beam_size=1, max_depth=60)
    assert got == want
    s.close()


def test_search_rule_contract():
    dims, _, wh = weights("test-a")
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
