"""The oracle's per-token log-probs (tests/oracle_logprobs.py), which the GPU tests of wb_session_last_logprobs compare against:
the opt-in return changes no id, greedy values are the chosen entries of the search's own log-softmax rows, a beam row sums to
the score the search chose it by, the greedy loop marks exactly its rule-appended EOTs NaN, and the merge carries every log-prob
with its id."""
import dataclasses
import math

import numpy as np
import pytest
import torch

import oracle_greedy_loop as loop
import oracle_logprobs as olp
from oracle import audio as o_audio, synth, transcribe as o_tr

EOT_ID = 500   # as in test_greedy_loop_gpu.py: an ordinary id of test-a whose logit is sometimes within ln 2 of the arg-max


@pytest.fixture(scope="module")
def test_a():
    dims, _, w_t = synth.make_weights("test-a", seed=0)
    return dims, w_t, synth.special_tokens(dims)


def mel_of(wave):
    return o_audio.prep_audio(torch.from_numpy(wave)[None])


def window(i):
    return synth.waveform(16000 * (3 + 4 * (i % 4)) + 1600 * (i // 4), seed=100 + i)


@pytest.mark.parametrize("beam_size", [1, 5])
def test_opt_in_gives_the_default_ids(test_a, beam_size):
    dims, w_t, sp = test_a
    mel = mel_of(window(1))
    ids, lps, _ = olp.mels_to_token_logprobs(w_t, dims, sp, mel, beam_size, 12)
    assert ids == o_tr.mels_to_tokens(w_t, dims, sp, mel, beam_size, 12)
    assert len(lps) == len(ids) and lps[:4] == [0.0] * 4
    assert all(math.isfinite(v) and v <= 0 for v in lps)


def test_greedy_values_are_the_chosen_log_softmax_entries(test_a):
    dims, w_t, sp = test_a
    for i in range(3):
        tr = {}
        ids, lps, score = olp.mels_to_token_logprobs(w_t, dims, sp, mel_of(window(i)), 1, 15, trace=tr)
        rows = tr["log_probs"]
        assert len(rows) == len(ids) - 4
        for s, t in enumerate(ids[4:]):
            assert lps[4 + s] == float(np.float32(rows[s][0][t]))
        assert score == sum(lps)


@pytest.mark.parametrize("beam_size", [2, 3, 4, 5, 6, 7])
def test_beam_row_sums_to_its_carried_score(test_a, beam_size):
    dims, w_t, sp = test_a
    for i in (0, 2):
        ids, lps, score = olp.mels_to_token_logprobs(w_t, dims, sp, mel_of(window(i)), beam_size, 12)
        total = 0.0
        for v in lps:   # left to right in f64, as the search accumulates (transcribe.rs:291-299)
            total += v
        assert total == score
        assert all(v == float(np.float32(v)) for v in lps)   # widened f32 values


def test_greedy_loop_marks_exactly_its_appended_eots(test_a):
    dims, w_t, sp = test_a
    sp = dataclasses.replace(sp, eot=EOT_ID)
    stops = set()
    for max_depth in (40, 3):
        for i in range(4):
            tr = {}
            ids, lps = olp.greedy_loop_logprobs(w_t, dims, sp, mel_of(window(i)), max_depth, trace=tr)
            assert ids == loop.mels_to_tokens_greedy_loop(w_t, dims, sp, mel_of(window(i)), max_depth)
            stops.add(tr["stop"])
            nan = [j for j, v in enumerate(lps) if math.isnan(v)]
            appended = tr["stop"] != "eot" or len(ids) - 4 > len(tr["eot_gap"])   # EOT after the arg-max id
            assert nan == ([len(ids) - 1] if appended else []), (tr["stop"], ids)
            assert all(v <= 0 for v in lps if not math.isnan(v))
    assert "context" in stops and len(stops) >= 2, stops


def test_greedy_loop_values_are_unmasked_teacher_forced_scores(test_a):
    dims, w_t, sp = test_a
    sp = dataclasses.replace(sp, eot=EOT_ID)
    mel = mel_of(window(1))
    ids, lps = olp.greedy_loop_logprobs(w_t, dims, sp, mel, 20)
    from oracle import model as o_model
    xa = o_model.forward_encoder(w_t, dims, o_tr.pad_mel(mel, dims.n_audio_ctx))
    rows = o_tr.greedy_path_log_probs(w_t, dims, olp.unmasked(sp), xa, ids)
    for j in range(4, len(ids)):
        if not math.isnan(lps[j]):
            assert abs(lps[j] - float(rows[j - 4][ids[j]])) < 1e-5


def test_merged_log_probs_follow_their_ids(test_a):
    dims, w_t, sp = test_a
    wave = synth.waveform(16000 * 35, seed=77)   # 3 reference windows
    window_len = o_audio.max_waveform_samples(dims.n_audio_ctx - o_tr.PADDING)
    per = []
    for s, e in o_tr.window_bounds(len(wave), 16000, window_len):
        ids, lps, _ = olp.mels_to_token_logprobs(w_t, dims, sp, mel_of(np.ascontiguousarray(wave[s:e])), 1, 20)
        per.append((ids, lps))
    assert len(per) == 3
    ids, lps = olp.merge(per)
    assert ids == o_tr.waveform_to_tokens(w_t, dims, sp, wave, beam_size=1, max_depth=20)
    # every merged (id, log-prob) pair is a pair of some window, in window order
    src = [(t, v) for w_ids, w_lps in per for t, v in zip(w_ids, w_lps)]
    k = 0
    for pair in zip(ids, lps):
        while src[k] != pair:
            k += 1
        k += 1
