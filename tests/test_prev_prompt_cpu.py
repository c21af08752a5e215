"""CPU tests of the previous-text prompt's oracle restatement (tests/oracle_prev_prompt.py), which the GPU tests of
test_prev_prompt_gpu.py compare against: the prompt rule of transcribe.rs:43-54, 195-203 without the shadowing at :201."""
import numpy as np
import torch

import oracle_prev_prompt as opp
import wb200  # noqa: F401
from oracle import audio as o_audio, synth, transcribe as o_tr


def test_prompt_from_merged_tokens():
    dims = synth.MODEL_DIMS["test-a"]
    sp = synth.special_tokens(dims)
    assert sp.startofprev == sp.eot + 5 and sp.is_special(sp.startofprev)
    assert sp.startofprev not in (sp.sot, sp.lang, sp.transcribe, sp.notimestamps, sp.eot)
    head = [sp.sot, sp.lang, sp.transcribe, sp.notimestamps]
    assert opp.build_prompt(sp, []) == head   # window 0
    assert opp.build_prompt(sp, [7, 8]) == [sp.startofprev, 7, 8] + head
    merged = head + [1, 2, sp.eot, 3, 4, sp.startofprev, 5, 6] + head
    assert opp.prev_nonspecial(merged, sp.is_special) == [2, 3, 4, 5, 6]   # specials skipped, last 5 in order
    assert opp.prev_nonspecial(head + [9, sp.eot], sp.is_special) == [9]   # fewer than 5 available
    assert opp.prev_nonspecial(head, sp.is_special) == []


def test_rule_off_equals_oracle_waveform_to_tokens_and_on_differs():
    dims, _, w_t = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    win = o_audio.max_waveform_samples(dims.n_audio_ctx - o_tr.PADDING)
    wave = synth.waveform(win + 2 * (win - 48000) - 100, seed=101)   # 3 windows
    off = opp.waveform_to_tokens(w_t, dims, sp, wave, 1, 16, prev_prompt=False)
    assert off == o_tr.waveform_to_tokens(w_t, dims, opp.oracle_special(sp), wave, beam_size=1, max_depth=16)
    per_on, per_off = [], []
    opp.waveform_to_tokens(w_t, dims, sp, wave, 1, 16, per_window=per_on)
    opp.waveform_to_tokens(w_t, dims, sp, wave, 1, 16, prev_prompt=False, per_window=per_off)
    assert per_on[0] == per_off[0]
    assert all(len(p) > 4 for p, _ in per_on[1:])
    # the ids generated after the prompt differ in at least one later window, so the GPU tests can tell the rule from none
    assert any(t[len(p):] != u[4:] for (p, t), (_, u) in zip(per_on[1:], per_off[1:]))


def test_long_prompt_is_never_masked():
    dims, _, w_t = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    assert o_tr.masks_specials(5) and not o_tr.masks_specials(6)
    mel = o_audio.prep_audio(torch.from_numpy(synth.waveform(48000, seed=3))[None])
    enc = o_tr.model.forward_encoder(w_t, dims, o_tr.pad_mel(mel, dims.n_audio_ctx))
    prompt = opp.build_prompt(sp, [11])   # 6 ids: the first step's sequence already has 6 tokens
    rows = o_tr.greedy_path_log_probs(w_t, dims, opp.oracle_special(sp), enc, prompt + [0], n_prompt=len(prompt))
    assert torch.isfinite(rows[0][sp.first_special:]).all()
    rows4 = o_tr.greedy_path_log_probs(w_t, dims, opp.oracle_special(sp), enc, opp.build_prompt(sp, []) + [0])
    assert torch.isinf(rows4[0][sp.first_special:]).all()
