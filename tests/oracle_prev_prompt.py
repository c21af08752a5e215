"""Oracle restatement of the previous-text prompt (TEST INFRASTRUCTURE): what src/transcribe.rs computes with line 201
(`let mut initial_tokens = Vec::new();`) removed.

  * waveform_to_text (transcribe.rs:43-54) collects the last at most 5 ids of the merged tokens that are not special, in
    order, and passes them to mels_to_text as prev_nonspecial_tokens;
  * mels_to_text (transcribe.rs:195-203) prompts the window with [startofprev] + prev + [sot, lang, transcribe,
    notimestamps] when prev is not empty, else with the 4 ids.

mels_to_tokens of oracle.transcribe takes any prompt through SpecialTokens.prompt(); its cached prefill and the mask rule
(masks_specials on the longest beam) need nothing else."""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Sequence

import numpy as np
import torch

from oracle import audio, transcribe as o_tr

N_PREV = 5   # transcribe.rs:48, .take(5)


@dataclasses.dataclass(frozen=True)
class PromptedTokens(o_tr.SpecialTokens):
    """The special ids with a given prompt in place of the 4-id one."""
    given: tuple = ()

    def prompt(self) -> List[int]:
        return list(self.given)


def oracle_special(sp) -> o_tr.SpecialTokens:
    return o_tr.SpecialTokens(sot=sp.sot, lang=sp.lang, transcribe=sp.transcribe, notimestamps=sp.notimestamps, eot=sp.eot,
                              first_special=sp.first_special, n_vocab=sp.n_vocab)


def build_prompt(sp, prev: Sequence[int], startofprev: Optional[int] = None) -> List[int]:
    """transcribe.rs:195-203 without the shadowing at :201."""
    sop = sp.startofprev if startofprev is None else startofprev
    head = [sp.sot, sp.lang, sp.transcribe, sp.notimestamps]
    return ([sop] + [int(t) for t in prev] + head) if len(prev) else head


def prev_nonspecial(tokens: Sequence[int], is_special) -> List[int]:
    """transcribe.rs:43-50: the last at most 5 ids with is_special 0, in their original order."""
    out = [int(t) for t in reversed(tokens) if not is_special(int(t))][:N_PREV]
    return out[::-1]


def with_prompt(sp, prompt: Sequence[int]) -> PromptedTokens:
    b = oracle_special(sp)
    return PromptedTokens(**dataclasses.asdict(b), given=tuple(int(t) for t in prompt))


def mels_to_tokens(w, dims, sp, mel: torch.Tensor, prompt: Sequence[int], beam_size: int, max_depth: int, **kw) -> List[int]:
    """mels_to_text from a given prompt."""
    return o_tr.mels_to_tokens(w, dims, with_prompt(sp, prompt), mel, beam_size, max_depth, **kw)


def waveform_to_tokens(w, dims, sp, waveform: np.ndarray, beam_size: int, max_depth: int, prev_prompt: bool = True,
                       sample_rate: int = 16000, per_window: Optional[list] = None, **kw) -> List[int]:
    """waveform_to_text (transcribe.rs:23-74) with the previous-text prompt when prev_prompt, else exactly
    oracle.transcribe.waveform_to_tokens.  per_window receives (prompt, new_tokens) of every window."""
    window_len = audio.max_waveform_samples(dims.n_audio_ctx - o_tr.PADDING)
    tokens: List[int] = []
    for (s, e) in o_tr.window_bounds(len(waveform), sample_rate, window_len):
        mel = audio.prep_audio(torch.from_numpy(np.ascontiguousarray(waveform[s:e])).unsqueeze(0), float(sample_rate))
        prompt = build_prompt(sp, prev_nonspecial(tokens, sp.is_special) if prev_prompt else [])
        new_tokens = mels_to_tokens(w, dims, sp, mel, prompt, beam_size, max_depth, **kw)
        if per_window is not None:
            per_window.append((prompt, list(new_tokens)))
        ov = o_tr.find_chunk_overlap(tokens, new_tokens, 40, 3)
        if ov is not None:
            tokens = tokens[:ov[0]] + new_tokens[ov[1]:]
        else:
            tokens = tokens + new_tokens
    return tokens
