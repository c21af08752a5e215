"""Oracle restatement of the reference's greedy loop (src/transcribe.rs:314-380, left commented out there), line by line, for
the tests of WB_SEARCH_GREEDY_LOOP.  It sits beside the oracle package and uses only it: the cached decoder, raw logits,
torch's first-max argmax, the f64 EOT test and the oracle's find_repeated_tokens_index.

    loop {
        if tokens.len() >= n_ctx_max_decoder { tokens.push(end_token); break; }            :317-320
        ... last_row = logits of the last position (no special-token mask)                 :322-332
        token_id = argmax(last_row); token_logit, eot_logit as f64                         :334-349
        tokens.push(token_id);
        if (eot_logit - token_logit).exp() > 0.5 { if token_id != end_token { push EOT } break; }     :351-356
        if let Some((_, end)) = find_repeated_tokens_index(&tokens, 5, 4) { truncate(end); push EOT; break; }   :358-377
    }

max_depth caps the loop as the library does: the context stop fires at min(n_text_ctx, len(prompt) + max_depth) tokens;
max_depth = n_text_ctx - 4 is the reference's loop.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional

import numpy as np
import torch

from oracle import audio, model, transcribe

REPEAT_WINDOW = 5   # transcribe.rs:358
MIN_REPEATS = 4     # transcribe.rs:359
LN_HALF = math.log(0.5)


def greedy_loop(prompt: List[int], eot: int, n_text_ctx: int, logits_of: Callable[[List[int]], torch.Tensor],
                max_depth: Optional[int] = None, trace: Optional[dict] = None) -> List[int]:
    """The loop over any `logits_of(tokens)` -> f32 [V] raw logits of the position after `tokens`.  trace (optional) gets,
    per step, "eot_gap": (eot_logit - token_logit) - ln 0.5 (the EOT test fires when it is > 0) and "top_gap": the top-1 /
    top-2 logit gap, "second_id": the top-2 id, and "stop": "eot" | "repeat" | "context"."""
    limit = n_text_ctx if max_depth is None else min(n_text_ctx, len(prompt) + max_depth)
    tokens = list(prompt)
    if trace is not None:
        trace.setdefault("eot_gap", [])
        trace.setdefault("top_gap", [])
        trace.setdefault("second_id", [])
    while True:
        if len(tokens) >= limit:
            tokens.append(eot)
            stop = "context"
            break
        last_row = logits_of(tokens)
        token_id = int(torch.argmax(last_row))            # the first maximum
        token_logit = float(last_row[token_id])           # f32 -> f64
        eot_logit = float(last_row[eot])
        tokens.append(token_id)
        if trace is not None:
            top2 = torch.topk(last_row.double(), 2)
            trace["eot_gap"].append((eot_logit - token_logit) - LN_HALF)
            trace["top_gap"].append(float(top2.values[0] - top2.values[1]))
            trace["second_id"].append(int(top2.indices[1]))
        if math.exp(eot_logit - token_logit) > 0.5:
            if token_id != eot:
                tokens.append(eot)
            stop = "eot"
            break
        rep = transcribe.find_repeated_tokens_index(tokens, REPEAT_WINDOW, MIN_REPEATS)
        if rep is not None:
            _, end = rep
            del tokens[end:]
            tokens.append(eot)
            stop = "repeat"
            break
    if trace is not None:
        trace["stop"] = stop
    return tokens


def mels_to_tokens_greedy_loop(w: dict, dims: model.WhisperDims, sp, mels: torch.Tensor, max_depth: Optional[int] = None,
                               opts: model.OracleOptions = model.DEFAULT_OPTS, trace: Optional[dict] = None) -> List[int]:
    """mels_to_text (transcribe.rs:148-383) with the greedy loop instead of the beam search, ids only."""
    mels = transcribe.pad_mel(mels, dims.n_audio_ctx)
    encoder_output = model.forward_encoder(w, dims, mels, opts)
    dec = model.CachedDecoder(w, dims, encoder_output, opts)
    last = {"logits": None}

    def logits_of(tokens):
        for t in tokens[dec.t:]:                          # tokens only grow between calls
            last["logits"] = dec.step(torch.tensor([t], dtype=torch.int64))[0]
        return last["logits"]

    return greedy_loop(sp.prompt(), sp.eot, dims.n_text_ctx, logits_of, max_depth, trace)


def waveform_to_tokens(w: dict, dims: model.WhisperDims, sp, waveform: np.ndarray, sample_rate: int = 16000,
                       beam_size: int = transcribe.BEAM_SIZE, max_depth: int = transcribe.MAX_DEPTH,
                       opts: model.OracleOptions = model.DEFAULT_OPTS, search: str = "beam") -> List[int]:
    """oracle.transcribe.waveform_to_tokens with a search rule: "beam" is that function, "greedy_loop" decodes every window
    with the loop (beam_size must be 1).  Windowing and the overlap merge are the same."""
    if search == "beam":
        return transcribe.waveform_to_tokens(w, dims, sp, waveform, sample_rate, beam_size, max_depth, opts=opts)
    if search != "greedy_loop" or beam_size != 1:
        raise ValueError(f"search {search!r} with beam_size {beam_size}")
    window_len = audio.max_waveform_samples(dims.n_audio_ctx - transcribe.PADDING)
    tokens: List[int] = []
    for (s, e) in transcribe.window_bounds(len(waveform), sample_rate, window_len):
        mel = audio.prep_audio(torch.from_numpy(np.ascontiguousarray(waveform[s:e])).unsqueeze(0), float(sample_rate))
        new_tokens = mels_to_tokens_greedy_loop(w, dims, sp, mel, max_depth, opts)
        ov = transcribe.find_chunk_overlap(tokens, new_tokens, 40, 3)
        if ov is not None:
            tokens = tokens[:ov[0]] + new_tokens[ov[1]:]
        else:
            tokens = tokens + new_tokens
    return tokens
