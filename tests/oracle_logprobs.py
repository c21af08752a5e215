"""The oracle's per-token log-probs, for the tests of wb_session_last_logprobs.  The oracle carries them already: its beam search
runs over (token, log-prob) pairs, BeamSearchToken { token, log_prob } of the reference (src/transcribe.rs:142-146, prompt at
0.0, :205-208), and strips them at the end (:309-312).  This module returns them instead, without changing the oracle:

  * mels_to_token_logprobs: oracle.transcribe.mels_to_tokens, returning (ids, log-probs, the winning beam's carried score);
  * greedy_loop_logprobs: the greedy loop of oracle_greedy_loop, with log_softmax of the unmasked logits at each arg-max id
    and NaN for an EOT a rule appended (EOT test, repetition cut, context stop);
  * unmasked: special tokens that mask nothing, so oracle.transcribe.greedy_path_log_probs scores a greedy-loop path;
  * merge: the overlap merge of waveform_to_text (transcribe.rs:56-63) carrying each log-prob with its id.
"""
from __future__ import annotations

import contextlib
import dataclasses
import math
from typing import List, Optional, Tuple

import numpy as np
import torch

import oracle_greedy_loop as loop
from oracle import beam, model, transcribe


@contextlib.contextmanager
def _capture_best_beam(out: dict):
    """While active, oracle.beam.beam_search records the (token, log-prob) sequence it returns and, from its step trace, the
    carried log-prob of that beam (BeamNode.log_prob, 0.0 when no step ran)."""
    search = beam.beam_search

    def recording(initial_beams, next_fn, is_finished, beam_size, max_depth, trace=None):
        steps = [] if trace is None else trace
        seq = search(initial_beams, next_fn, is_finished, beam_size, max_depth, trace=steps)
        final = [beam.BeamNode(list(s), lp) for s, lp in steps[-1]] if steps else initial_beams
        best = beam._max_by_last(final)
        assert best is not None and list(best.seq) == seq
        out["seq"], out["score"] = seq, best.log_prob
        return seq

    beam.beam_search = recording
    try:
        yield
    finally:
        beam.beam_search = search


def mels_to_token_logprobs(w: dict, dims: model.WhisperDims, sp: transcribe.SpecialTokens, mels: torch.Tensor,
                           beam_size: int = transcribe.BEAM_SIZE, max_depth: int = transcribe.MAX_DEPTH,
                           opts: model.OracleOptions = model.DEFAULT_OPTS, trace: Optional[dict] = None
                           ) -> Tuple[List[int], List[float], float]:
    """oracle.transcribe.mels_to_tokens with the log-prob of every returned id (f32 log_softmax values widened to f64, 0.0 for
    the prompt) and the carried score of the returned beam."""
    rec: dict = {}
    with _capture_best_beam(rec):
        ids = transcribe.mels_to_tokens(w, dims, sp, mels, beam_size, max_depth, opts=opts, trace=trace)
    assert [t for t, _ in rec["seq"]] == ids
    return ids, [lp for _, lp in rec["seq"]], rec["score"]


def greedy_loop_logprobs(w: dict, dims: model.WhisperDims, sp, mels: torch.Tensor, max_depth: Optional[int] = None,
                         opts: model.OracleOptions = model.DEFAULT_OPTS, trace: Optional[dict] = None
                         ) -> Tuple[List[int], List[float]]:
    """oracle_greedy_loop.mels_to_tokens_greedy_loop with, per id: 0.0 for the prompt, log_softmax of the step's raw
    logits at the arg-max id it appended, NaN for the EOT a rule appended."""
    mels = transcribe.pad_mel(mels, dims.n_audio_ctx)
    dec = model.CachedDecoder(w, dims, model.forward_encoder(w, dims, mels, opts), opts)
    last = {"logits": None}
    rows = []

    def logits_of(tokens):
        for t in tokens[dec.t:]:
            last["logits"] = dec.step(torch.tensor([t], dtype=torch.int64))[0]
        rows.append(model.log_softmax_last(last["logits"][None])[0])
        return last["logits"]

    tr = {} if trace is None else trace
    prompt = sp.prompt()
    ids = loop.greedy_loop(prompt, sp.eot, dims.n_text_ctx, logits_of, max_depth, tr)
    P = len(prompt)
    lps = [0.0 if i < P else float(rows[i - P][t]) if i - P < len(rows) else math.nan for i, t in enumerate(ids)]
    chose_eot = tr["stop"] == "eot" and len(rows) > 0 and int(torch.argmax(last["logits"])) == sp.eot
    if not chose_eot:
        lps[-1] = math.nan
    return ids, lps


def unmasked(sp: transcribe.SpecialTokens) -> transcribe.SpecialTokens:
    """The same ids with no special-token mask (is_special never holds): greedy_path_log_probs then scores the raw logits,
    as the greedy loop ranks them."""
    return dataclasses.replace(sp, first_special=sp.n_vocab)


def merge(windows: List[Tuple[List[int], List[float]]]) -> Tuple[List[int], List[float]]:
    """waveform_to_text's merge (transcribe.rs:42-71) of per-window (ids, log-probs): each log-prob follows its id."""
    ids: List[int] = []
    lps: List[float] = []
    for new_ids, new_lps in windows:
        assert len(new_ids) == len(new_lps)
        ov = transcribe.find_chunk_overlap(ids, list(new_ids), 40, 3)
        if ov is not None:
            ids, lps = ids[:ov[0]] + list(new_ids[ov[1]:]), lps[:ov[0]] + list(new_lps[ov[1]:])
        else:
            ids, lps = ids + list(new_ids), lps + list(new_lps)
    return ids, lps


def same(a, b) -> bool:
    """Equal float arrays, NaN equal to NaN."""
    return np.array_equal(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), equal_nan=True)
