"""The oracle's n-best lists, for the tests of wb_session_last_nbest (TEST INFRASTRUCTURE).  The reference's beam::beam_search
(src/beam.rs:9-37) ranks its final carried list with Iterator::max_by and drops all but the winner; this restates that list and
its ranking without changing the oracle:

  * beam_search_final: beam.rs:9-32, the carried list when the search stops (``beams`` at beam.rs:33), in carried order;
  * rank_final: beam.rs:33-36's max_by applied again to what remains after each pick: descending log_prob, exact ties ordered
    by the LATER carried node first, so element 0 is what beam_search returns;
  * mels_to_nbest: oracle.transcribe.mels_to_tokens (any prompt through SpecialTokens.prompt()) returning the ranked final
    list as (ids, float32 log-prob of each id (0 for the prompt), f64 cumulative score, finished) per hypothesis.
"""
from __future__ import annotations

import contextlib
from typing import List, Sequence

import numpy as np

from oracle import beam, model, transcribe


def beam_search_final(initial_beams, next_fn, is_finished, beam_size: int, max_depth: int, trace: list | None = None):
    """beam.rs:9-32, the loop of oracle.beam.beam_search."""
    beams = initial_beams
    for _ in range(max_depth):
        best = beam._max_by_last(beams)
        if best is not None and is_finished(best.seq):
            break
        beams = beam.beam_search_step(beams, next_fn, is_finished, beam_size)
        if trace is not None:
            trace.append([(list(b.seq), b.log_prob) for b in beams])
    return beams


def rank_final(beams: Sequence[beam.BeamNode]) -> List[beam.BeamNode]:
    """max_by (last maximum, beam.rs:33-36) applied repeatedly to what remains."""
    rest = list(beams)
    out = []
    while rest:
        best = None
        for i, b in enumerate(rest):
            if best is None or not (b.log_prob < rest[best].log_prob):
                best = i
        out.append(rest.pop(best))
    return out


@contextlib.contextmanager
def _capture_final(out: dict):
    """While active, oracle.beam.beam_search records its final carried list and is_finished rule."""
    search = beam.beam_search

    def recording(initial_beams, next_fn, is_finished, beam_size, max_depth, trace=None):
        final = beam_search_final(initial_beams, next_fn, is_finished, beam_size, max_depth, trace)
        out["final"], out["is_finished"] = final, is_finished
        best = beam._max_by_last(final)
        return list(best.seq) if best is not None else []

    beam.beam_search = recording
    try:
        yield
    finally:
        beam.beam_search = search


def mels_to_nbest(w: dict, dims: model.WhisperDims, sp: transcribe.SpecialTokens, mels, beam_size: int, max_depth: int,
                  opts: model.OracleOptions = model.DEFAULT_OPTS):
    """The ranked final list of oracle.transcribe.mels_to_tokens; element 0's ids are what mels_to_tokens returns."""
    rec: dict = {}
    with _capture_final(rec):
        ids = transcribe.mels_to_tokens(w, dims, sp, mels, beam_size, max_depth, opts=opts)
    ranked = [([t for t, _ in b.seq], np.asarray([lp for _, lp in b.seq], dtype=np.float32), float(b.log_prob),
               bool(rec["is_finished"](b.seq))) for b in rank_final(rec["final"])]
    assert ranked[0][0] == ids
    return ranked
