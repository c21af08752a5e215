"""Mirror of the reference's ``beam`` module (src/beam.rs): the search itself runs in the library's
C++ code (host/beam.hpp); this exposes its selection primitive and a table-driven search for tests."""
from __future__ import annotations

import numpy as np

from . import ffi


def get_top_elements(scores, num: int) -> list[int]:
    """beam::get_top_elements (beam.rs:81-110) over f64 scores: kept indices, ascending score."""
    s = np.ascontiguousarray(scores, dtype=np.float64)
    out = np.empty(max(num, 1), dtype=np.int64)
    import ctypes as C
    n = ffi.lib().wb_beam_get_top_elements(s.ctypes.data_as(C.POINTER(C.c_double)), s.shape[0], num, ffi.i64ptr(out))
    if n < 0:
        raise ffi.WbError(ffi.WB_ERR_INVALID_ARG, "get_top_elements: bad arguments")
    return [int(v) for v in out[:n]]


def beam_search_table(table, first_token: int, eot: int, beam_size: int, max_depth: int, fixed: bool = False) -> list[int]:
    """beam::beam_search (beam.rs:9-37) in the library's C++ code (host/beam.hpp) over a table-driven `next`:
    log-prob of token v after a beam ending in t with length n = table[(t * 131 + n) % n_ctx][v].  Each live beam
    contributes its beam_size best table entries, as the device contributes its top-k; beam_size 1 .. 7.
    fixed: kept for existing callers.  The search has one stepping, the fixed-capacity step the device runs, so both
    values give the same result."""
    import ctypes as C
    t = np.ascontiguousarray(table, dtype=np.float64)
    out = np.zeros(max_depth + 2, dtype=np.int64)
    n = ffi.lib().wb_beam_search_table(t.ctypes.data_as(C.POINTER(C.c_double)), t.shape[0], t.shape[1], first_token, eot,
                                       beam_size, max_depth, ffi.i64ptr(out), out.shape[0])
    if n < 0:
        raise ffi.WbError(ffi.WB_ERR_INVALID_ARG, "beam_search_table: bad arguments")
    return [int(v) for v in out[:n]]


def nbest_table(table, first_token: int, eot: int, beam_size: int, max_depth: int, fixed: bool = False):
    """The ranked final carried list of beam_search_table's search (wb_beam_nbest_table): (ids, f64 score, finished) per
    hypothesis, best first; element 0's ids are what beam_search_table returns.  fixed: as in beam_search_table."""
    import ctypes as C
    t = np.ascontiguousarray(table, dtype=np.float64)
    max_hyps, cap = 2 * max(beam_size, 1), max_depth + 1
    ids = np.zeros((max_hyps, cap), dtype=np.int64)
    lens = np.zeros(max_hyps, dtype=np.int64)
    scores = np.zeros(max_hyps, dtype=np.float64)
    fin = np.zeros(max_hyps, dtype=np.int32)
    n = ffi.lib().wb_beam_nbest_table(t.ctypes.data_as(C.POINTER(C.c_double)), t.shape[0], t.shape[1], first_token, eot,
                                      beam_size, max_depth, max_hyps, cap, ffi.i64ptr(ids), ffi.i64ptr(lens),
                                      scores.ctypes.data_as(C.POINTER(C.c_double)), ffi.i32ptr(fin))
    if n < 0:
        raise ffi.WbError(ffi.WB_ERR_INVALID_ARG, "nbest_table: bad arguments")
    return [([int(v) for v in ids[r, :lens[r]]], float(scores[r]), bool(fin[r])) for r in range(n)]
