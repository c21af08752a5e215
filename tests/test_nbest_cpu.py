"""CPU tests of the n-best ranking (wb_session_last_nbest): the final carried list of the table-driven search (wb_beam_nbest_table),
stepped by the host window loop and the fixed-capacity step the on-device search runs (host/beam.hpp), ranked by
beamfx::rank_final, must be the oracle's list (tests/oracle_nbest.py) exactly: ids, order, finished flags and f64
scores.  Rank 0 is the sequence wb_beam_search_table returns, and exact ties put the later carried node first."""
import json
from pathlib import Path

import numpy as np
import pytest

import oracle_nbest as onb
import wb200  # noqa: F401
from oracle import beam as o_beam
from whisper_burn_b200 import beam, ffi

G = Path(__file__).resolve().parent / "golden"
N_CTX, V, EOT, FIRST = 37, 23, 22, 3


@pytest.fixture(scope="module", autouse=True)
def built():
    if not ffi.library_path().exists():
        import __graft_entry__ as ge
        ge.build()


def oracle_final(table, first, eot, beam_size, max_depth):
    n_ctx, n_vocab = table.shape

    def next_fn(beams):
        return [[(v, b.log_prob + float(table[(b.seq[-1] * 131 + len(b.seq)) % n_ctx, v])) for v in range(n_vocab)]
                for b in beams]

    return onb.beam_search_final([o_beam.BeamNode(seq=[first], log_prob=0.0)], next_fn, lambda s: s[-1] == eot, beam_size,
                                 max_depth)


def oracle_nbest(table, first, eot, beam_size, max_depth):
    return [(list(b.seq), b.log_prob, b.seq[-1] == eot) for b in onb.rank_final(oracle_final(table, first, eot, beam_size, max_depth))]


def check(table, first, eot, beam_size, max_depth):
    want = oracle_nbest(table, first, eot, beam_size, max_depth)
    got = beam.nbest_table(table, first, eot, beam_size, max_depth)
    assert got == want, (beam_size, max_depth)   # ids, order, finished, f64 scores bit-equal
    assert got[0][0] == beam.beam_search_table(table, first, eot, beam_size, max_depth)
    return want


def make_table(rng, quant, eot_boost):
    table = np.log(rng.dirichlet(np.ones(V) * 0.7, size=N_CTX))
    if quant:
        table = np.round(table, quant)          # exact score ties
    table[:, EOT] += eot_boost
    return table


@pytest.mark.parametrize("beam_size", [1, 2, 3, 4, 5, 6, 7])
@pytest.mark.parametrize("quant", [0, 1, 2])
@pytest.mark.parametrize("eot_boost", [-30.0, 0.0, 3.0])
def test_nbest_table_matches_oracle(beam_size, quant, eot_boost):
    rng = np.random.default_rng(4000 + 97 * beam_size + 13 * quant + int(eot_boost))
    for trial in range(3):
        table = make_table(rng, quant, eot_boost)
        for max_depth in (0, 1, 30):
            want = check(table, FIRST, EOT, beam_size, max_depth)
            assert len(want) <= 2 * beam_size
            if max_depth == 0:
                assert want == [([FIRST], 0.0, False)]
            if beam_size == 1:
                assert len(want) == 1


def test_nbest_table_holds_live_and_finished():
    """EOT reached by some beams but not by the best one at max_depth: the list carries live ones first, then finished ones
    (beam.rs:71-78), and the ranking interleaves them by score"""
    rng = np.random.default_rng(3)
    seen = set()
    for boost in (0.5, 1.0, 1.5, 2.0):
        for _ in range(6):
            table = make_table(rng, 2, boost)
            for b in (3, 5, 7):
                want = check(table, FIRST, EOT, b, 8)
                fin = [f for _, _, f in want]
                if any(fin) and not all(fin):
                    seen.add("mixed")
                if fin[0]:
                    seen.add("finished best")
    assert seen == {"mixed", "finished best"}


@pytest.mark.parametrize("case", range(len(json.loads((G / "beam_ties.json").read_text()))))
def test_nbest_table_beam_ties_cases(case):
    """every get_top_elements tie case of beam_ties.json as a one-context table: each step sees the same scores"""
    c = json.loads((G / "beam_ties.json").read_text())[case]
    scores = np.asarray(c["scores"], dtype=np.float64)
    if scores.size == 0:
        scores = np.zeros(1)
    table = scores[None, :]
    b = max(1, min(c["num"], 7))
    for eot in sorted({0, int(np.argmax(scores)), len(scores) - 1}):
        for max_depth in (1, 3, 6):
            check(table, FIRST % len(scores), eot, b, max_depth)


def test_nbest_exact_ties_put_the_later_node_first():
    """every continuation scores 0: the carried nodes all tie, and the ranking is the carried order reversed (max_by keeps the
    LAST maximum, beamfx::rank_final applies it again to what remains)"""
    table = np.zeros((1, 8))   # eot 7 never wins a tie: get_top_elements keeps the earlier of equal elements
    for b in (2, 3, 5, 7):
        final = oracle_final(table, 1, 7, b, 3)
        assert len(final) == b and len({f.log_prob for f in final}) == 1
        want = [(list(f.seq), 0.0, False) for f in reversed(final)]
        assert beam.nbest_table(table, 1, 7, b, 3) == want
        assert beam.beam_search_table(table, 1, 7, b, 3) == list(final[-1].seq)


def test_rank_final_restatement():
    """the oracle's rank_final is max_by (last maximum) applied repeatedly: descending score, later node first on ties"""
    nodes = [o_beam.BeamNode([i], s) for i, s in enumerate([-1.0, -0.5, -1.0, -0.5, -2.0, -0.5])]
    assert [n.seq[0] for n in onb.rank_final(nodes)] == [5, 3, 1, 2, 0, 4]


def test_nbest_table_rejects_bad_arguments():
    """beam_size must be 1 .. 7 (beamfx::MAX_BEAM, the sessions' limit)"""
    table = np.zeros((N_CTX, V))
    for b in (0, 8, 11):
        with pytest.raises(ffi.WbError):
            beam.nbest_table(table, FIRST, EOT, b, 3)
        with pytest.raises(ffi.WbError):
            beam.beam_search_table(table, FIRST, EOT, b, 3)
