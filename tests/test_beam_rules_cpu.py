"""CPU tests of the library's beam search (host/beam.hpp): the fixed-capacity step that the on-device search runs, driven
by the host window loop over a table-defined `next`, must pick the same sequences as the oracle, with exact score ties common,
EOT reached early, late or never, and max_depth 0, 1 and 30."""
import numpy as np
import pytest

import wb200  # noqa: F401
from oracle import beam as o_beam
from whisper_burn_b200 import beam, ffi

N_CTX, V, EOT, FIRST = 37, 23, 22, 3


@pytest.fixture(scope="module", autouse=True)
def built():
    if not ffi.library_path().exists():
        import __graft_entry__ as ge
        ge.build()


def oracle_search(table, beam_size, max_depth):
    def next_fn(beams):
        return [[(v, b.log_prob + float(table[(b.seq[-1] * 131 + len(b.seq)) % N_CTX, v])) for v in range(V)] for b in beams]

    return o_beam.beam_search([o_beam.BeamNode(seq=[FIRST], log_prob=0.0)], next_fn, lambda s: s[-1] == EOT, beam_size, max_depth)


def make_table(rng, quant, eot_boost):
    table = np.log(rng.dirichlet(np.ones(V) * 0.7, size=N_CTX))
    if quant:
        table = np.round(table, quant)          # exact score ties
    table[:, EOT] += eot_boost
    return table


# eot_boost: -30 never finishes, 0 finishes late or never, 3 finishes within a few steps
@pytest.mark.parametrize("beam_size", [1, 2, 3, 4, 5, 6, 7])
@pytest.mark.parametrize("quant", [0, 1, 2])
@pytest.mark.parametrize("eot_boost", [-30.0, 0.0, 3.0])
def test_fixed_step_matches_host_search_and_oracle(beam_size, quant, eot_boost):
    rng = np.random.default_rng(1000 + 97 * beam_size + 13 * quant + int(eot_boost))
    for trial in range(3):
        table = make_table(rng, quant, eot_boost)
        for max_depth in (0, 1, 30):
            want = oracle_search(table, beam_size, max_depth)
            got = beam.beam_search_table(table, FIRST, EOT, beam_size, max_depth)
            assert got == want, (trial, max_depth)
            if eot_boost == -30.0:
                assert EOT not in got and len(got) == 1 + max_depth


def test_fixed_step_eot_early_and_late():
    """A table where EOT wins at the first step, and one where it only wins after many steps: the search stops where the
    oracle's does and keeps carrying the finished beams."""
    rng = np.random.default_rng(7)
    seen = set()
    for boost in (6.0, 1.0, 0.5, 0.2):
        for _ in range(4):
            table = make_table(rng, 2, boost)
            for b in (2, 5, 7):
                want = oracle_search(table, b, 30)
                assert beam.beam_search_table(table, FIRST, EOT, b, 30) == want
                if want[-1] == EOT:
                    seen.add("early" if len(want) <= 4 else "late")
    assert seen == {"early", "late"}


def test_fixed_step_rejects_bad_arguments():
    table = np.zeros((N_CTX, V))
    for b in (0, 8):
        with pytest.raises(ffi.WbError):
            beam.beam_search_table(table, FIRST, EOT, b, 3)
