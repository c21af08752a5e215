"""CPU tests of the greedy loop (WB_SEARCH_GREEDY_LOOP, src/transcribe.rs:314-380).

The oracle loop (tests/oracle_greedy_loop.py) is driven by table-defined logits through each of its stopping rules: the EOT
test with and without EOT as the arg-max, the repetition cut, the EOT test taking precedence over the cut at the same step,
and the context stop at n_text_ctx and at 4 + max_depth.  The rules the persistent decoders run (host/loop_rules.hpp, one
__host__ __device__ definition) are compiled for the host and compared with host/repeat.hpp and the oracle on the same
inputs."""
import ctypes as C
import math
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_greedy_loop as loop
from oracle import transcribe as o_tr

ROOT = Path(__file__).resolve().parent.parent
V, EOT = 32, 31
PROMPT = [27, 28, 29, 30]


def logits_fn(choose, eot_logit=-10.0, eot_at=None):
    """Logits of the position after `tokens`: 0 everywhere, 1 on choose(tokens), EOT at eot_logit (or eot_at(tokens))."""
    def f(tokens):
        row = torch.zeros(V, dtype=torch.float32)
        row[choose(tokens)] = 1.0
        row[EOT] = eot_at(tokens) if eot_at else eot_logit
        return row
    return f


def test_eot_stop_appends_eot_when_argmax_is_not_eot():
    # exp(0.4 - 1) = 0.55 > 0.5 at the first step: the arg-max 7 is kept, EOT follows
    tr = {}
    got = loop.greedy_loop(PROMPT, EOT, 448, logits_fn(lambda t: 7, eot_logit=0.4), trace=tr)
    assert got == PROMPT + [7, EOT] and tr["stop"] == "eot"
    assert tr["eot_gap"][0] == pytest.approx((0.4 - 1.0) - math.log(0.5), abs=1e-6)
    # exp(0.3 - 1) = 0.497: no stop
    got = loop.greedy_loop(PROMPT, EOT, 12, logits_fn(lambda t: len(t) % 20, eot_logit=0.3), trace=tr)
    assert got[-1] == EOT and len(got) == 13


def test_eot_stop_when_argmax_is_eot_appends_nothing():
    got = loop.greedy_loop(PROMPT, EOT, 448, logits_fn(lambda t: 3 if len(t) < 7 else EOT, eot_at=lambda t: 1.0 if len(t) >= 7 else -9.0))
    assert got == PROMPT + [3, 3, 3, EOT]


def test_repetition_cut_truncates_at_the_second_repeat():
    # always 7: after k sevens the all-7 windows at 4 .. 4 + k - 10 repeat the last; the 4th repeat appears at k = 13, the
    # first two are at 4 and 5, so the sequence is cut to 5 tokens and EOT appended
    tr = {}
    got = loop.greedy_loop(PROMPT, EOT, 448, logits_fn(lambda t: 7), trace=tr)
    assert got == PROMPT + [7, EOT] and tr["stop"] == "repeat"
    assert len(tr["eot_gap"]) == 13
    # a period-3 loop: windows repeating the last one start every 3 tokens
    cyc = [5, 6, 8]
    got = loop.greedy_loop(PROMPT, EOT, 448, logits_fn(lambda t: cyc[(len(t) - 4) % 3]))
    seq = PROMPT + [cyc[i % 3] for i in range(40)]
    for n in range(5, len(seq) + 1):
        rep = o_tr.find_repeated_tokens_index(seq[:n], 5, 4)
        if rep is not None:
            break
    assert got == seq[:rep[1]] + [EOT]


def test_eot_test_takes_precedence_over_the_cut():
    # the EOT test fires at the 13th step, the one at which the cut would: EOT is appended, nothing is cut
    got = loop.greedy_loop(PROMPT, EOT, 448, logits_fn(lambda t: 7, eot_at=lambda t: 0.5 if len(t) == 4 + 12 else -9.0))
    assert got == PROMPT + [7] * 13 + [EOT]


@pytest.mark.parametrize("n_text_ctx,max_depth,n_out", [(20, None, 21), (448, 6, 11), (20, 30, 21), (448, 0, 5)])
def test_context_stop(n_text_ctx, max_depth, n_out):
    tr = {}
    got = loop.greedy_loop(PROMPT, EOT, n_text_ctx, logits_fn(lambda t: len(t) % 27), max_depth=max_depth, trace=tr)
    assert len(got) == n_out and got[-1] == EOT and EOT not in got[:-1] and tr["stop"] == "context"
    assert got[4:-1] == [i % 27 for i in range(4, n_out - 1)]


# ---- host build of host/loop_rules.hpp ---------------------------------------------------------------------------------
SHIM = r"""
#include <cstdint>
#include "loop_rules.hpp"
#include "repeat.hpp"
extern "C" int cut_loop_rules(const int64_t* t, int n) { return wb::loop::repeat_cut_host(t, n); }
extern "C" int cut_repeat_hpp(const int64_t* t, int n) {
    int64_t first = 0, end = 0;
    const int r = wb::repeat::find_repeated_tokens_index(t, n, wb::loop::REPEAT_WINDOW, wb::loop::MIN_REPEATS, &first, &end);
    return r == 1 ? (int)end : (r == 0 ? -1 : -2);
}
extern "C" int eot_stop(float e, float t) { return wb::loop::eot_stop(e, t) ? 1 : 0; }
"""


@pytest.fixture(scope="module")
def rules(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    assert cxx, "a host C++ compiler is needed (the CUDA build uses it too)"
    d = tmp_path_factory.mktemp("loop_rules")
    (d / "shim.cpp").write_text(SHIM)
    so = d / "shim.so"
    subprocess.run([cxx, "-std=c++17", "-O2", "-shared", "-fPIC", "-I", str(ROOT / "whisper-burn_b200" / "host"),
                    str(d / "shim.cpp"), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    i64 = C.POINTER(C.c_int64)
    for name in ("cut_loop_rules", "cut_repeat_hpp"):
        getattr(lib, name).argtypes = [i64, C.c_int]
        getattr(lib, name).restype = C.c_int
    lib.eot_stop.argtypes = [C.c_float, C.c_float]
    lib.eot_stop.restype = C.c_int
    return lib


def test_host_build_of_the_repetition_cut_matches_repeat_hpp_and_oracle(rules):
    rng = np.random.default_rng(5)
    hits = 0
    for trial in range(3000):
        n = int(rng.integers(0, 120))
        alphabet = int(rng.integers(1, 4))
        if trial % 3 == 0:   # a loop with a period, entered after a random prefix
            per = int(rng.integers(1, 9))
            pre = int(rng.integers(0, 30))
            cyc = rng.integers(0, 6, per)
            t = np.concatenate([rng.integers(0, 50, pre), np.resize(cyc, max(n - pre, 0))]).astype(np.int64)[:n]
        else:
            t = rng.integers(0, alphabet + 1, n).astype(np.int64)
        t = np.ascontiguousarray(t)
        p = t.ctypes.data_as(C.POINTER(C.c_int64))
        got, want = rules.cut_loop_rules(p, len(t)), rules.cut_repeat_hpp(p, len(t))
        rep = o_tr.find_repeated_tokens_index(t.tolist(), 5, 4)
        assert got == want == (-1 if rep is None else rep[1]), (t.tolist(), got, want, rep)
        hits += got >= 0
    assert hits > 500
    # every 32-window boundary of the ballot rounds: the 4th repeat in round 0, 1, 2
    for n in range(10, 160):
        t = np.ascontiguousarray(np.full(n, 3, np.int64))
        t[:max(n - 14, 0)] = np.arange(100, 100 + max(n - 14, 0))
        p = t.ctypes.data_as(C.POINTER(C.c_int64))
        rep = o_tr.find_repeated_tokens_index(t.tolist(), 5, 4)
        assert rules.cut_loop_rules(p, n) == (-1 if rep is None else rep[1])


def test_host_build_of_the_eot_test_matches_the_oracle(rules):
    rng = np.random.default_rng(9)
    top = rng.normal(0, 8, 4000).astype(np.float32)
    gap = np.concatenate([rng.normal(math.log(0.5), 1e-6, 2000), rng.normal(0, 2, 2000)]).astype(np.float32)
    eot = (top + gap).astype(np.float32)
    for e, t in zip(eot.tolist(), top.tolist()):
        assert rules.eot_stop(e, t) == (1 if math.exp(float(np.float32(e)) - float(np.float32(t))) > 0.5 else 0)
    assert rules.eot_stop(1.0, 1.0) == 1
