"""Generates tests/golden/nbest_beam.json from the CPU oracle: each window's n-best list (the beam search's final carried list
ranked by tests/oracle_nbest.py) for the tests of wb_session_last_nbest (tests/test_nbest_gpu.py), so the GPU run does not
re-derive them on the CPU.

  test_a:  the POOL windows of make_golden_beam.py at beam sizes 2..7, depth 12, fp32 and fp16 K/V (the same jobs);
  tiny_en: the three reference windows of chunk 0 at beam 5, depth 30, fp32 and fp16 K/V;
  eot_case: the two windows of make_golden_beam.py's eot case at beam 5, depth 30, fp32 (EOT = a token the search emits:
            both searches stop early on a finished best, several steps apart, with live hypotheses carried behind it;
            the test_a lists at depth 12 are the depth-limit case: live hypotheses only);
  prev:    four POOL windows of test-a with previous-text prompts of 0, 2, 5 and 1 ids (one launch, prompts of 4, 7, 10 and
           6 ids) at beam 5, depth 12, fp32.
Every hypothesis has its ids, f32 log-probs, f64 score and finished flag; every list also has `gaps`, the score differences of
adjacent ranks (a swap of two ranks on the GPU is only acceptable where their gap is within rounding).
Run from the repo root:  python tests/golden/make_golden_nbest.py
"""
import json
import sys
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))
import make_golden_beam as mgb  # noqa: E402
import oracle_nbest as onb  # noqa: E402
import oracle_prev_prompt as opp  # noqa: E402
from oracle import audio, model, synth, transcribe  # noqa: E402

OUT = HERE / "nbest_beam.json"
PREV_LENS = (0, 2, 5, 1)
PREV_SEED = 5


def prev_ids(sp):
    rng = np.random.default_rng(PREV_SEED)
    return [[int(t) for t in rng.integers(0, sp.first_special, size=k)] for k in PREV_LENS]


def run(job):
    name, kv, b, depth, lo, hi, eot, prev = job
    torch.set_num_threads(1)
    dims, _, w = synth.make_weights(name, seed=0)
    sp = synth.special_tokens(dims)
    if eot is not None:
        sp = transcribe.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, eot, sp.first_special, sp.n_vocab)
    if prev is not None:
        sp = opp.with_prompt(sp, opp.build_prompt(synth.special_tokens(dims), prev))
    wave = synth.chunk_waveform(0)[lo:hi]
    mel = audio.prep_audio(torch.from_numpy(wave)[None])
    hyps = onb.mels_to_nbest(w, dims, sp, mel, b, depth, opts=model.OracleOptions(kv_dtype=kv))
    return {"hyps": [{"ids": ids, "lps": [float(x) for x in lps], "score": score, "finished": fin} for ids, lps, score, fin in hyps],
            "gaps": [hyps[i][2] - hyps[i + 1][2] for i in range(len(hyps) - 1)]}


def main():
    te = json.loads((HERE / "tokens_tiny_en.json").read_text())
    ta = json.loads((HERE / "tokens_test_a.json").read_text())
    jobs, keys = [], []
    for kv in ("f32", "f16"):   # make_golden_beam.py's job list
        for b in range(2, 8):
            n_win = min(len(mgb.POOL), 24 // b + (1 if b == 5 else 0))
            for i, (off, n) in enumerate(mgb.POOL[:n_win]):
                jobs.append(("test-a", kv, b, mgb.DEPTH_A, off, off + n, None, None))
                keys.append(("test_a", kv, str(b)))
        for s, e in te["bounds"]:
            jobs.append(("tiny.en", kv, 5, mgb.DEPTH_TINY, s, e, None, None))
            keys.append(("tiny_en", kv, "5"))
    eot = ta["eot_case_beam5"]["eot"]
    for hi in (238559, 98882):
        jobs.append(("test-a", "f32", 5, 30, 0, hi, eot, None))
        keys.append(("eot_case", "f32", "5"))
    sp_a = synth.special_tokens(synth.make_weights("test-a", seed=0)[0])
    prevs = prev_ids(sp_a)
    for (off, n), prev in zip(mgb.POOL, prevs):
        jobs.append(("test-a", "f32", 5, mgb.DEPTH_A, off, off + n, None, prev))
        keys.append(("prev", "f32", "5"))
    with ProcessPoolExecutor() as ex:
        res = list(ex.map(run, jobs))
    out = {"pool": mgb.POOL, "depth_test_a": mgb.DEPTH_A, "depth_tiny_en": mgb.DEPTH_TINY, "eot": eot, "depth_eot": 30,
           "prev_lens": list(PREV_LENS), "prev_ids": prevs, "test_a": {}, "tiny_en": {}, "eot_case": {}, "prev": {}}
    for (kind, kv, b), r in zip(keys, res):
        out[kind].setdefault(kv, {}).setdefault(b, []).append(r)
    OUT.write_text(json.dumps(out))


if __name__ == "__main__":
    main()
