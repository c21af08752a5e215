"""Generates tests/golden/tokens_beam.json from the CPU oracle: beam-search ids for the on-device beam search tests
(tests/test_device_beam_gpu.py), so the GPU run does not spend minutes re-deriving them on the CPU.

  test_a:  oracle ids of every window of POOL (windows of T = 750, 6, 314, 65, 750, 314 encoder positions, slices of
           synth.chunk_waveform(0)) for beam sizes 2..7 at depth 12, fp32 and fp16 K/V (the windows a <= 24-row batch of
           that beam size uses; one more at beam 5);
  tiny_en: the three reference windows of chunk 0 at beam 5, depth 30, fp32 and fp16 K/V;
  eot:     window 1 of the eot_case of tokens_test_a.json (EOT = a token the search emits, window 0 stops early) at beam 5.
Run from the repo root:  python tests/golden/make_golden_beam.py
"""
import json
import sys
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
from oracle import audio, model, synth, transcribe  # noqa: E402

OUT = Path(__file__).resolve().parent
POOL = [(0, 238559), (50000, 400), (120000, 98882), (7000, 19040), (241441, 238559), (381118, 98882)]   # (offset, samples)
DEPTH_A, DEPTH_TINY = 12, 30


def run(job):
    name, kv, b, depth, lo, hi, eot = job
    torch.set_num_threads(1)
    dims, _, w = synth.make_weights(name, seed=0)
    sp = synth.special_tokens(dims)
    if eot is not None:
        sp = transcribe.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, eot, sp.first_special, sp.n_vocab)
    wave = synth.chunk_waveform(0)[lo:hi]
    mel = audio.prep_audio(torch.from_numpy(wave)[None])
    return transcribe.mels_to_tokens(w, dims, sp, mel, beam_size=b, max_depth=depth, opts=model.OracleOptions(kv_dtype=kv))


def main():
    te = json.loads((OUT / "tokens_tiny_en.json").read_text())
    ta = json.loads((OUT / "tokens_test_a.json").read_text())
    jobs, keys = [], []
    for kv in ("f32", "f16"):
        for b in range(2, 8):
            n_win = min(len(POOL), 24 // b + (1 if b == 5 else 0))   # beam 5: also the 25-row batch the device search leaves to the host
            for i, (off, n) in enumerate(POOL[:n_win]):
                jobs.append(("test-a", kv, b, DEPTH_A, off, off + n, None))
                keys.append(("test_a", kv, str(b), i))
        for i, (s, e) in enumerate(te["bounds"]):
            jobs.append(("tiny.en", kv, 5, DEPTH_TINY, s, e, None))
            keys.append(("tiny_en", kv, "5", i))
    eot = ta["eot_case_beam5"]["eot"]
    jobs.append(("test-a", "f32", 5, 30, 0, 98882, eot))
    keys.append(("eot", "f32", "5", 1))
    with ProcessPoolExecutor() as ex:
        res = list(ex.map(run, jobs))
    out = {"pool": POOL, "depth_test_a": DEPTH_A, "depth_tiny_en": DEPTH_TINY, "eot": eot, "test_a": {}, "tiny_en": {}, "eot_window1": None}
    for (kind, kv, b, i), toks in zip(keys, res):
        if kind == "eot":
            out["eot_window1"] = toks
            continue
        lst = out[kind].setdefault(kv, {}).setdefault(b, [])
        assert len(lst) == i
        lst.append(toks)
    (OUT / "tokens_beam.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
