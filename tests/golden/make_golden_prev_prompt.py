"""Golden token fixture of the previous-text prompt (transcribe.rs:43-54, 195-203 without the shadowing at :201), from the
CPU oracle restatement tests/oracle_prev_prompt.py.

  tiny.en        seed 0, 1 120 000 samples (70 s, synth.waveform seed 2024), R-mode: 6 windows decoded in order under the
                 waveform rule; greedy depth 100 with fp32 and fp16 K/V, and beam 5 depth 30 (fp32)
  small.en       seed 0, chunk 0 (30 s, 3 R-mode windows) under the waveform rule; greedy depth 100 with fp32 and fp16 K/V,
                 and beam 5 depth 20 (fp32; the host search on decoder5)
  tiny.en-native seed 0, the same 70 s waveform in N-mode windows (3 windows) under the waveform rule, greedy depth 100, fp32
  ragged         tiny.en seed 0, the 3 R-mode windows of chunk 1 and the first window of chunk 2 with explicit previous ids
                 of 0, 1, 5 and 12 non-special ids, greedy depth 100, fp32

Every window record has its prompt, its ids, the log-prob of each generated id (greedy) and the top-1/top-2 log-prob margin of
each step (greedy) or the smallest margin met (beam).  Waveform-rule records also have the merged ids.
Run from the repo root:  python tests/golden/make_golden_prev_prompt.py
"""
import dataclasses
import json
import sys
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import oracle_prev_prompt as opp  # noqa: E402
from oracle import audio, model, synth, transcribe  # noqa: E402

OUT = Path(__file__).resolve().parent / "tokens_prev_prompt.json"
LONG_SAMPLES, LONG_SEED = 1120000, 2024
RAGGED_PREV_LENS = (0, 1, 5, 12)


def long_wave():
    return synth.waveform(LONG_SAMPLES, seed=LONG_SEED, kind="mix")


def margins(trace):
    g = []
    for st in trace["log_probs"]:
        for row in st:
            if row is not None:
                s = np.partition(row, row.shape[0] - 2)[-2:]
                g.append(float(abs(s[1] - s[0])))
    return g


def decode_window(w, dims, sp, wave, prompt, beam, depth, kv):
    mel = audio.prep_audio(torch.from_numpy(np.ascontiguousarray(wave))[None])
    tr = {}
    toks = opp.mels_to_tokens(w, dims, sp, mel, prompt, beam, depth, opts=model.OracleOptions(kv_dtype=kv), trace=tr)
    rec = {"prompt": list(prompt), "tokens": toks, "min_margin": min(margins(tr), default=1.0)}
    if beam == 1:
        rec["margins"] = [round(g, 7) for g in margins(tr)]
        rec["lps"] = [float(st[0][toks[len(prompt) + s]]) for s, st in enumerate(tr["log_probs"]) if len(prompt) + s < len(toks)]
    return rec


def rule_case(name, wave_kind, native, beam, depth, kv):
    """The waveform rule over one waveform: windows in order, each prompted from the merged ids before it."""
    torch.set_num_threads(1)
    dims, _, w = synth.make_weights(name, seed=0)
    sp = synth.special_tokens(dims)
    wave = long_wave() if wave_kind == "long" else synth.chunk_waveform(0)
    odims = dataclasses.replace(dims, n_audio_ctx=2 * dims.n_audio_ctx) if native else dims
    window_len = audio.max_waveform_samples(odims.n_audio_ctx - transcribe.PADDING)
    merged, windows = [], []
    for (s, e) in transcribe.window_bounds(len(wave), 16000, window_len):
        prompt = opp.build_prompt(sp, opp.prev_nonspecial(merged, sp.is_special))
        rec = decode_window(w, odims, sp, wave[s:e], prompt, beam, depth, kv)
        rec["bounds"] = [s, e]
        windows.append(rec)
        ov = transcribe.find_chunk_overlap(merged, rec["tokens"], 40, 3)
        merged = merged[:ov[0]] + rec["tokens"][ov[1]:] if ov is not None else merged + rec["tokens"]
    return {"model": name, "waveform": wave_kind, "native": native, "beam": beam, "depth": depth, "kv": kv,
            "windows": windows, "merged": merged}


def ragged_case():
    torch.set_num_threads(1)
    dims, _, w = synth.make_weights("tiny.en", seed=0)
    sp = synth.special_tokens(dims)
    window_len = audio.max_waveform_samples(dims.n_audio_ctx - transcribe.PADDING)
    waves = [(1, b) for b in transcribe.window_bounds(480000, 16000, window_len)]
    waves.append((2, transcribe.window_bounds(480000, 16000, window_len)[0]))
    rng = np.random.default_rng(7)
    windows = []
    for (c, (s, e)), k in zip(waves, RAGGED_PREV_LENS):
        prev = [int(t) for t in rng.integers(0, sp.first_special, size=k)]
        rec = decode_window(w, dims, sp, synth.chunk_waveform(c)[s:e], opp.build_prompt(sp, prev), 1, 100, "f32")
        rec.update(chunk=c, bounds=[s, e], prev=prev)
        windows.append(rec)
    return {"model": "tiny.en", "beam": 1, "depth": 100, "kv": "f32", "windows": windows}


CASES = {
    "tiny.en-f32": (rule_case, ("tiny.en", "long", False, 1, 100, "f32")),
    "tiny.en-f16": (rule_case, ("tiny.en", "long", False, 1, 100, "f16")),
    "tiny.en-beam": (rule_case, ("tiny.en", "long", False, 5, 30, "f32")),
    "small.en-f32": (rule_case, ("small.en", "chunk0", False, 1, 100, "f32")),
    "small.en-f16": (rule_case, ("small.en", "chunk0", False, 1, 100, "f16")),
    "small.en-beam": (rule_case, ("small.en", "chunk0", False, 5, 20, "f32")),
    "tiny.en-native": (rule_case, ("tiny.en", "long", True, 1, 100, "f32")),
    "ragged": (ragged_case, ()),
}


def main():
    t0 = time.time()
    with ProcessPoolExecutor(len(CASES)) as ex:
        futs = {k: ex.submit(f, *a) for k, (f, a) in CASES.items()}
        out = {k: f.result() for k, f in futs.items()}
    out["generation_s"] = round(time.time() - t0, 1)
    OUT.write_text(json.dumps(out))
    for k, v in out.items():
        if isinstance(v, dict):
            print(k, [len(r["tokens"]) for r in v["windows"]], min(r["min_margin"] for r in v["windows"]))
    print(f"{time.time() - t0:.0f} s")


if __name__ == "__main__":
    main()
