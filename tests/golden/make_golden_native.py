"""Golden token fixtures of native windowing (T up to 1500 encoder positions per window), from the CPU oracle.

Native windowing changes one rule of the reference's path: a window gives the encoder up to 2 * n_audio_ctx mel frames
instead of n_audio_ctx (transcribe.rs:32-34, 161-177 with that limit).  The oracle reads n_audio_ctx only as that frame
limit (pad_mel, forward_encoder's assert, the window length of waveform_to_tokens), so its native mode is the oracle run on
dims with n_audio_ctx doubled (native_dims); weights, positional embedding rows 0..T-1 and every decoder rule are unchanged.

  tiny.en        seed 0, greedy, depth 100, fp32 and fp16 K/V: one batch of 4 windows, T = 1500, 1500, 1005 (a ragged window
                 past the reference's 750) and 205; per-step top-1/top-2 margins and top-5 (id, log-prob)
  tiny.en-beam   seed 0, beam 5, depth 30, fp32 and fp16 K/V: 2 windows, T = 1500 and 1005 (decoder6's device beam search)
  small.en       seed 0, greedy, depth 100, fp32 and fp16 K/V: 2 windows at T = 1500; per-step margins and top-5
  small.en-beam  seed 0, beam 5, depth 20, fp32 K/V: 1 window at T = 1500 (the host search on decoder5)
  tiny.en-long   seed 0, waveform_to_tokens of 1 120 000 samples (70 s: chunks 0, 1 and the first 10 s of chunk 2), greedy,
                 depth 100, fp32 K/V: 3 native windows [0, 478559), [430559, 909118), [861118, 1120000) and the overlap merge

Every record has the smallest top-1/top-2 log-prob margin met on its decoded path.
Run from the repo root:  python tests/golden/make_golden_native.py
It takes about 35 s on 8 CPU cores (cases run side by side, one torch thread each; the synthetic models are cheap).
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
from oracle import audio, model, synth, transcribe  # noqa: E402

OUT = Path(__file__).resolve().parent / "tokens_native.json"

# (chunk id, samples) of each window: 480 000 samples -> F = 3000, keep 2990, Tm = 3000, T = 1500;
# 320 000 -> F = 2000, Tm = 2010, T = 1005; 64 000 -> F = 400, Tm = 410, T = 205
TINY_WINDOWS = [(0, 480000), (1, 480000), (2, 320000), (3, 64000)]
TINY_BEAM_WINDOWS = [(4, 480000), (5, 320000)]
SMALL_WINDOWS = [(0, 480000), (1, 480000)]
SMALL_BEAM_WINDOWS = [(2, 480000)]
LONG_SAMPLES = 1120000


def native_dims(dims):
    """dims of the oracle's native mode: the encoder frame limit n_audio_ctx doubled."""
    return dataclasses.replace(dims, n_audio_ctx=2 * dims.n_audio_ctx)


def margins(trace):
    g = []
    for st in trace["log_probs"]:
        for row in st:
            if row is not None:
                s = np.partition(row, row.shape[0] - 2)[-2:]
                g.append(float(abs(s[1] - s[0])))
    return g


def window_wave(chunk_id, n):
    return synth.chunk_waveform(chunk_id)[:n]


def decode(name, window, beam, depth, kv):
    """One window through the oracle's native mels_to_tokens; greedy records per-step margins and top-5."""
    torch.set_num_threads(1)
    dims, _, w = synth.make_weights(name, seed=0)
    sp = synth.special_tokens(dims)
    wave = window_wave(*window)
    mel = audio.prep_audio(torch.from_numpy(np.ascontiguousarray(wave))[None])
    tr = {}
    toks = transcribe.mels_to_tokens(w, native_dims(dims), sp, mel, beam_size=beam, max_depth=depth,
                                     opts=model.OracleOptions(kv_dtype=kv), trace=tr)
    rec = {"window": list(window), "T": int(tr["encoder_output"].shape[1]), "tokens": toks, "min_margin": min(margins(tr))}
    if beam == 1:
        rec["margins"] = [round(g, 7) for g in margins(tr)]
        top = []
        for st in tr["log_probs"]:
            lp = st[0]
            order = np.lexsort((np.arange(lp.shape[0]), -lp))[:5]
            top.append([[int(i) for i in order], [float(lp[i]) for i in order]])
        rec["top5"] = top
    return rec


def long_form():
    torch.set_num_threads(1)
    dims, _, w = synth.make_weights("tiny.en", seed=0)
    sp = synth.special_tokens(dims)
    wave = np.concatenate([synth.chunk_waveform(0), synth.chunk_waveform(1), synth.chunk_waveform(2)])[:LONG_SAMPLES]
    nd = native_dims(dims)
    bounds = transcribe.window_bounds(len(wave), 16000, audio.max_waveform_samples(nd.n_audio_ctx - transcribe.PADDING))
    per = []
    toks = transcribe.waveform_to_tokens(w, nd, sp, wave, beam_size=1, max_depth=100, per_window=per)
    return {"samples": LONG_SAMPLES, "chunks": [0, 1, 2], "beam": 1, "depth": 100, "kv": "f32", "bounds": bounds,
            "per_window": per, "tokens": toks}


def main():
    t0 = time.time()
    jobs = {}
    with ProcessPoolExecutor(8) as ex:
        for kv in ("f32", "f16"):
            for i, win in enumerate(SMALL_WINDOWS):
                jobs[("small.en", kv, i)] = ex.submit(decode, "small.en", win, 1, 100, kv)
        jobs[("small.en-beam", "f32", 0)] = ex.submit(decode, "small.en", SMALL_BEAM_WINDOWS[0], 5, 20, "f32")
        for kv in ("f32", "f16"):
            for i, win in enumerate(TINY_WINDOWS):
                jobs[("tiny.en", kv, i)] = ex.submit(decode, "tiny.en", win, 1, 100, kv)
            for i, win in enumerate(TINY_BEAM_WINDOWS):
                jobs[("tiny.en-beam", kv, i)] = ex.submit(decode, "tiny.en", win, 5, 30, kv)
        long_job = ex.submit(long_form)
        data = {
            "tiny.en": {"model": "tiny.en", "seed": 0, "beam": 1, "depth": 100, "windows": TINY_WINDOWS},
            "tiny.en-beam": {"model": "tiny.en", "seed": 0, "beam": 5, "depth": 30, "windows": TINY_BEAM_WINDOWS},
            "small.en": {"model": "small.en", "seed": 0, "beam": 1, "depth": 100, "windows": SMALL_WINDOWS},
            "small.en-beam": {"model": "small.en", "seed": 0, "beam": 5, "depth": 20, "windows": SMALL_BEAM_WINDOWS},
        }
        for (case, kv, i), fut in sorted(jobs.items()):
            data[case].setdefault(kv, []).append(fut.result())
        for case in data.values():
            for kv in ("f32", "f16"):
                if kv in case:
                    case[f"min_margin_{kv}"] = min(r["min_margin"] for r in case[kv])
        data["tiny.en-long"] = long_job.result()
    OUT.write_text(json.dumps(data))
    print("written in", round(time.time() - t0), "s", flush=True)


if __name__ == "__main__":
    main()
