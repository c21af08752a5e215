"""Cost of the previous-text prompt (Session.set_prev_prompt) in waveforms_to_tokens: R-mode windows, greedy depth 100,
fp32 K/V, on tiny.en 1 x 30 s, tiny.en 8 x 30 s and small.en 8 x 30 s.  The default (all windows of all waveforms in
batches of max_windows) and the rule (round i decodes window i of every waveform) run alternately in one process on one
session, warm-up first.  Prints per case and arm: audio-s/s (host clock around the call, which ends in a device
synchronise), the decode-phase ms of the last decoder call (the last round under the rule), and the rounds and mean rows
per decoder launch computed from the window counts (not counted), with the card and its power limit.

  python scripts/bench_prev_prompt.py [--calls 5] [--warmup 2]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import wb200  # noqa: E402,F401
from oracle import synth  # noqa: E402
from whisper_burn_b200 import model, transcribe  # noqa: E402

CASES = (("tiny.en", 1), ("tiny.en", 8), ("small.en", 8))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def run_case(name, n_chunks, calls, warmup):
    dims, w_np, _ = synth.make_weights(name, seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    waves = [synth.chunk_waveform(c) for c in range(n_chunks)]
    window_len = transcribe.window_samples(dims.n_audio_ctx)
    n_win = [len(transcribe.window_bounds(len(w), 16000, window_len)) for w in waves]
    max_windows = sum(n_win)
    sess = transcribe.Session(wh, max_windows=max_windows, max_beams=1, max_text_len=10 + 100 + 1)
    bitmap = sp.is_special_bitmap()
    arms = {"default": -1, "prev_prompt": sp.startofprev}
    t = {a: [] for a in arms}
    dec = {}
    for i in range(warmup + calls):
        for arm, sop in arms.items():
            sess.set_prev_prompt(sop)
            t0 = time.perf_counter()
            sess.waveforms_to_tokens(waves, sp, bitmap, beam_size=1, max_depth=100)
            dt = time.perf_counter() - t0
            if i >= warmup:
                t[arm].append(dt)
                dec[arm] = sess.last_timings_ms()["decode"]
    audio_s = sum(len(w) for w in waves) / 16000.0
    rounds = {"default": 1, "prev_prompt": max(n_win)}
    rows = {"default": max_windows / 1, "prev_prompt": max_windows / max(n_win)}
    out = []
    for arm in arms:
        out.append({"case": f"{name} {n_chunks}x30 s", "arm": arm, "audio_s_per_s": audio_s / float(np.median(t[arm])),
                    "call_ms": 1e3 * float(np.median(t[arm])), "decode_ms_last_call": dec[arm], "rounds": rounds[arm],
                    "rows_per_launch": rows[arm]})
    sess.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    gpu, power = card()
    for name, n in CASES:
        for r in run_case(name, n, a.calls, a.warmup):
            r.update(gpu=gpu, power_limit=power)
            print(json.dumps(r))


if __name__ == "__main__":
    main()
