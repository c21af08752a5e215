"""Cost of reading each window's n-best list (Session.last_nbest, wb_session_last_nbest) after transcribe_windows at beam 5,
depth 100, fp32 K/V: tiny.en 1 x 30 s (3 R-mode windows, the on-device search in one decoder6 launch) and small.en 8 x 30 s
(24 windows, the host search).  Both arms run the same decode, which always keeps the final carried lists (on the device
search, one device-to-host copy of them in the stream sync that ends the launch); the "nbest" arm then reads every window's
list through the C ABI.  The arms alternate call by call on one session, warm-up first.  Prints per case and arm: the median
call time (host clock around work that ends in a device synchronise), audio-s/s, the decode-phase ms of the last call, the
decoder the search ran on, and the card with its power limit.

  python scripts/bench_nbest.py [--calls 7] [--warmup 2]"""
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

CASES = (("tiny.en", 1), ("small.en", 8))
BEAM, DEPTH = 5, 100


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def run_case(name, n_chunks, calls, warmup):
    dims, w_np, _ = synth.make_weights(name, seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    window_len = transcribe.window_samples(dims.n_audio_ctx)
    waves = []
    for c in range(n_chunks):
        chunk = synth.chunk_waveform(c)
        waves += [chunk[s:e] for s, e in transcribe.window_bounds(len(chunk), 16000, window_len)]
    sess = transcribe.Session(wh, max_windows=len(waves), max_beams=BEAM, max_text_len=4 + DEPTH + 1)
    bitmap = sp.is_special_bitmap()
    t = {"row": [], "nbest": []}
    dec, hyps = {}, 0
    for i in range(warmup + calls):
        for arm in t:
            t0 = time.perf_counter()
            sess.transcribe_windows(waves, sp, bitmap, beam_size=BEAM, max_depth=DEPTH)
            if arm == "nbest":
                hyps = sum(len(sess.last_nbest(w)) for w in range(len(waves)))
            dt = time.perf_counter() - t0
            if i >= warmup:
                t[arm].append(dt)
                dec[arm] = sess.last_timings_ms()["decode"]
    audio_s = sum(len(w) for w in waves) / 16000.0
    out = []
    for arm in t:
        out.append({"case": f"{name} {n_chunks}x30 s", "arm": arm, "windows": len(waves), "decoder": sess.last_decoder(),
                    "call_ms": 1e3 * float(np.median(t[arm])), "audio_s_per_s": audio_s / float(np.median(t[arm])),
                    "decode_ms_last_call": dec[arm], "hypotheses_read": hyps if arm == "nbest" else 0})
    sess.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    gpu, power = card()
    for name, n in CASES:
        for r in run_case(name, n, a.calls, a.warmup):
            r.update(gpu=gpu, power_limit=power)
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
