"""Token alignment (Session.align_tokens) against scoring and decoding the same sequences.

For tiny.en, 1 x 30 s chunk, and small.en, 8 x 30 s chunks (reference windows, fp32 K/V): the windows are greedy-decoded to
depth 100, then exactly those sequences are aligned (default heads, first = 4) and scored, warm-up first, the two calls
alternating.  Prints per case:
  * ms per align call and per score call (host clock around the call, which ends in a device synchronise);
  * the decode-phase ms of the same positions (last_timings_ms()["decode"] of the greedy run);
  * the device time of each alignment kernel in one align call (torch.profiler, a run of its own), the DTW kernel's among
    them, with the card and its power limit.

  python scripts/bench_align.py [--calls 20] [--warmup 3]"""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def kernel_ms(sess, ids):
    """device ms per alignment kernel (and in all) of one align call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sess.align_tokens(ids, list(range(len(ids))), [4] * len(ids))
        torch.cuda.synchronize()
    out, total = {}, 0.0
    for e in prof.key_averages():
        if e.device_time_total <= 0:
            continue
        total += e.device_time_total
        for k in ("align_qk", "align_softmax", "align_stats", "align_filter", "align_dtw"):
            if k in e.key:
                out[k] = out.get(k, 0.0) + e.device_time_total / 1000.0
    out["all_kernels"] = total / 1000.0
    return {k: round(v, 3) for k, v in out.items()}


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
    bitmap = (np.arange(dims.n_vocab) >= sp.first_special).astype(np.uint8)
    sess = transcribe.Session(wh, max_windows=len(waves), max_beams=1, max_text_len=105)
    ids = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=100)
    decode_ms = sess.last_timings_ms()["decode"]
    wins, first = list(range(len(ids))), [4] * len(ids)
    for _ in range(warmup):
        sess.align_tokens(ids, wins, first)
        sess.score_tokens(ids, wins)
    t_align, t_score = [], []
    for _ in range(calls):
        t0 = time.perf_counter()
        sess.align_tokens(ids, wins, first)
        t_align.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        sess.score_tokens(ids, wins)
        t_score.append((time.perf_counter() - t0) * 1e3)
    gpu, limit = card()
    print(json.dumps({
        "case": f"{name} {n_chunks}x30s", "windows": len(waves), "positions": sum(len(t) for t in ids),
        "aligned_ids": sum(len(t) - 4 for t in ids),
        "align_ms_median": round(float(np.median(t_align)), 3), "align_ms_min": round(float(np.min(t_align)), 3),
        "score_ms_median": round(float(np.median(t_score)), 3), "decode_ms": round(decode_ms, 3),
        "kernels_ms": kernel_ms(sess, ids), "gpu": gpu, "power_limit": limit}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    for name, n in CASES:
        run_case(name, n, a.calls, a.warmup)


if __name__ == "__main__":
    main()
