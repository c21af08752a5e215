"""Teacher-forced scoring (Session.score_tokens) against the decode that produced the same positions.

For tiny.en, 1 x 30 s chunk, and small.en, 8 x 30 s chunks (reference windows), with fp32 and with fp16 K/V: the windows
are greedy-decoded to depth 100, then exactly those sequences are scored, warm-up first, the two K/V arms alternating call
by call.  Prints per case and arm:
  * ms per score call (host clock around the call, which ends in a device synchronise) and positions scored per second;
  * the decode-phase ms of the same positions (last_timings_ms()["decode"] of the greedy run);
  * the logits stage (the statistics GEMM, one torch.profiler run of its own) against the larger of its FLOP bound
    (2 planes x 2 P V d at 989 TFLOP/s dense fp16) and its byte bound (3.35 TB/s HBM3), with the card and its power limit.

  python scripts/bench_score.py [--calls 20] [--warmup 3]"""
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
from whisper_burn_b200 import ffi, model, transcribe  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12   # H100 SXM data sheet: dense fp16, HBM3
CASES = (("tiny.en", 1), ("small.en", 8))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def logits_kernel_ms(sess, seqs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sess.score_tokens(seqs, list(range(len(seqs))))
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if "LogitArgs" in e.key) / 1000.0


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
    arms = {}
    for kv in ("f32", "f16"):
        sess = transcribe.Session(wh, max_windows=len(waves), max_beams=1, max_text_len=105,
                                  kv_dtype=ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32)
        ids = sess.transcribe_windows(waves, sp, bitmap, beam_size=1, max_depth=100)
        arms[kv] = {"sess": sess, "ids": ids, "decode_ms": sess.last_timings_ms()["decode"], "t": []}
        for _ in range(warmup):
            sess.score_tokens(ids, list(range(len(ids))), apply_special_mask=True, is_special=bitmap)
    for _ in range(calls):
        for kv, a in arms.items():
            t0 = time.perf_counter()
            a["sess"].score_tokens(a["ids"], list(range(len(a["ids"]))), apply_special_mask=True, is_special=bitmap)
            a["t"].append((time.perf_counter() - t0) * 1e3)
    d, V = dims.n_text_state, dims.n_vocab
    for kv, a in arms.items():
        P = sum(len(t) - 1 for t in a["ids"])                      # rows of the pass: every position but the last
        n_tiles = (V + 127) // 128
        flop_s = 2 * 2 * P * V * d / PEAK_FLOPS
        byte_s = (V * d * 2 + 2 * P * d * 2 + P * n_tiles * 12 + P * 12) / PEAK_BYTES
        lg_ms = logits_kernel_ms(a["sess"], a["ids"])
        ms = float(np.median(a["t"]))
        print(json.dumps({
            "case": f"{name} {n_chunks}x30s", "kv": kv, "windows": len(waves), "positions": P + len(a["ids"]),
            "score_ms_median": round(ms, 3), "score_ms_min": round(float(np.min(a["t"])), 3),
            "positions_per_s": round((P + len(a["ids"])) / (ms / 1e3)),
            "decode_ms_same_positions": round(a["decode_ms"], 3),
            "logits_stage_ms": round(lg_ms, 4), "logits_bound_ms": round(max(flop_s, byte_s) * 1e3, 4),
            "logits_bound": "flop" if flop_s >= byte_s else "bytes",
            "logits_share_of_bound": round(max(flop_s, byte_s) * 1e3 / lg_ms, 3) if lg_ms > 0 else None}))
        a["sess"].close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}))
    for case, n in CASES:
        run_case(case, n, args.calls, args.warmup)


if __name__ == "__main__":
    main()
