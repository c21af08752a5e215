#!/usr/bin/env python
"""Reference (R-mode) against native (N-mode) windowing on the GPU, one JSON line (DESIGN.md section 6).

    python scripts/bench_windows.py [--steps 5] [--warmup 3] [--max-depth 100]

A step is the hot path over synthetic 30 s chunks of 480 000 samples, already in HBM (bench.py's device path):
  R-mode: the reference's windowing, 3 windows per chunk (T = 750, 750, 314), wb_transcribe_windows_dev over all of them;
  N-mode: one 480 000-sample window per chunk (T = 1500, the last 0.1 s clipped), the same call on a native session.
Workloads: tiny.en x 1 chunk and small.en x 8 chunks, fp32 and fp16 K/V, greedy.  The two modes of a workload alternate step by
step in one process; the method is bench.py's (warm-up, a 256 MB write between steps to flush the 50 MB L2, wall clock around a
synchronised call, CUDA events on the library stream for the phases).  The card's name and power limit are read in the same run.
Algorithmic bytes of the decoder launch are bench.algorithmic_bytes with each session's real T (bench.py's version hard-codes the
reference clip)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from bench import CHUNK_SAMPLES as CHUNK, ClockSampler  # noqa: E402

WORKLOADS = [("tiny.en", 1, "f32"), ("tiny.en", 1, "f16"), ("small.en", 8, "f32"), ("small.en", 8, "f16")]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as ex:   # noqa: BLE001
        return {"error": str(ex)}


def algorithmic_bytes(dims, Ts, wbytes, kvb, steps):
    """bench.algorithmic_bytes with the encoder lengths Ts the session really has."""
    d, V, L, R = dims.n_text_state, dims.n_vocab, dims.n_text_layer, len(Ts)
    n_pos = steps + 3
    per_pos = L * 14 * d * d * wbytes + L * 2 * sum(Ts) * d * kvb
    self_kv = sum(L * 2 * (t + 1) * d * kvb * R for t in range(n_pos))
    return per_pos * n_pos + steps * V * d * wbytes + self_kv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-depth", type=int, default=100)
    a = ap.parse_args()
    import torch
    import wb200  # noqa: F401
    from whisper_burn_b200 import ffi, model, synth, transcribe
    if not torch.cuda.is_available():
        raise SystemExit("bench_windows.py: no CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    sampler = ClockSampler(0)
    sampler.start()
    rows = []
    for model_name, n_chunks, kv in WORKLOADS:
        dims, w_np = synth.make_weights(model_name, seed=0)
        sp = synth.special_tokens(dims)
        is_special = (np.arange(dims.n_vocab) >= sp.first_special).astype(np.uint8)
        wh = model.Whisper(dims, w_np)
        del w_np
        flat = np.concatenate([synth.chunk_waveform(c, CHUNK) for c in range(n_chunks)])
        wave_dev = torch.from_numpy(flat).to(dev)
        arms = {}
        for mode in ("reference", "native"):
            bounds = transcribe.window_bounds(CHUNK, 16000, transcribe.window_samples(dims.n_audio_ctx, mode))
            if mode == "native":
                bounds = [(0, CHUNK)]   # the 30 s chunk as one window (its last 0.1 s clipped)
            offs = [c * CHUNK + s for c in range(n_chunks) for s, _ in bounds]
            lens = [e - s for _ in range(n_chunks) for s, e in bounds]
            sess = transcribe.Session(wh, max_windows=len(lens), max_beams=1, max_text_len=4 + a.max_depth + 1,
                                      kv_dtype=ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32, windows=mode)
            arms[mode] = {"sess": sess, "offs": offs, "lens": lens, "wall": [], "dev": [],
                          "phase": {"logmel": 0.0, "encoder": 0.0, "decode": 0.0}}

        def step(arm):
            return arm["sess"].transcribe_windows_dev(wave_dev.data_ptr(), arm["offs"], arm["lens"], sp, is_special, 1,
                                                      a.max_depth)
        for _ in range(a.warmup):
            for arm in arms.values():
                step(arm)
        import gc
        gc.collect()
        gc.disable()
        for _ in range(a.steps):
            for arm in arms.values():   # alternated, step by step
                flush.fill_(1)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                arm["toks"] = step(arm)
                torch.cuda.synchronize()
                arm["wall"].append(1000.0 * (time.perf_counter() - t0))
                t = arm["sess"].last_timings_ms()
                arm["dev"].append(t["total"])
                for k in arm["phase"]:
                    arm["phase"][k] += t[k] / a.steps
        gc.enable()
        for mode, arm in arms.items():
            sess = arm["sess"]
            Ts = [sess.get_encoder_output(i).shape[0] for i in range(len(arm["lens"]))]
            decoder, steps_run = sess.last_decoder(), sess.last_steps()
            k_ms, _ = sess.profile_decode(sp, a.max_depth)
            n_pos = a.max_depth + 3
            alg = algorithmic_bytes(dims, Ts, 2 if wh.weights_fp16_exact else 4, 2 if kv == "f16" else 4, a.max_depth)
            ms = float(np.mean(arm["wall"]))
            rows.append({
                "mode": "N" if mode == "native" else "R", "windows": mode, "model": model_name, "chunks": n_chunks, "kv_cache": kv,
                "windows_per_step": len(Ts), "T": Ts, "decoder": decoder,
                "value": 30.0 * n_chunks / (ms / 1000.0), "unit": "audio-s/s", "ms_per_step": ms,
                "device_ms_per_step": float(np.mean(arm["dev"])), "phase_ms": arm["phase"],
                "wall_ms_each": [round(v, 3) for v in arm["wall"]],
                "decode_steps_executed": steps_run,
                "decoder_launch": {"ms": k_ms * n_pos, "positions": n_pos, "algorithmic_bytes": int(alg),
                                   "achieved_GBps": alg / (k_ms * n_pos * 1e-3) / 1e9},
                "tokens_checksum": int(sum(sum(t) for t in arm["toks"]) % (1 << 31)),
            })
            sess.close()
        del wh
    line = {"metric": "audio-seconds/sec", "card": card(), "clocks": sampler.stop(), "steps": a.steps, "warmup": a.warmup,
            "max_depth": a.max_depth, "greedy": True,
            "method": "wall clock around the synchronous wb_transcribe_windows_dev call (waveforms in HBM), L2 flushed by a 256 MB "
                      "write between steps, R and N alternated; phases and the decoder launch by CUDA events on the library stream",
            "rows": rows}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
