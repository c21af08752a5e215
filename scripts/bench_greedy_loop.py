#!/usr/bin/env python
"""The beam rule's greedy search against the greedy loop (WB_SEARCH_GREEDY_LOOP) on the GPU, one JSON line (DESIGN.md section 6).

    python scripts/bench_greedy_loop.py [--steps 5] [--warmup 2]

A step is wb_transcribe_windows_dev over synthetic 30 s chunks already in HBM, in the reference's windowing (3 windows per
chunk), fp32 K/V.  Workloads: tiny.en x 1 chunk and small.en x 8 chunks.  Arms, alternated step by step in one process:
  beam:       WB_SEARCH_BEAM, beam_size 1, max_depth 100 (the greedy path bench.py times);
  loop-100:   WB_SEARCH_GREEDY_LOOP, max_depth 100 (same bound, the loop's stopping rules);
  loop-444:   WB_SEARCH_GREEDY_LOOP, max_depth n_text_ctx - 4 (the reference's loop).
Per arm: the positions the decoder ran (prompt prefill + steps to the last finished row), decode ms (CUDA events on the
library stream) and decode us per position.  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))

from bench import CHUNK_SAMPLES as CHUNK  # noqa: E402
from bench_windows import card  # noqa: E402

WORKLOADS = [("tiny.en", 1), ("small.en", 8)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    import wb200  # noqa: F401
    from whisper_burn_b200 import ffi, model, synth, transcribe
    if not torch.cuda.is_available():
        raise SystemExit("bench_greedy_loop.py: no CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    rows = []
    for model_name, n_chunks in WORKLOADS:
        dims, w_np = synth.make_weights(model_name, seed=0)
        sp = synth.special_tokens(dims)
        is_special = sp.is_special_bitmap()
        wh = model.Whisper(dims, w_np)
        del w_np
        flat = np.concatenate([synth.chunk_waveform(c, CHUNK) for c in range(n_chunks)])
        wave_dev = torch.from_numpy(flat).to(dev)
        bounds = transcribe.window_bounds(CHUNK, 16000, transcribe.window_samples(dims.n_audio_ctx))
        offs = [c * CHUNK + s for c in range(n_chunks) for s, _ in bounds]
        lens = [e - s for _ in range(n_chunks) for s, e in bounds]
        arms = {}
        for name, search, depth in (("beam", "beam", 100), ("loop-100", "greedy_loop", 100),
                                    ("loop-444", "greedy_loop", dims.n_text_ctx - 4)):
            sess = transcribe.Session(wh, max_windows=len(lens), max_beams=1, max_text_len=dims.n_text_ctx,
                                      kv_dtype=ffi.WB_KV_F32, search=search)
            arms[name] = {"sess": sess, "depth": depth, "wall": [], "decode": [], "steps": []}

        def step(arm):
            return arm["sess"].transcribe_windows_dev(wave_dev.data_ptr(), offs, lens, sp, is_special, 1, arm["depth"])
        for _ in range(a.warmup):
            for arm in arms.values():
                step(arm)
        for _ in range(a.steps):
            for arm in arms.values():   # alternated, step by step
                flush.fill_(1)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                arm["toks"] = step(arm)
                torch.cuda.synchronize()
                arm["wall"].append(1000.0 * (time.perf_counter() - t0))
                arm["decode"].append(arm["sess"].last_timings_ms()["decode"])
                arm["steps"].append(arm["sess"].last_steps())
        for name, arm in arms.items():
            positions = 3 + int(arm["steps"][-1])
            dec_ms = float(np.median(arm["decode"]))
            rows.append({
                "model": model_name, "chunks": n_chunks, "windows": len(lens), "arm": name, "max_depth": arm["depth"],
                "decoder": arm["sess"].last_decoder(), "positions": positions,
                "decode_ms": dec_ms, "decode_ms_each": [round(v, 3) for v in arm["decode"]],
                "us_per_position": 1000.0 * dec_ms / positions, "wall_ms": float(np.median(arm["wall"])),
                "tokens_per_window": [len(t) for t in arm["toks"]],
            })
            arm["sess"].close()
        del wh
    print(json.dumps({"card": card(), "steps": a.steps, "warmup": a.warmup, "kv_cache": "f32",
                      "method": "decode phase by CUDA events on the library stream (median over steps), arms alternated step "
                                "by step, L2 flushed by a 256 MB write between steps",
                      "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
