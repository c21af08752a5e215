"""Cost of converting audio to 16 kHz mono on the GPU (resample.cu), printed as JSON lines with the card and its power limit.

Kernel: 8 x 30 s at 44.1 kHz stereo, 48 kHz stereo, 22.05 kHz mono and 8 kHz mono, each case as one wb_resample call on the
8 chunks back to back (the bytes and taps of 8 waveforms in one launch).  The kernel time is the mean resample_poly_kernel
duration from torch.profiler (CUDA activities) over --calls calls, in a run of its own after warm-up.  Beside it: the
algorithmic bytes 4*n*C + 4*n_out and f64 FLOP 2*n_out*ceil((2*half + 1)/up) (DESIGN.md section 5), the least time each
needs at the H100 SXM data-sheet rates (3.35 TB/s HBM3, 34 TFLOP/s FP64 non-tensor; data-sheet figures, not measured), which
of the two bounds the kernel, and the host scipy.signal.resample_poly time on the same input, for scale.

End to end: tiny.en synthetic weights, 8 x 30 s chunks, greedy depth 100 as bench.py.  waveforms_to_tokens_resampled on the
chunks as 44.1 kHz stereo against waveforms_to_tokens on the same audio already converted to 16 kHz mono, alternating the
two, --repeats timed calls each after warm-up; audio-s/s (host clock around each call, which ends in a device synchronise),
best and spread, and the difference of the best times.

  python scripts/bench_resample.py [--calls 20] [--repeats 7]"""
import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import wb200  # noqa: E402,F401
from whisper_burn_b200 import audio, model, synth, transcribe  # noqa: E402

CHUNKS, CHUNK_SECONDS = 8, 30
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
FP64_FLOP_PER_S = 34e12     # H100 SXM data sheet, FP64 non-tensor
CASES = ((44100, 2), (48000, 2), (22050, 1), (8000, 1))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def emit(line):
    print(json.dumps(line), flush=True)


def ratio(sr):
    g = math.gcd(sr, 16000)
    return 16000 // g, sr // g


def signal(sr, channels, seed):
    """CHUNKS x 30 s at sr with `channels` channels: seeded noise plus tones, f32 [n, channels]"""
    rng = np.random.default_rng(seed)
    n = CHUNKS * CHUNK_SECONDS * sr
    t = np.arange(n) / sr
    x = 0.05 * rng.standard_normal((n, channels))
    for c in range(channels):
        x[:, c] += 0.1 * np.sin(2 * np.pi * (440.0 + 110 * c) * t)
    return x.astype(np.float32)


def kernel_case(sr, channels, calls):
    import scipy.signal
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    x = signal(sr, channels, seed=sr + channels)
    up, down = ratio(sr)
    half = 0 if up == down else 10 * max(up, down)
    n, n_out = x.shape[0], audio.resampled_length(x.shape[0], sr)
    bytes_ = 4 * n * channels + 4 * n_out
    flop = 2 * n_out * -(-(2 * half + 1) // up)
    for _ in range(3):
        y = audio.resample(x, sr)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            audio.resample(x, sr)
        torch.cuda.synchronize()
    times = [e.time_range.elapsed_us() for e in prof.events()
             if e.device_type == DeviceType.CUDA and "resample_poly_kernel" in e.name]   # us
    assert len(times) == calls, f"found {len(times)} resample_poly_kernel launches for {calls} calls"
    kernel_us = float(np.mean(times))
    t0 = time.perf_counter()
    ref = scipy.signal.resample_poly(x.astype(np.float64).mean(axis=1), up, down)
    host_s = time.perf_counter() - t0
    t_bytes, t_flop = bytes_ / HBM_BYTES_PER_S, flop / FP64_FLOP_PER_S
    emit({"case": f"{CHUNKS}x{CHUNK_SECONDS}s {sr} Hz C={channels}", "up": up, "down": down, "half": half,
          "n_frames": n, "n_out": n_out, "kernel_us_mean": round(kernel_us, 2), "kernel_us_min": round(float(np.min(times)), 2),
          "algorithmic_bytes": bytes_, "f64_flop": flop,
          "achieved_GB_per_s": round(bytes_ / kernel_us / 1e3, 1), "achieved_f64_TFLOP_per_s": round(flop / kernel_us / 1e6, 3),
          "datasheet_min_us_bytes": round(t_bytes * 1e6, 2), "datasheet_min_us_flop": round(t_flop * 1e6, 2),
          "bound": "bytes" if t_bytes >= t_flop else "f64 FLOP",
          "share_of_datasheet_bound": round(max(t_bytes, t_flop) * 1e6 / kernel_us, 3),
          "host_scipy_resample_poly_ms": round(host_s * 1e3, 1),
          "max_abs_diff_vs_scipy": float(np.abs(y.astype(np.float64) - ref).max())})


def end_to_end(repeats):
    import scipy.signal
    dims, w_np = synth.make_weights("tiny.en", seed=0)
    sp = synth.special_tokens(dims)
    wh = model.Whisper(dims, w_np)
    del w_np
    is_special = (np.arange(dims.n_vocab) >= sp.first_special).astype(np.uint8)
    # the bench.py chunks, brought to 44.1 kHz stereo on the host (the second channel 0.9x the first)
    x44 = []
    for c in range(CHUNKS):
        m = scipy.signal.resample_poly(synth.chunk_waveform(c).astype(np.float64), 441, 160)
        x44.append(np.stack([m, 0.9 * m], axis=1).astype(np.float32))
    conv = [audio.resample(x, 44100) for x in x44]
    window_len = transcribe.window_samples(dims.n_audio_ctx)
    n_win = sum(len(transcribe.window_bounds(len(c), 16000, window_len)) for c in conv)
    sess = transcribe.Session(wh, max_windows=n_win, max_beams=1, max_text_len=4 + 100 + 1)
    arms = {"resampled_44k1_stereo": lambda: sess.waveforms_to_tokens_resampled(x44, [44100] * CHUNKS, sp, is_special, 1, 100),
            "16k_mono_converted": lambda: sess.waveforms_to_tokens(conv, sp, is_special, 16000, 1, 100)}
    out = {k: f() for k, f in arms.items()}   # warm-up
    assert out["resampled_44k1_stereo"] == out["16k_mono_converted"], "token ids differ between the arms"
    for f in arms.values():
        f()
    times = {k: [] for k in arms}
    for _ in range(repeats):
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    audio_s = CHUNKS * CHUNK_SECONDS
    line = {"case": f"end to end tiny.en {CHUNKS}x{CHUNK_SECONDS}s greedy depth 100", "windows": n_win, "repeats": repeats,
            "ids_identical": True}
    for k, ts in times.items():
        line[k] = {"best_audio_s_per_s": round(audio_s / min(ts), 1), "worst_audio_s_per_s": round(audio_s / max(ts), 1),
                   "best_ms": round(min(ts) * 1e3, 2), "median_ms": round(float(np.median(ts)) * 1e3, 2)}
    diffs = [a - b for a, b in zip(times["resampled_44k1_stereo"], times["16k_mono_converted"])]
    line["extra_ms_best"] = round((min(times["resampled_44k1_stereo"]) - min(times["16k_mono_converted"])) * 1e3, 2)
    line["extra_ms_per_pair_min_median_max"] = [round(v * 1e3, 2) for v in (min(diffs), float(np.median(diffs)), max(diffs))]
    emit(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    name, power = card()
    emit({"gpu": name, "power_limit": power})
    for sr, c in CASES:
        kernel_case(sr, c, args.calls)
    end_to_end(args.repeats)


if __name__ == "__main__":
    main()
