"""Stage trace of the persistent decoder: WB200_TRACE=<file> python scripts/trace_decode.py [model] [chunks] [kv] [depth]
Prints the mean gap between consecutive time stamps of CTA 0 (ns) per stamp index within a position."""
import os, sys
from pathlib import Path
import numpy as np
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import wb200  # noqa
from whisper_burn_b200 import audio, ffi, model, synth, transcribe

name = sys.argv[1] if len(sys.argv) > 1 else "tiny.en"
chunks = int(sys.argv[2]) if len(sys.argv) > 2 else 1
kv = sys.argv[3] if len(sys.argv) > 3 else "f32"
depth = int(sys.argv[4]) if len(sys.argv) > 4 else 20
dims, w = synth.make_weights(name, 0)
sp = synth.special_tokens(dims)
wh = model.Whisper(dims, w)
bounds = transcribe.window_bounds(480000, 16000, audio.max_waveform_samples(dims.n_audio_ctx - 10))
waves = [synth.chunk_waveform(c)[s:e] for c in range(chunks) for s, e in bounds]
sess = transcribe.Session(wh, len(waves), 1, 4 + depth + 1, ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32)
isp = (np.arange(dims.n_vocab) >= sp.first_special).astype(np.uint8)
trace_file = os.environ.pop("WB200_TRACE", None)
sess.transcribe_windows(waves, sp, isp, 1, depth)       # warm
if trace_file:
    os.environ["WB200_TRACE"] = trace_file
sess.transcribe_windows(waves, sp, isp, 1, depth)
print("decoder", sess.last_decoder())
if trace_file:
    t = np.array([int(x) for x in open(trace_file).read().split()], dtype=np.int64)
    d = np.diff(t)
    n_pos = 3 + depth
    # prefill positions have fewer stamps than logits positions: report the tail (logits positions)
    per = (len(t) - 1) // n_pos if n_pos else 0
    print("stamps", len(t), "total us", (t[-1] - t[0]) / 1e3, "per position us", (t[-1] - t[0]) / 1e3 / n_pos)
    np.save(trace_file + ".npy", t)
