"""A/B of the decoder5.cu options on one GPU (model built once): python scripts/ab_decode5.py [model] [n_chunks] [depth]
For each (kv, WB200_D5_SPLIT) combination: decode ms of a warm run, us per position, and whether the token ids equal those of the
unsplit configuration of the same K/V dtype.  (The first version of this script also toggled an L2 prefetch of the cross K/V block
and bulk-copy staging of the activation planes: both measured slower and were removed from the kernel.)"""
import itertools, json, os, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import wb200  # noqa
from whisper_burn_b200 import ffi, model, synth, transcribe

name = sys.argv[1] if len(sys.argv) > 1 else "small.en"
n_chunks = int(sys.argv[2]) if len(sys.argv) > 2 else 8
depth = int(sys.argv[3]) if len(sys.argv) > 3 else 100
dims, w_np = synth.make_weights(name)
sp = synth.special_tokens(dims)
wh = model.Whisper(dims, w_np)
del w_np
waves = []
for c in range(n_chunks):
    chunk = synth.chunk_waveform(c)
    waves += [chunk[:238559], chunk[190559:429118], chunk[381118:]]
combos = ["0", "1"]
for kv in ("f32", "f16"):
    base = None
    for split in combos:
        os.environ["WB200_D5_SPLIT"] = split
        sess = transcribe.Session(wh, len(waves), 1, 4 + depth + 1, kv_dtype=ffi.WB_KV_F16 if kv == "f16" else ffi.WB_KV_F32)
        for _ in range(2):
            toks = sess.transcribe_windows(waves, sp, sp.is_special_bitmap(), beam_size=1, max_depth=depth)
        t = sess.last_timings_ms()
        if base is None:
            base = toks
        print(json.dumps({"model": name, "rows": len(waves), "kv": kv, "split": split, "decoder": sess.last_decoder(),
                          "ms": t, "decode_us_per_position": 1e3 * t.get("decode", 0.0) / (3 + depth), "same_tokens_as_unsplit": toks == base}), flush=True)
        sess.close()
