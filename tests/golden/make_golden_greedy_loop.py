"""Golden token fixture of the greedy loop (WB_SEARCH_GREEDY_LOOP, src/transcribe.rs:314-380), from the CPU oracle loop
(tests/oracle_greedy_loop.py).

  tiny.en  seed 0, one 30 s chunk (synth.chunk_waveform(0)) in the reference's 3 windows, fp32 and fp16 K/V,
           max_depth = n_text_ctx - 4 = 444 (the reference's loop exactly), the synthetic special ids (EOT = 50256)

Every record has the token ids, the rule that stopped the window, and per step the EOT-test gap
(eot_logit - token_logit) - ln 0.5 and the top-1 / top-2 logit gap.
Run from the repo root:  python tests/golden/make_golden_greedy_loop.py
"""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import oracle_greedy_loop as loop  # noqa: E402
from oracle import audio, model, synth, transcribe  # noqa: E402

OUT = Path(__file__).resolve().parent / "tokens_greedy_loop.json"


def main():
    torch.set_num_threads(8)
    dims, _, w = synth.make_weights("tiny.en", seed=0)
    sp = synth.special_tokens(dims)
    chunk = synth.chunk_waveform(0)
    window_len = audio.max_waveform_samples(dims.n_audio_ctx - transcribe.PADDING)
    bounds = transcribe.window_bounds(len(chunk), 16000, window_len)
    max_depth = dims.n_text_ctx - 4
    rec = {"model": "tiny.en", "seed": 0, "chunk": 0, "eot": sp.eot, "max_depth": max_depth, "bounds": bounds}
    for kv in ("f32", "f16"):
        opts = model.OracleOptions(kv_dtype=kv)
        rows = []
        for (s, e) in bounds:
            mel = audio.prep_audio(torch.from_numpy(chunk[s:e].copy()).unsqueeze(0), 16000.0)
            tr = {}
            toks = loop.mels_to_tokens_greedy_loop(w, dims, sp, mel, max_depth, opts, trace=tr)
            rows.append({"tokens": toks, "stop": tr["stop"], "eot_gap": tr["eot_gap"], "top_gap": tr["top_gap"]})
            print(kv, (s, e), len(toks), tr["stop"], flush=True)
        rec[kv] = rows
    OUT.write_text(json.dumps(rec))


if __name__ == "__main__":
    main()
