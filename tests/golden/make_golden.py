"""Generates the committed golden fixtures in tests/golden/ from the CPU oracle.

The reference (Rust + un-vendored burn/libtorch) cannot be built or run here and ships no test
vectors ("parity unpinned", oracle/__init__.py), so these fixtures are outputs of the oracle
restatement -- they pin the oracle against regressions and spare the GPU tests minutes of re-deriving
tiny.en sequences on the CPU.
Run from the repo root:  python tests/golden/make_golden.py
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
from oracle import audio, beam, model, synth, transcribe  # noqa: E402

OUT = Path(__file__).resolve().parent

MEL_CASES = [  # (n_samples, kind, seed, frame_stride)
    (400, "noise", 3, 1), (16000, "chirp", 3, 1), (16000, "mix", 1, 1), (4000, "click", 3, 1),
    (98882, "mix", 3, 25), (238559, "mix", 1234, 50),
]


def margins(trace):
    g = []
    for st in trace["log_probs"]:
        for row in st:
            if row is not None:
                s = np.sort(row)[::-1]
                g.append(float(s[0] - s[1]))
    return g


def main():
    torch.manual_seed(0)
    # ---- (i) log-mel
    mel = {}
    for n, kind, seed, stride in MEL_CASES:
        w = synth.waveform(n, seed=seed, kind=kind)
        m = audio.prep_audio(torch.from_numpy(w)[None]).numpy()[0]
        mel[f"{n}_{kind}_{seed}_{stride}"] = m[:, ::stride].astype(np.float32)
    np.savez_compressed(OUT / "mel_golden.npz", **mel)

    # ---- (iv) get_top_elements tie-break table (beam.rs:81-110)
    rng = np.random.default_rng(5)
    cases = [
        {"scores": [1.0, 3.0, 3.0, 2.0, 3.0], "num": 2},      # ties at the top: earlier indices survive
        {"scores": [5.0, 5.0, 5.0, 5.0], "num": 1},           # k=1: first-index argmax
        {"scores": [0.0, -1.0, 0.0, -1.0, 0.0, 0.0], "num": 3},
        {"scores": [2.0, 1.0], "num": 5},                     # fewer elements than num
        {"scores": [], "num": 3},
    ]
    for _ in range(20):
        n = int(rng.integers(1, 30))
        cases.append({"scores": [float(v) for v in rng.integers(-3, 4, size=n)], "num": int(rng.integers(1, 6))})
    for c in cases:
        idx = list(range(len(c["scores"])))
        c["expect"] = beam.get_top_elements(idx, lambda i: c["scores"][i], c["num"])
    (OUT / "beam_ties.json").write_text(json.dumps(cases, indent=1))

    # ---- (ii)/(iii) small model: encoder output + tokens
    chunk = synth.chunk_waveform(0)
    out = {}
    dims, w_np, w = synth.make_weights("test-a", seed=0)
    sp = synth.special_tokens(dims)
    waves = {"w238559": chunk[:238559], "w98882": chunk[:98882]}
    ta = {"model": "test-a", "seed": 0, "cases": {}}
    for name, wv in waves.items():
        m = audio.prep_audio(torch.from_numpy(wv)[None])
        for bs, depth in ((1, 30), (5, 12)):
            tr = {}
            toks = transcribe.mels_to_tokens(w, dims, sp, m, beam_size=bs, max_depth=depth, trace=tr)
            ta["cases"][f"{name}_beam{bs}_depth{depth}"] = {"tokens": toks, "min_margin": min(margins(tr))}
        if name == "w98882":
            out["test_a_enc_w98882"] = tr["encoder_output"].numpy()[0, ::8].astype(np.float32)
    # EOT handling: declare the token greedy emits at generated step 17 to be EOT -> the search must stop there
    base = ta["cases"]["w238559_beam1_depth30"]["tokens"]
    eot_tok = base[4 + 17]
    sp2 = transcribe.SpecialTokens(sp.sot, sp.lang, sp.transcribe, sp.notimestamps, eot_tok, sp.first_special, sp.n_vocab)
    toks = transcribe.mels_to_tokens(w, dims, sp2, audio.prep_audio(torch.from_numpy(waves["w238559"])[None]), beam_size=1, max_depth=30)
    ta["eot_case"] = {"eot": int(eot_tok), "tokens": toks}
    toks5 = transcribe.mels_to_tokens(w, dims, sp2, audio.prep_audio(torch.from_numpy(waves["w238559"])[None]), beam_size=5, max_depth=30)
    ta["eot_case_beam5"] = {"eot": int(eot_tok), "tokens": toks5}
    (OUT / "tokens_test_a.json").write_text(json.dumps(ta, indent=1))

    # ---- tiny.en shapes: chunk 0 = 3 reference windows, greedy to depth 100; beam 5 on the short window
    dims, w_np, w = synth.make_weights("tiny.en", seed=0)
    sp = synth.special_tokens(dims)
    window_len = audio.max_waveform_samples(dims.n_audio_ctx - transcribe.PADDING)
    bounds = transcribe.window_bounds(len(chunk), 16000, window_len)
    te = {"model": "tiny.en", "seed": 0, "bounds": bounds, "windows": [], "min_margin": None}
    gaps = []
    for i, (s, e) in enumerate(bounds):
        m = audio.prep_audio(torch.from_numpy(chunk[s:e])[None])
        tr = {}
        toks = transcribe.mels_to_tokens(w, dims, sp, m, beam_size=1, max_depth=100, trace=tr)
        te["windows"].append(toks)
        gaps += margins(tr)
        if i == 2:
            out["tiny_en_enc_w2"] = tr["encoder_output"].numpy()[0, ::16].astype(np.float32)
            toks5 = transcribe.mels_to_tokens(w, dims, sp, m, beam_size=5, max_depth=30)
            te["window2_beam5_depth30"] = toks5
    te["min_margin"] = min(gaps)
    te["merged"] = transcribe.waveform_to_tokens(w, dims, sp, chunk, beam_size=1, max_depth=100)
    (OUT / "tokens_tiny_en.json").write_text(json.dumps(te))
    np.savez_compressed(OUT / "encoder_golden.npz", **out)
    print("golden written; tiny.en min top-1/top-2 margin", te["min_margin"])


if __name__ == "__main__":
    main()
