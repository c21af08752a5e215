"""Oracle restatement of the transcribe pipeline (reference: src/transcribe.rs), token side only.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The tokenizer (src/token.rs, HF ``tokenizers``)
is outside the hot path; it contributes 5 live special ids and an ``is_special`` bitmap
(transcribe.rs:179-185, 243-251), modelled by ``SpecialTokens``.

``use_cache=False`` is the reference-cost mode: stateless full-prefix ``forward_decoder`` on
every step for every beam with all-position logits (transcribe.rs:270, SURVEY.md F8); this is
what bench.py times as the CPU baseline.  ``use_cache=True`` runs the same arithmetic for the
last position only (oracle.model.CachedDecoder).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import audio, beam, model

BEAM_SIZE = 5      # transcribe.rs:232
MAX_DEPTH = 100    # transcribe.rs:233
PADDING = 10       # transcribe.rs:33
OVERLAP_S = 3      # transcribe.rs:120


@dataclass(frozen=True)
class SpecialTokens:
    """The ids mels_to_text looks up (transcribe.rs:179-185) + the is_special rule."""
    sot: int
    lang: int
    transcribe: int
    notimestamps: int
    eot: int
    first_special: int   # is_special(id) <=> id >= first_special (stand-in for token.rs:41-47)
    n_vocab: int

    def is_special(self, tok: int) -> bool:
        return tok >= self.first_special

    def maskout(self) -> np.ndarray:
        """special_tokens_maskout (transcribe.rs:243-251): -inf on special ids, 0 elsewhere."""
        m = np.zeros(self.n_vocab, dtype=np.float32)
        m[self.first_special:] = -np.inf
        return m

    def prompt(self) -> List[int]:
        """transcribe.rs:203 (prev-token prompt is shadowed by Vec::new(), :195-201)."""
        return [self.sot, self.lang, self.transcribe, self.notimestamps]


def window_bounds(n_samples: int, sample_rate: int, window_len: int) -> List[Tuple[int, int]]:
    """waveform_to_mel_tensor (transcribe.rs:114-138): [start, end) of every window."""
    chunk_overlap = sample_rate * OVERLAP_S
    shift = max(max(window_len - chunk_overlap, 0), 1)
    iter_len = max(n_samples - 1, 0) // shift + 1
    return [(i * shift, min(i * shift + window_len, n_samples)) for i in range(iter_len)]


def pad_mel(mels: torch.Tensor, n_ctx_max_encoder: int, padding: int = PADDING) -> torch.Tensor:
    """transcribe.rs:161-177: clip to n_ctx_max-padding frames of batch 0, append `padding` zeros."""
    _, n_mel, n_ctx = mels.shape
    keep = min(n_ctx, n_ctx_max_encoder - padding)
    return torch.cat([mels[0:1, :, 0:keep], torch.zeros(1, n_mel, padding)], dim=2)


def find_chunk_overlap(prev_tokens, curr_tokens, max_n_offsets: int, min_n_overlaps: int):
    """transcribe.rs:76-110."""
    max_overlap = 0
    max_overlap_indices = (0, 0)
    n_offsets = min(len(prev_tokens), len(curr_tokens), max_n_offsets)
    for offset in range(n_offsets):
        prev_start_index = len(prev_tokens) - 1 - offset
        matches = [i for i, (old, new) in enumerate(zip(prev_tokens[prev_start_index:], curr_tokens)) if old == new]
        n_overlap = len(matches)
        if n_overlap > max_overlap:
            max_overlap = n_overlap
            curr_overlap_index = matches[0]
            max_overlap_indices = (prev_start_index + curr_overlap_index, curr_overlap_index)
    return max_overlap_indices if max_overlap >= min_n_overlaps else None


def _prefilter(lp: np.ndarray, k: int) -> np.ndarray:
    """Indices (ascending) of every element >= the k-th largest value: a superset of what
    get_top_elements keeps; survivors' relative order only depends on survivors."""
    if lp.shape[0] <= k:
        return np.arange(lp.shape[0])
    kth = np.partition(lp, lp.shape[0] - k)[lp.shape[0] - k]
    return np.nonzero(lp >= kth)[0]


def masks_specials(max_seq_len: int) -> bool:
    """transcribe.rs:271: the special tokens are masked out while the longest beam has at most 5 tokens."""
    return not (max_seq_len > 5)


def greedy_path_log_probs(w: dict, dims: model.WhisperDims, sp: SpecialTokens, xa: torch.Tensor, tokens: List[int],
                          n_prompt: int = 4, opts: model.OracleOptions = model.DEFAULT_OPTS) -> torch.Tensor:
    """Teacher-forced greedy scoring of one window: the log-softmax rows the greedy search (beam_size 1) evaluates when it
    picks tokens[n_prompt], tokens[n_prompt + 1], ... on the path `tokens` (prompt first), with the special-token mask of
    mels_to_tokens.  xa [1, T, d] is the window's encoder output; the rows [len(tokens) - n_prompt, V] come in the dtype of
    the weights (float64 weights: a float64 reference of what the GPU computes along the same path)."""
    dec = model.CachedDecoder(w, dims, xa, opts)
    for t in tokens[:n_prompt - 1]:
        dec.step(torch.tensor([t], dtype=torch.int64))
    maskout = torch.from_numpy(sp.maskout())
    rows = []
    for i in range(n_prompt - 1, len(tokens) - 1):
        logits = dec.step(torch.tensor([tokens[i]], dtype=torch.int64))
        if masks_specials(i + 1):
            logits = logits + maskout
        rows.append(model.log_softmax_last(logits)[0])
    return torch.stack(rows)


def mels_to_tokens(w: dict, dims: model.WhisperDims, sp: SpecialTokens, mels: torch.Tensor,
                   beam_size: int = BEAM_SIZE, max_depth: int = MAX_DEPTH, use_cache: bool = True,
                   opts: model.OracleOptions = model.DEFAULT_OPTS, exact_topk: bool = False,
                   trace: Optional[dict] = None) -> List[int]:
    """mels_to_text (transcribe.rs:148-383) without detokenisation."""
    mels = pad_mel(mels, dims.n_audio_ctx)
    encoder_output = model.forward_encoder(w, dims, mels, opts)
    maskout = torch.from_numpy(sp.maskout())
    eot = sp.eot

    def is_finished(seq) -> bool:                      # transcribe.rs:235-241
        return len(seq) > 0 and seq[-1][0] == eot

    cache = {"dec": None, "rows": None}               # rows: tuple of token tuples per cache row

    def next_fn(beams: List[beam.BeamNode]):           # transcribe.rs:253-307
        max_seq_len = max((len(b.seq) for b in beams), default=0)
        if not use_cache:
            toks = [[t for t, _ in b.seq] + [0] * (max_seq_len - len(b.seq)) for b in beams]
            logits = model.forward_decoder(w, dims, torch.tensor(toks, dtype=torch.int64),
                                           encoder_output.repeat(len(beams), 1, 1), opts)
            if masks_specials(max_seq_len):
                logits = logits + maskout
            log_probs = model.log_softmax_last(logits)
            rows = [log_probs[i, len(b.seq) - 1].numpy() for i, b in enumerate(beams)]
            live = list(range(len(beams)))
        else:
            # only live beams are evaluated; continuations of finished ones are discarded (beam.rs:56-57)
            live = [i for i, b in enumerate(beams) if not is_finished(b.seq)]
            seqs = [tuple(t for t, _ in beams[i].seq) for i in live]
            dec = cache["dec"]
            if dec is None:
                dec = model.CachedDecoder(w, dims, encoder_output, opts)
                for p in range(len(seqs[0]) - 1):
                    dec.step(torch.tensor([s[p] for s in seqs], dtype=torch.int64))
                cache["dec"] = dec
            else:
                prev = cache["rows"]
                dec.reorder([prev.index(s[:-1]) for s in seqs])
            cache["rows"] = seqs
            logits = dec.step(torch.tensor([s[-1] for s in seqs], dtype=torch.int64))
            if masks_specials(max_seq_len):
                logits = logits + maskout
            log_probs = model.log_softmax_last(logits)
            rows = [None] * len(beams)
            for r, i in enumerate(live):
                rows[i] = log_probs[r].numpy()
        if trace is not None:
            trace.setdefault("log_probs", []).append([None if r is None else r.copy() for r in rows])
        out = []
        for i, b in enumerate(beams):
            if rows[i] is None:
                out.append([])
                continue
            lp = rows[i]
            idx = np.arange(lp.shape[0]) if exact_topk else _prefilter(lp, beam_size)
            out.append([((int(t), float(lp[t])), b.log_prob + float(lp[t])) for t in idx])
        return out

    initial = beam.BeamNode(seq=[(t, 0.0) for t in sp.prompt()], log_prob=0.0)
    steps: list = []
    seq = beam.beam_search([initial], next_fn, is_finished, beam_size, max_depth, trace=steps)
    if trace is not None:
        trace["n_steps"] = len(steps)
        trace["encoder_output"] = encoder_output
    return [t for t, _ in seq]


def waveform_to_tokens(w: dict, dims: model.WhisperDims, sp: SpecialTokens, waveform: np.ndarray,
                       sample_rate: int = 16000, beam_size: int = BEAM_SIZE, max_depth: int = MAX_DEPTH,
                       use_cache: bool = True, opts: model.OracleOptions = model.DEFAULT_OPTS,
                       per_window: Optional[list] = None) -> List[int]:
    """waveform_to_text (transcribe.rs:23-74) without detokenisation: merged token ids."""
    window_len = audio.max_waveform_samples(dims.n_audio_ctx - PADDING)
    tokens: List[int] = []
    for (s, e) in window_bounds(len(waveform), sample_rate, window_len):
        mel = audio.prep_audio(torch.from_numpy(np.ascontiguousarray(waveform[s:e])).unsqueeze(0), float(sample_rate))
        new_tokens = mels_to_tokens(w, dims, sp, mel, beam_size, max_depth, use_cache, opts)
        if per_window is not None:
            per_window.append(list(new_tokens))
        ov = find_chunk_overlap(tokens, new_tokens, 40, 3)
        if ov is not None:
            prev_index, curr_index = ov
            tokens = tokens[:prev_index] + new_tokens[curr_index:]
        else:
            tokens = tokens + new_tokens
    return tokens


# ---- repetition heuristics the reference compiles but only its commented-out greedy loop calls (transcribe.rs:314-447) ----
def first_repetition_end(tokens, period: int) -> int:
    """transcribe.rs:385-393.  `tokens.len() - period` is usize arithmetic: period > len panics there, ValueError here."""
    n = len(tokens)
    if period > n:
        raise ValueError("attempt to subtract with overflow")
    for i in reversed(range(period, n - period)):
        if list(tokens[i - period:i]) != list(tokens[i:i + period]):
            return i + 1
    return period


def repetition_period(tokens, min_repetitions: int):
    """transcribe.rs:395-419."""
    n = len(tokens)
    for i in reversed(range(n)):
        period = n - i
        if i // period < min_repetitions:
            return None
        if all(list(tokens[i - period * j - period:i - period * j]) == list(tokens[i:i + period]) for j in range(min_repetitions)):
            return period
    return None


def find_repeated_tokens_index(tokens, window_size: int, min_repeat_count: int):
    """transcribe.rs:421-447.  `repeats.next().unwrap()` twice: fewer than two repeats that still satisfy
    min_repeat_count panic in the reference (ValueError here)."""
    n = len(tokens)
    if 2 * window_size > n:
        return None
    last_index = n - window_size
    last_window = list(tokens[last_index:])
    repeats = [i for i in range(0, last_index - window_size + 1) if list(tokens[i:i + window_size]) == last_window]
    if len(repeats) >= min_repeat_count:
        if len(repeats) < 2:
            raise ValueError("called `Option::unwrap()` on a `None` value")
        return repeats[0], repeats[1]
    return None

