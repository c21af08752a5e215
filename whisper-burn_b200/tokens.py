"""Tokenizer bridge (SURVEY.md 8f row 3): the hot path needs only the special-token ids and the is_special bitmap
that src/transcribe.rs:179-185,243-251 obtains from `Gpt2Tokenizer` (src/token.rs:26-47, a wrapper of
tokenizers::Tokenizer::from_file("tokenizer.json")).  This reads them straight from the tokenizer.json file (Hugging
Face `tokenizers` serialisation, plain JSON); no tokenizer library is needed and no text is ever (de)tokenised here.

  * special_token(t)  = token_to_id(str(t))                          (token.rs:26-30, strings at :280-294)
  * is_special(id)    = decode([id], skip_special_tokens=True) == ""  (token.rs:37-43): true exactly for the added
    tokens flagged "special" (the decoder drops them), plus any vocabulary entry that is the empty string
  * vocab_size        = get_vocab_size(with_added_tokens=True)        (token.rs:45-47)
"""
from __future__ import annotations

import json
from typing import Dict

import numpy as np

from .synth import SpecialTokens


def _tables(path) -> (Dict[str, int], set):
    with open(path, "r", encoding="utf-8") as f:
        tj = json.load(f)
    vocab = dict(tj.get("model", {}).get("vocab", {}))
    special = set()
    for t in tj.get("added_tokens", []):
        vocab[t["content"]] = int(t["id"])
        if t.get("special", False):
            special.add(int(t["id"]))
    return vocab, special


def vocab_size(path) -> int:
    vocab, _ = _tables(path)
    return len(set(vocab.values()))


def is_special_bitmap(path, n_vocab: int = 0) -> np.ndarray:
    """[V] uint8, 1 where the reference's special_tokens_maskout holds -inf (transcribe.rs:243-244).  n_vocab pads /
    truncates to the model's vocabulary size (the reference builds the mask with the tokenizer's own size)."""
    vocab, special = _tables(path)
    v = n_vocab or len(set(vocab.values()))
    bm = np.zeros(v, dtype=np.uint8)
    for i in special:
        if i < v:
            bm[i] = 1
    for content, i in vocab.items():
        if content == "" and i < v:
            bm[i] = 1
    return bm


def special_tokens(path, language: str = "en", n_vocab: int = 0) -> SpecialTokens:
    """The ids mels_to_text looks up (transcribe.rs:179-185): prompt = [sot, <|lang|>, transcribe, notimestamps], and
    <|startofprev|>, which begins a previous-text prompt (transcribe.rs:195-199)."""
    vocab, special = _tables(path)

    def tid(s: str) -> int:
        if s not in vocab:
            raise KeyError(f"tokenizer.json has no token {s!r} (token.rs:26-30 would return None and the caller unwrap() panic)")
        return vocab[s]

    v = n_vocab or len(set(vocab.values()))
    return SpecialTokens(sot=tid("<|startoftranscript|>"), lang=tid(f"<|{language}|>"), transcribe=tid("<|transcribe|>"),
                         notimestamps=tid("<|notimestamps|>"), eot=tid("<|endoftext|>"),
                         first_special=min(special) if special else v, n_vocab=v, startofprev=vocab.get("<|startofprev|>", -1))
