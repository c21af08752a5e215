"""Mirror of the reference's ``transcribe`` module (src/transcribe.rs), token side, over the C ABI.
Detokenisation (src/token.rs) stays with the caller: the library needs 5 ids and a bitmap."""
from __future__ import annotations

import base64
import ctypes as C
import gzip
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import ffi
from .model import Whisper


WINDOW_MODES = {"reference": ffi.WB_WINDOWS_REFERENCE, "native": ffi.WB_WINDOWS_NATIVE}
SEARCH_RULES = {"beam": ffi.WB_SEARCH_BEAM, "greedy_loop": ffi.WB_SEARCH_GREEDY_LOOP}


def window_samples(n_audio_ctx: int, mode: str = "reference") -> int:
    """Samples of one window (transcribe.rs:32-34) in a window mode: "reference" clips a window at n_audio_ctx mel frames,
    "native" at 2 * n_audio_ctx (the encoder's full n_audio_ctx positions)."""
    n = int(ffi.lib().wb_window_samples(n_audio_ctx, WINDOW_MODES[mode]))
    if n < 0:
        raise ValueError(f"window_samples: n_audio_ctx {n_audio_ctx} out of range")
    return n


def _special(is_special: Optional[np.ndarray]):
    """The is_special bitmap as a pointer argument (None: NULL, which the greedy loop accepts)."""
    return None if is_special is None else ffi.u8ptr(np.ascontiguousarray(is_special, dtype=np.uint8))


def _special_ids(special) -> ffi.SpecialIds:
    """The five ids the decode calls take (wb_special_ids) from a tokenizer's special tokens."""
    return ffi.SpecialIds(special.sot, special.lang, special.transcribe, special.notimestamps, special.eot)


def _host_waves(waves: Sequence[np.ndarray]):
    """(float32 arrays, which must outlive the call, their pointers, int64 sample counts) for calls taking host waveforms."""
    ws = [np.ascontiguousarray(w, dtype=np.float32) for w in waves]
    return ws, (ffi._F * len(ws))(*[ffi.fptr(w) for w in ws]), np.asarray([len(w) for w in ws], dtype=np.int64)


class Session:
    """KV-cached decoding session (wb_session): encoder output, cross/self K/V, workspaces.
    windows="reference" (default) gives the encoder at most n_audio_ctx mel frames per window, as the reference does;
    "native" gives it 2 * n_audio_ctx frames, i.e. n_audio_ctx encoder positions (one 30 s window of T = 1500).
    search="beam" (default) decodes with the reference's beam search (greedy = beam_size 1); "greedy_loop" with the greedy
    loop it leaves commented out (transcribe.rs:314-380: no special-token mask, EOT-probability stop, repetition cut, context
    stop; beam_size must be 1 and is_special may be None)."""

    def __init__(self, whisper: Whisper, max_windows: int, max_beams: int = 5, max_text_len: int = 104,
                 kv_dtype: int = ffi.WB_KV_F32, windows: str = "reference", search: str = "beam"):
        if windows not in WINDOW_MODES:
            raise ValueError(f"windows must be one of {sorted(WINDOW_MODES)}, not {windows!r}")
        if search not in SEARCH_RULES:
            raise ValueError(f"search must be one of {sorted(SEARCH_RULES)}, not {search!r}")
        self.whisper = whisper
        self.max_windows = max_windows
        self.windows = windows
        n_ctx = whisper.config.n_audio_ctx
        self.max_mel_frames = 2 * n_ctx if windows == "native" else n_ctx
        self._h = C.c_void_p()
        ffi.check(ffi.lib().wb_session_create_windows(whisper.handle, max_windows, max_beams, max_text_len, kv_dtype,
                                                      WINDOW_MODES[windows], C.byref(self._h)))
        self.search = search
        ffi.check(ffi.lib().wb_session_set_search(self._h, SEARCH_RULES[search]))

    def close(self):
        if getattr(self, "_h", None):
            ffi.lib().wb_session_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- encode
    def set_prev_prompt(self, startofprev: int) -> None:
        """The previous-text prompt of waveform(s)_to_tokens (wb_session_set_prev_prompt): -1 (the default) decodes every window
        from [sot, lang, transcribe, notimestamps]; the <|startofprev|> id prompts window i of a waveform with
        [startofprev] + the last (at most) 5 non-special merged ids so far + those 4 ids, the windows of a waveform in order."""
        ffi.check(ffi.lib().wb_session_set_prev_prompt(self._h, startofprev))

    def encode_waveforms(self, waves: Sequence[np.ndarray]) -> None:
        ws, ptrs, lens = _host_waves(waves)
        ffi.check(ffi.lib().wb_session_encode_waveforms(self._h, ptrs, ffi.i64ptr(lens), len(ws)))

    def encode_mels(self, mels: np.ndarray) -> None:
        mels = np.ascontiguousarray(mels, dtype=np.float32)
        n, n_mels, n_ctx = mels.shape
        ffi.check(ffi.lib().wb_session_encode_mels(self._h, ffi.fptr(mels), n, n_mels, n_ctx))

    def get_mel(self, window: int) -> np.ndarray:
        cap = 80 * self.max_mel_frames
        buf = np.empty(cap, dtype=np.float32)
        n = C.c_int64(0)
        ffi.check(ffi.lib().wb_session_get_mel(self._h, window, ffi.fptr(buf), cap, C.byref(n)))
        return buf[:80 * n.value].reshape(80, n.value).copy()

    def get_encoder_output(self, window: int) -> np.ndarray:
        d = self.whisper.config.n_audio_state
        cap = d * ((self.max_mel_frames - 1) // 2 + 1)
        buf = np.empty(cap, dtype=np.float32)
        n = C.c_int64(0)
        ffi.check(ffi.lib().wb_session_get_encoder_output(self._h, window, ffi.fptr(buf), cap, C.byref(n)))
        return buf[:d * n.value].reshape(n.value, d).copy()

    # ---- decode
    def begin(self, prompt: Sequence[int]) -> None:
        p = np.asarray(prompt, dtype=np.int64)
        ffi.check(ffi.lib().wb_session_begin(self._h, ffi.i64ptr(p), len(p)))

    def step(self, window_of_row, parent_row, token, apply_special_mask: bool, is_special: Optional[np.ndarray], k: int):
        w = np.asarray(window_of_row, dtype=np.int32)
        pr = np.asarray(parent_row, dtype=np.int32)
        tk = np.asarray(token, dtype=np.int64)
        n = len(w)
        ids = np.empty((n, k), dtype=np.int64)
        lps = np.empty((n, k), dtype=np.float32)
        ffi.check(ffi.lib().wb_session_step(self._h, n, ffi.i32ptr(w), ffi.i32ptr(pr), ffi.i64ptr(tk),
                                           1 if apply_special_mask else 0, _special(is_special), k, ffi.i64ptr(ids),
                                           ffi.fptr(lps)))
        return ids, lps

    # ---- pipelines
    def transcribe_windows(self, waves: Sequence[np.ndarray], special, is_special: np.ndarray, beam_size: int = 5,
                           max_depth: int = 100) -> List[List[int]]:
        """mels_to_text for a batch of windows (transcribe.rs:148-383), ids only."""
        ws, ptrs, lens = _host_waves(waves)
        cap = 4 + max_depth + 1
        out = np.zeros((len(ws), cap), dtype=np.int64)
        out_len = np.zeros(len(ws), dtype=np.int64)
        ffi.check(ffi.lib().wb_transcribe_windows(self._h, ptrs, ffi.i64ptr(lens), len(ws), beam_size, max_depth,
                                                 C.byref(_special_ids(special)), _special(is_special), ffi.i64ptr(out), cap,
                                                 ffi.i64ptr(out_len)))
        return [[int(t) for t in out[i, :out_len[i]]] for i in range(len(ws))]

    def transcribe_windows_prev(self, waves: Sequence[np.ndarray], prev: Sequence[Sequence[int]], special,
                                is_special: Optional[np.ndarray], beam_size: int = 5, max_depth: int = 100,
                                startofprev: Optional[int] = None) -> List[List[int]]:
        """mels_to_text with its prev_nonspecial_tokens given per window (wb_transcribe_windows_prev): window i is decoded
        from [startofprev] + prev[i] + [sot, lang, transcribe, notimestamps], or the 4 ids when prev[i] is empty; rows hold
        the prompt first.  startofprev defaults to special.startofprev."""
        ws, ptrs, lens = _host_waves(waves)
        if len(prev) != len(ws):
            raise ValueError(f"transcribe_windows_prev: {len(ws)} windows but {len(prev)} previous-id lists")
        prev_lens = np.asarray([len(p) for p in prev], dtype=np.int64)
        prev_toks = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.int64) for p in prev] + [np.zeros(1, np.int64)]))
        cap = max([4] + [len(p) + 5 for p in prev if len(p)]) + max_depth + 1
        out = np.zeros((len(ws), cap), dtype=np.int64)
        out_len = np.zeros(len(ws), dtype=np.int64)
        sop = special.startofprev if startofprev is None else startofprev
        ffi.check(ffi.lib().wb_transcribe_windows_prev(self._h, ptrs, ffi.i64ptr(lens), len(ws), ffi.i64ptr(prev_toks),
                                                      ffi.i64ptr(prev_lens), sop, beam_size, max_depth,
                                                      C.byref(_special_ids(special)),
                                                      _special(is_special), ffi.i64ptr(out), cap, ffi.i64ptr(out_len)))
        return [[int(t) for t in out[i, :out_len[i]]] for i in range(len(ws))]

    def transcribe_windows_dev(self, wave_dev_ptr: int, offsets, lens, special, is_special: np.ndarray,
                               beam_size: int = 5, max_depth: int = 100) -> List[List[int]]:
        """Same, windows already resident in HBM (device pointer + element offsets)."""
        offs = np.asarray(offsets, dtype=np.int64)
        ln = np.asarray(lens, dtype=np.int64)
        cap = 4 + max_depth + 1
        out = np.zeros((len(ln), cap), dtype=np.int64)
        out_len = np.zeros(len(ln), dtype=np.int64)
        ffi.check(ffi.lib().wb_transcribe_windows_dev(self._h, C.c_void_p(wave_dev_ptr), ffi.i64ptr(offs), ffi.i64ptr(ln),
                                                     len(ln), beam_size, max_depth, C.byref(_special_ids(special)),
                                                     _special(is_special), ffi.i64ptr(out), cap, ffi.i64ptr(out_len)))
        return [[int(t) for t in out[i, :out_len[i]]] for i in range(len(ln))]

    def waveform_to_tokens(self, waveform: np.ndarray, special, is_special: np.ndarray, sample_rate: int = 16000,
                           beam_size: int = 5, max_depth: int = 100) -> List[int]:
        w = np.ascontiguousarray(waveform, dtype=np.float32)
        cap = (len(w) // 1000 + 2) * (10 + max_depth + 1) + 16
        out = np.zeros(cap, dtype=np.int64)
        n = C.c_int64(0)
        ffi.check(ffi.lib().wb_waveform_to_tokens(self._h, ffi.fptr(w), len(w), sample_rate, beam_size, max_depth,
                                                 C.byref(_special_ids(special)), _special(is_special), ffi.i64ptr(out), cap,
                                                 C.byref(n)))
        return [int(t) for t in out[:n.value]]

    def waveforms_to_tokens(self, waveforms: Sequence[np.ndarray], special, is_special: np.ndarray, sample_rate: int = 16000,
                            beam_size: int = 5, max_depth: int = 100) -> List[List[int]]:
        """Batched waveform_to_tokens: all windows of all waveforms decoded together (wb_waveforms_to_tokens)."""
        ws, ptrs, lens = _host_waves(waveforms)
        cap = (max(len(w) for w in ws) // 1000 + 2) * (10 + max_depth + 1) + 16
        out = np.zeros((len(ws), cap), dtype=np.int64)
        n = np.zeros(len(ws), dtype=np.int64)
        ffi.check(ffi.lib().wb_waveforms_to_tokens(self._h, ptrs, ffi.i64ptr(lens), len(ws), sample_rate, beam_size, max_depth,
                                                  C.byref(_special_ids(special)), _special(is_special), ffi.i64ptr(out), cap,
                                                  ffi.i64ptr(n)))
        return [[int(t) for t in out[i, :n[i]]] for i in range(len(ws))]

    def waveforms_to_tokens_resampled(self, waveforms: Sequence[np.ndarray], sample_rates: Sequence[int], special,
                                      is_special: np.ndarray, beam_size: int = 5, max_depth: int = 100) -> List[List[int]]:
        """waveforms_to_tokens for waveforms of any rate and channel count (wb_waveforms_to_tokens_resampled): waveform i is
        1-D (mono) or 2-D [n_frames, channels] at sample_rates[i]; all are converted to 16 kHz mono on the GPU as
        audio.resample does, then decoded as waveforms_to_tokens decodes the converted audio."""
        from .audio import _frames, resampled_length
        ws = [_frames(w) for w in waveforms]
        if len(sample_rates) != len(ws):
            raise ValueError("one sample rate per waveform")
        ptrs = (ffi._F * len(ws))(*[ffi.fptr(w) for w in ws])
        frames = np.asarray([w.shape[0] for w in ws], dtype=np.int64)
        channels = np.asarray([w.shape[1] for w in ws], dtype=np.int64)
        rates = np.asarray(sample_rates, dtype=np.int64)
        n16 = max(max(resampled_length(int(n), int(r)) for n, r in zip(frames, rates)), 0)
        cap = (n16 // 1000 + 2) * (10 + max_depth + 1) + 16
        out = np.zeros((len(ws), cap), dtype=np.int64)
        n = np.zeros(len(ws), dtype=np.int64)
        ffi.check(ffi.lib().wb_waveforms_to_tokens_resampled(self._h, ptrs, ffi.i64ptr(frames), ffi.i64ptr(channels),
                                                            ffi.i64ptr(rates), len(ws), beam_size, max_depth,
                                                            C.byref(_special_ids(special)), _special(is_special),
                                                            ffi.i64ptr(out), cap, ffi.i64ptr(n)))
        return [[int(t) for t in out[i, :n[i]]] for i in range(len(ws))]

    def last_logprobs(self, index: int) -> np.ndarray:
        """float32 log-prob of each id of row `index` (window or waveform) of the last transcribe_windows[_dev] /
        waveform(s)_to_tokens call: 0 for the prompt, the log-prob the search chose the id with, NaN for an EOT the greedy
        loop's rules appended (wb_session_last_logprobs)."""
        n = C.c_int64(0)
        ffi.check(ffi.lib().wb_session_last_logprobs(self._h, index, None, 0, C.byref(n)))
        out = np.empty(n.value, dtype=np.float32)
        ffi.check(ffi.lib().wb_session_last_logprobs(self._h, index, ffi.fptr(out), n.value, C.byref(n)))
        return out

    def last_nbest(self, index: int):
        """The n-best list of window `index` of the last transcribe_windows[_dev/_prev] call, or of window `index` in
        waveform-major order of the last waveform(s)_to_tokens call (wb_session_last_nbest): the beam search's final carried
        list, best first, as (ids, float32 log-probs (0 for the prompt), f64 score = their left-to-right sum, finished).
        Rank 0 is the row the call returned.  WbError (WB_ERR_STATE) after a greedy-loop call."""
        n = C.c_int64(0)
        ffi.check(ffi.lib().wb_session_last_nbest(self._h, index, 0, 0, None, None, None, None, None, C.byref(n)))
        lens = np.zeros(max(n.value, 1), dtype=np.int64)
        ffi.check(ffi.lib().wb_session_last_nbest(self._h, index, n.value, 0, None, None, ffi.i64ptr(lens), None, None,
                                                  C.byref(n)))
        cap = max(int(lens[:n.value].max(initial=0)), 1)
        ids = np.zeros((max(n.value, 1), cap), dtype=np.int64)
        lps = np.zeros((max(n.value, 1), cap), dtype=np.float32)
        scores = np.zeros(max(n.value, 1), dtype=np.float64)
        fin = np.zeros(max(n.value, 1), dtype=np.int32)
        ffi.check(ffi.lib().wb_session_last_nbest(self._h, index, n.value, cap, ffi.i64ptr(ids), ffi.fptr(lps), ffi.i64ptr(lens),
                                                  scores.ctypes.data_as(C.POINTER(C.c_double)), ffi.i32ptr(fin), C.byref(n)))
        return [([int(t) for t in ids[r, :lens[r]]], lps[r, :lens[r]].copy(), float(scores[r]), bool(fin[r]))
                for r in range(n.value)]

    def score_tokens(self, seqs: Sequence[Sequence[int]], windows: Sequence[int], apply_special_mask: bool = False,
                     is_special: Optional[np.ndarray] = None):
        """Teacher-forced scoring of token sequences against the encoded windows (wb_session_score_tokens): sequence i on
        window windows[i].  Returns per sequence (lp float32[len], argmax int64[len]): lp[j] is the log-softmax of position
        j - 1's logits at seqs[i][j] and argmax[j] that row's arg-max id, for j >= 1; lp[0] = 0, argmax[0] = -1.
        apply_special_mask: special ids get -inf in the rows whose prefix has <= 5 tokens (the beam search's rule)."""
        lens = np.asarray([len(s) for s in seqs], dtype=np.int64)
        toks = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int64) for s in seqs]) if len(seqs)
                                    else np.zeros(0, dtype=np.int64), dtype=np.int64)
        win = np.ascontiguousarray(windows, dtype=np.int32)
        if len(win) != len(lens):
            raise ValueError(f"score_tokens: {len(lens)} sequences but {len(win)} windows")
        lp = np.empty(max(len(toks), 1), dtype=np.float32)
        am = np.empty(max(len(toks), 1), dtype=np.int64)
        ffi.check(ffi.lib().wb_session_score_tokens(self._h, len(lens), ffi.i32ptr(win), ffi.i64ptr(toks), ffi.i64ptr(lens),
                                                   1 if apply_special_mask else 0, _special(is_special), ffi.fptr(lp),
                                                   ffi.i64ptr(am)))
        offs = np.concatenate([[0], np.cumsum(lens)])
        return [(lp[offs[i]:offs[i + 1]].copy(), am[offs[i]:offs[i + 1]].copy()) for i in range(len(lens))]

    def align_tokens(self, seqs: Sequence[Sequence[int]], windows: Sequence[int], first: Sequence[int],
                     heads: Optional[Sequence[Tuple[int, int]]] = None, return_matrix: bool = False):
        """When each token was spoken (wb_session_align_tokens): openai-whisper's find_alignment over the encoded windows,
        sequence i on window windows[i] with its aligned ids seqs[i][first[i]:] (first = 4 for a default transcribe row, the
        prompt length for a previous-text row).  heads: (layer, head) pairs, None for every head of the second half of the
        decoder layers (alignment_heads_from_openai gives a checkpoint's tuned heads).  Returns per sequence (start, end),
        int32 encoder positions of each aligned id (20 ms each from the window's start), with return_matrix also its
        float32 alignment matrix [len - first, C]."""
        lens = np.asarray([len(s) for s in seqs], dtype=np.int64)
        toks = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int64) for s in seqs]) if len(seqs)
                                    else np.zeros(0, dtype=np.int64), dtype=np.int64)
        win = np.ascontiguousarray(windows, dtype=np.int32)
        fst = np.ascontiguousarray(first, dtype=np.int64)
        if len(win) != len(lens) or len(fst) != len(lens):
            raise ValueError(f"align_tokens: {len(lens)} sequences, {len(win)} windows and {len(fst)} first indices")
        hs = np.ascontiguousarray(np.asarray(heads if heads is not None else [], dtype=np.int32).reshape(-1, 2))
        n_ids = int(np.clip(lens - fst, 1, None).sum()) if len(lens) else 1
        start = np.empty(max(n_ids, 1), dtype=np.int32)
        end = np.empty(max(n_ids, 1), dtype=np.int32)
        cap = n_ids * self.whisper.config.n_audio_ctx if return_matrix else 0   # C <= n_audio_ctx
        mat = np.empty(max(cap, 1), dtype=np.float32)
        ffi.check(ffi.lib().wb_session_align_tokens(self._h, len(lens), ffi.i32ptr(win), ffi.i64ptr(toks), ffi.i64ptr(lens),
                                                   ffi.i64ptr(fst), len(hs), ffi.i32ptr(hs) if len(hs) else None,
                                                   ffi.i32ptr(start), ffi.i32ptr(end), ffi.fptr(mat) if return_matrix else None,
                                                   cap))
        out, a, m = [], 0, 0
        for L, f in zip(lens, fst):
            n = int(L - f)
            st, en = start[a:a + n].copy(), end[a:a + n].copy()
            if return_matrix:
                c = int(en[-1])   # end of the last aligned id = the column count
                out.append((st, en, mat[m:m + n * c].reshape(n, c).copy()))
                m += n * c
            else:
                out.append((st, en))
            a += n
        return out

    def last_decoder(self) -> int:
        return int(ffi.lib().wb_session_last_decoder(self._h))

    def last_topk(self, n_rows: int, k: int = 1):
        """(ids [n_rows, k] int64, log-probs [n_rows, k] float32) the last decoder launch selected at its last position."""
        ids = np.empty((n_rows, k), dtype=np.int64)
        lps = np.empty((n_rows, k), dtype=np.float32)
        ffi.check(ffi.lib().wb_session_last_topk(self._h, n_rows, k, ffi.i64ptr(ids), ffi.fptr(lps)))
        return ids, lps

    def last_timings_ms(self):
        buf = np.zeros(4, dtype=np.float32)
        ffi.check(ffi.lib().wb_session_last_timings(self._h, ffi.fptr(buf)))
        return {"logmel": float(buf[0]), "encoder": float(buf[1]), "decode": float(buf[2]), "total": float(buf[3])}

    def profile_decode(self, special, n_steps: int = 50):
        """(average logits-GEMV ms, average whole-step ms) over n_steps re-run greedy steps."""
        a, b = C.c_float(0), C.c_float(0)
        ffi.check(ffi.lib().wb_session_profile_decode(self._h, C.byref(_special_ids(special)), n_steps, C.byref(a), C.byref(b)))
        return float(a.value), float(b.value)

    def last_steps(self) -> int:
        n = C.c_int64(0)
        ffi.check(ffi.lib().wb_session_last_steps(self._h, C.byref(n)))
        return int(n.value)


def waveform_to_text(whisper: Whisper, special, is_special: np.ndarray, waveform: np.ndarray, sample_rate: int = 16000,
                     beam_size: int = 5, max_depth: int = 100, max_windows: int = 8) -> List[int]:
    """transcribe::waveform_to_text (transcribe.rs:23-74) without detokenisation: merged token ids.
    (`bpe` and `lang` of the reference signature collapse into `special` / `is_special`.)"""
    s = Session(whisper, max_windows=max_windows, max_beams=max(beam_size, 1), max_text_len=4 + max_depth + 1)
    try:
        return s.waveform_to_tokens(waveform, special, is_special, sample_rate, beam_size, max_depth)
    finally:
        s.close()


def align_dtw(matrix: np.ndarray, device: int = 0):
    """(start, end) int32 per row of the DTW on -matrix that wb_session_align_tokens runs, alone, on the GPU (wb_align_dtw):
    matrix float32 [N, C], N in [1, 448]."""
    m = np.ascontiguousarray(matrix, dtype=np.float32)
    if m.ndim != 2:
        raise ValueError("align_dtw: matrix must be 2-D")
    start = np.empty(max(m.shape[0], 1), dtype=np.int32)
    end = np.empty(max(m.shape[0], 1), dtype=np.int32)
    ffi.check(ffi.lib().wb_align_dtw(device, ffi.fptr(m), m.shape[0], m.shape[1], ffi.i32ptr(start), ffi.i32ptr(end)))
    return start[:m.shape[0]], end[:m.shape[0]]


def alignment_heads_from_openai(b85: str | bytes, dims) -> List[Tuple[int, int]]:
    """The (layer, head) pairs of an openai-whisper alignment-head mask (whisper/__init__.py _ALIGNMENT_HEADS): base85 of a
    gzip'ed bool array [n_text_layer][n_text_head], ascending."""
    raw = gzip.decompress(base64.b85decode(b85))
    if len(raw) != dims.n_text_layer * dims.n_text_head:
        raise ValueError(f"alignment heads: {len(raw)} mask entries, not n_text_layer x n_text_head = "
                         f"{dims.n_text_layer * dims.n_text_head}")
    mask = np.frombuffer(raw, dtype=bool).reshape(dims.n_text_layer, dims.n_text_head)
    return [(int(l), int(h)) for l, h in zip(*np.nonzero(mask))]


def window_bounds(n_samples: int, sample_rate: int, window_len: int):
    n = int(ffi.lib().wb_window_count(n_samples, sample_rate, window_len))
    st = np.zeros(n, dtype=np.int64)
    en = np.zeros(n, dtype=np.int64)
    ffi.check(ffi.lib().wb_window_bounds(n_samples, sample_rate, window_len, ffi.i64ptr(st), ffi.i64ptr(en)))
    return [(int(a), int(b)) for a, b in zip(st, en)]


def find_chunk_overlap(prev_tokens, curr_tokens, max_n_offsets: int, min_n_overlaps: int):
    p = np.asarray(prev_tokens, dtype=np.int64)
    c = np.asarray(curr_tokens, dtype=np.int64)
    pi, ci = C.c_int64(0), C.c_int64(0)
    found = ffi.lib().wb_find_chunk_overlap(ffi.i64ptr(p), len(p), ffi.i64ptr(c), len(c), max_n_offsets, min_n_overlaps,
                                            C.byref(pi), C.byref(ci))
    return (pi.value, ci.value) if found else None


def first_repetition_end(tokens, period: int) -> int:
    """transcribe.rs:385-393 (ValueError where the reference's usize arithmetic underflows)."""
    t = np.asarray(tokens, dtype=np.int64)
    r = int(ffi.lib().wb_first_repetition_end(ffi.i64ptr(t), len(t), period))
    if r < 0:
        raise ValueError("first_repetition_end: period exceeds the token count")
    return r


def repetition_period(tokens, min_repetitions: int):
    """transcribe.rs:395-419: the period, or None."""
    t = np.asarray(tokens, dtype=np.int64)
    r = int(ffi.lib().wb_repetition_period(ffi.i64ptr(t), len(t), min_repetitions))
    if r < 0:
        raise ValueError("repetition_period: invalid argument")
    return r if r > 0 else None


def find_repeated_tokens_index(tokens, window_size: int, min_repeat_count: int):
    """transcribe.rs:421-447: (index of the first repeat, index of the second) or None (ValueError where the reference panics)."""
    t = np.asarray(tokens, dtype=np.int64)
    a, b = C.c_int64(0), C.c_int64(0)
    r = int(ffi.lib().wb_find_repeated_tokens_index(ffi.i64ptr(t), len(t), window_size, min_repeat_count, C.byref(a), C.byref(b)))
    if r < 0:
        raise ValueError("find_repeated_tokens_index: the reference unwraps a repeat that does not exist")
    return (a.value, b.value) if r else None
