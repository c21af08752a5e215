"""ctypes binding of include/whisper_b200.h (the same symbols the Rust shim in rust/ binds)."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent


class WbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"[wb status {code}] {msg}")
        self.code = code
        self.msg = msg


WB_OK, WB_ERR_INVALID_ARG, WB_ERR_CUDA, WB_ERR_OOM, WB_ERR_STATE, WB_ERR_UNSUPPORTED = range(6)
WB_KV_F32, WB_KV_F16 = 0, 1
WB_WINDOWS_REFERENCE, WB_WINDOWS_NATIVE = 0, 1
WB_SEARCH_BEAM, WB_SEARCH_GREEDY_LOOP = 0, 1


class Dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer",
        "n_vocab", "n_text_ctx", "n_text_state", "n_text_head", "n_text_layer")]


class SpecialIds(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("sot", "lang", "transcribe", "notimestamps", "eot")]


def library_path() -> Path:
    return Path(os.environ.get("WB200_LIB", _HERE / "libwhisper_b200.so"))


# every symbol include/whisper_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_F = C.POINTER(C.c_float)
_I64 = C.POINTER(C.c_int64)
_I32 = C.POINTER(C.c_int32)
_U8 = C.POINTER(C.c_uint8)
SYMBOLS = {
    "wb_version": (C.c_char_p, []),
    "wb_last_error": (C.c_char_p, []),
    "wb_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "wb_max_waveform_samples": (C.c_int64, [C.c_int64]),
    "wb_window_samples": (C.c_int64, [C.c_int64, C.c_int]),
    "wb_resampled_length": (C.c_int64, [C.c_int64, C.c_int64]),
    "wb_resample": (C.c_int, [C.c_int, _F, C.c_int64, C.c_int64, C.c_int64, _F, C.c_int64, _I64]),
    "wb_prep_audio": (C.c_int, [C.c_int, _F, C.c_int64, C.c_int64, _F, _I64]),
    "wb_prep_audio_dev": (C.c_int, [C.c_int, _P, C.c_int64, C.c_int64, _P, _I64]),
    "wb_model_create": (C.c_int, [C.POINTER(Dims), C.c_int, C.POINTER(_P)]),
    "wb_model_set_tensor": (C.c_int, [_P, C.c_char_p, _F, _I64, C.c_int]),
    "wb_npy_tree_probe": (C.c_int, [C.c_char_p, C.POINTER(Dims)]),
    "wb_model_load_npy_tree": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.POINTER(_P)]),
    "wb_model_set_layernorm_eps_mode": (C.c_int, [_P, C.c_int]),
    "wb_model_finalize": (C.c_int, [_P]),
    "wb_model_destroy": (None, [_P]),
    "wb_model_get_dims": (C.c_int, [_P, C.POINTER(Dims)]),
    "wb_model_weights_fp16_exact": (C.c_int, [_P]),
    "wb_forward_encoder": (C.c_int, [_P, _F, C.c_int64, C.c_int64, C.c_int64, _F]),
    "wb_forward_decoder": (C.c_int, [_P, _I64, C.c_int64, C.c_int64, _F, C.c_int64, _F]),
    "wb_session_create": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.POINTER(_P)]),
    "wb_session_create_windows": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int, C.POINTER(_P)]),
    "wb_session_destroy": (None, [_P]),
    "wb_session_set_search": (C.c_int, [_P, C.c_int]),
    "wb_session_set_prev_prompt": (C.c_int, [_P, C.c_int64]),
    "wb_session_encode_waveforms": (C.c_int, [_P, C.POINTER(_F), _I64, C.c_int64]),
    "wb_session_encode_waveforms_dev": (C.c_int, [_P, _P, _I64, _I64, C.c_int64]),
    "wb_session_encode_mels": (C.c_int, [_P, _F, C.c_int64, C.c_int64, C.c_int64]),
    "wb_session_get_mel": (C.c_int, [_P, C.c_int64, _F, C.c_int64, _I64]),
    "wb_session_get_encoder_output": (C.c_int, [_P, C.c_int64, _F, C.c_int64, _I64]),
    "wb_session_begin": (C.c_int, [_P, _I64, C.c_int64]),
    "wb_session_step": (C.c_int, [_P, C.c_int64, _I32, _I32, _I64, C.c_int, _U8, C.c_int, _I64, _F]),
    "wb_transcribe_windows": (C.c_int, [_P, C.POINTER(_F), _I64, C.c_int64, C.c_int, C.c_int,
                                        C.POINTER(SpecialIds), _U8, _I64, C.c_int64, _I64]),
    "wb_transcribe_windows_dev": (C.c_int, [_P, _P, _I64, _I64, C.c_int64, C.c_int, C.c_int,
                                            C.POINTER(SpecialIds), _U8, _I64, C.c_int64, _I64]),
    "wb_transcribe_windows_prev": (C.c_int, [_P, C.POINTER(_F), _I64, C.c_int64, _I64, _I64, C.c_int64, C.c_int, C.c_int,
                                             C.POINTER(SpecialIds), _U8, _I64, C.c_int64, _I64]),
    "wb_waveform_to_tokens": (C.c_int, [_P, _F, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                        C.POINTER(SpecialIds), _U8, _I64, C.c_int64, _I64]),
    "wb_waveforms_to_tokens": (C.c_int, [_P, C.POINTER(_F), _I64, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                         C.POINTER(SpecialIds), _U8, _I64, C.c_int64, _I64]),
    "wb_waveforms_to_tokens_resampled": (C.c_int, [_P, C.POINTER(_F), _I64, _I64, _I64, C.c_int64, C.c_int, C.c_int,
                                                   C.POINTER(SpecialIds), _U8, _I64, C.c_int64, _I64]),
    "wb_session_last_logprobs": (C.c_int, [_P, C.c_int64, _F, C.c_int64, _I64]),
    "wb_session_last_nbest": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int64, _I64, _F, _I64, C.POINTER(C.c_double), _I32, _I64]),
    "wb_session_score_tokens": (C.c_int, [_P, C.c_int64, _I32, _I64, _I64, C.c_int, _U8, _F, _I64]),
    "wb_session_align_tokens": (C.c_int, [_P, C.c_int64, _I32, _I64, _I64, _I64, C.c_int64, _I32, _I32, _I32, _F, C.c_int64]),
    "wb_align_dtw": (C.c_int, [C.c_int, _F, C.c_int64, C.c_int64, _I32, _I32]),
    "wb_session_last_decoder": (C.c_int, [_P]),
    "wb_session_last_topk": (C.c_int, [_P, C.c_int64, C.c_int64, _I64, _F]),
    "wb_beam_search_table": (C.c_int64, [C.POINTER(C.c_double), C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _I64, C.c_int64]),
    "wb_beam_nbest_table": (C.c_int64, [C.POINTER(C.c_double), C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                        C.c_int64, C.c_int64, _I64, _I64, C.POINTER(C.c_double), _I32]),
    "wb_load_wav": (C.c_int, [C.c_char_p, C.c_int, _F, C.c_int64, _I64, _I64, C.POINTER(C.c_int)]),
    "wb_window_count": (C.c_int64, [C.c_int64, C.c_int64, C.c_int64]),
    "wb_window_bounds": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, _I64, _I64]),
    "wb_find_chunk_overlap": (C.c_int, [_I64, C.c_int64, _I64, C.c_int64, C.c_int64, C.c_int64, _I64, _I64]),
    "wb_first_repetition_end": (C.c_int64, [_I64, C.c_int64, C.c_int64]),
    "wb_repetition_period": (C.c_int64, [_I64, C.c_int64, C.c_int64]),
    "wb_find_repeated_tokens_index": (C.c_int, [_I64, C.c_int64, C.c_int64, C.c_int64, _I64, _I64]),
    "wb_beam_get_top_elements": (C.c_int64, [C.POINTER(C.c_double), C.c_int64, C.c_int64, _I64]),
    "wb_kernel_launch_count": (C.c_int64, []),
    "wb_kernel_launch_count_reset": (None, []),
    "wb_session_last_timings": (C.c_int, [_P, _F]),
    "wb_session_last_steps": (C.c_int, [_P, _I64]),
    "wb_session_profile_decode": (C.c_int, [_P, C.POINTER(SpecialIds), C.c_int, _F, _F]),
}

_lib = None


def lib() -> C.CDLL:
    """Loads libwhisper_b200.so; raises WbError (never falls back) if it has not been built."""
    global _lib
    if _lib is None:
        path = library_path()
        if not path.exists():
            raise WbError(WB_ERR_STATE, f"{path} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                        f"or `make -C whisper-burn_b200/csrc` (there is no CPU fallback)")
        handle = C.CDLL(str(path))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(status: int) -> None:
    if status != WB_OK:
        raise WbError(status, (lib().wb_last_error() or b"").decode("utf-8", "replace"))


def fptr(a):
    return a.ctypes.data_as(_F)


def i64ptr(a):
    return a.ctypes.data_as(_I64)


def i32ptr(a):
    return a.ctypes.data_as(_I32)


def u8ptr(a):
    return a.ctypes.data_as(_U8)
