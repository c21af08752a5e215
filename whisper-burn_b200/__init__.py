"""whisper-burn_b200: H100-native Whisper hot path behind whisper-burn's API surface.

The product is ``libwhisper_b200.so`` (CUDA kernels + C++ host pipeline + C ABI, see
``include/whisper_b200.h``).  This Python package is only the test / bench harness side of the
boundary: a ctypes binding (``ffi``) and thin mirrors of the reference's public functions
(``audio.prep_audio``, ``model.Whisper.forward_encoder`` ..., ``transcribe.waveform_to_text``)
so that parity tests read like calls into the reference.

The directory name contains a hyphen (it mirrors the reference's name); import it with
``import wb200`` (repo-root shim) which registers this package as ``whisper_burn_b200``.
There is no CPU fallback anywhere in this package: every compute call goes through the C ABI
and raises ``WbError`` when the library or a CUDA device is missing.
"""
from .ffi import WbError, lib, library_path  # noqa: F401
from . import audio, beam, model, npytree, shard, synth, tokens, transcribe, wav  # noqa: F401
