"""whisper_b200 — H100-native (sm_90a) Whisper hot path: log-mel, encoder, KV-cached greedy decoder.

The product is the C-ABI shared library `libwhisper_b200.so` (include/whisper_b200.h) with the COM-style iModel / iContext shell
on top; this Python package is only the ctypes plumbing used by tests/ and bench.py plus the synthetic-input tooling.
"""
from . import capi, synth  # noqa: F401

__all__ = ["capi", "synth"]
