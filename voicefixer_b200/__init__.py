"""voicefixer_b200 — H100-native (sm_90a) implementation of VoiceFixer's restore() hot path.

Public API mirrors the reference package:  `from voicefixer_b200 import VoiceFixer, Vocoder`.
Importing this package does not touch CUDA; constructing VoiceFixer/Vocoder/Engine loads the
in-tree CUDA library and fails loudly if it is missing (no CPU or PyTorch fallback)."""


def __getattr__(name):
    if name in ("VoiceFixer", "Vocoder"):
        from . import api
        return getattr(api, name)
    if name == "Engine":
        from .engine import Engine
        return Engine
    raise AttributeError(name)


__all__ = ["VoiceFixer", "Vocoder", "Engine"]
