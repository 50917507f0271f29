"""Import alias so that code written against the reference runs unchanged:

    from voicefixer import VoiceFixer, Vocoder

resolves to the H100-native implementation in `voicefixer_b200` (same signatures, checkpoint
paths and error behaviour; see INTEGRATION.md).  Nothing is imported from the reference package."""
from voicefixer_b200 import __getattr__ as _lazy   # noqa: F401


def __getattr__(name):
    return _lazy(name)


__all__ = ["VoiceFixer", "Vocoder"]
