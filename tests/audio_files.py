"""Writes seeded audio files in every format the readers take (tests of VoiceFixer.restore_files): RIFF/WAVE with
unsigned 8-bit, signed 16 / 24 / 32-bit integer or 32 / 64-bit float samples, and 16-bit FLAC through the in-tree
encoder, at any rate and channel count."""
import struct

import numpy as np

FORMATS = ("u8", "s16", "s24", "s32", "f32", "f64", "flac")


def _riff(tag, bits, nch, sr, payload):
    block = nch * bits // 8
    fmt = struct.pack("<HHIIHH", tag, nch, sr, sr * block, block, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(payload)) + payload
    if len(payload) & 1:
        body += b"\x00"
    return b"RIFF" + struct.pack("<I", len(body)) + body


def encode(x, sr, fmt):
    """x: float (n, channels) in [-1, 1) -> the bytes of a file in fmt."""
    x = np.clip(np.asarray(x, np.float64), -1.0, 1.0 - 2 ** -15)
    nch = x.shape[1]
    if fmt == "u8":
        return _riff(1, 8, nch, sr, np.round(x * 127 + 128).astype(np.uint8).tobytes())
    if fmt == "s16":
        return _riff(1, 16, nch, sr, np.round(x * 32767).astype("<i2").tobytes())
    if fmt == "s24":
        v = np.round(x * 8388607).astype(np.int32)
        return _riff(1, 24, nch, sr, np.stack([(v >> s) & 0xFF for s in (0, 8, 16)], -1).astype(np.uint8).tobytes())
    if fmt == "s32":
        return _riff(1, 32, nch, sr, np.round(x * 2147483647).astype("<i4").tobytes())
    if fmt == "f32":
        return _riff(3, 32, nch, sr, x.astype("<f4").tobytes())
    if fmt == "f64":
        return _riff(3, 64, nch, sr, x.astype("<f8").tobytes())
    if fmt == "flac":
        from voicefixer_b200 import _hostio
        return _hostio.flac_encode_int16(np.round(x * 32767).astype(np.int16), sr)
    raise ValueError(fmt)


def speechlike(n, channels, seed):
    """n frames of a seeded, band-limited noisy signal per channel, float64 (n, channels)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 44100.0
    base = 0.3 * np.sin(2 * np.pi * (140 + 40 * np.sin(2 * np.pi * 3 * t)) * t)
    return np.stack([base * (1 + 0.1 * c) + 0.05 * rng.standard_normal(n) for c in range(channels)], -1)


def write(path, n, sr, channels, fmt, seed):
    """Writes n frames at sr Hz with `channels` channels in fmt to path; returns path."""
    with open(str(path), "wb") as f:
        f.write(encode(speechlike(n, channels, seed), sr, fmt))
    return str(path)
