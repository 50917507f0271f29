"""Host audio file I/O for the public API (librosa / soundfile are not in this image): WAV through
stdlib `wave`, FLAC through the in-tree C codec (include/vfx_hostio.h) -- the container follows the
file extension, as librosa.load / soundfile.write do for the reference (its test/test.py:48-57 is
FLAC in, FLAC out).

Mirrors voicefixer/tools/wav.py:9-37 (save_wave: x 2^15, int16 truncation) and :116-149
(read_wave) / librosa.load(sr=44100) mono mix used by VoiceFixer._load_wav (base.py:47-49)."""
import wave
import numpy as np


def _read_pcm(path):
    if str(path).lower().endswith(".flac"):
        from . import _hostio
        with open(str(path), "rb") as f:
            pcm, sr, bps = _hostio.flac_decode(f.read())
        return pcm.astype(np.float32) / np.float32(1 << (bps - 1)), sr
    return _read_riff(path)


def _read_riff(path):
    """RIFF/WAVE reader for what librosa.load (libsndfile) accepts on this path and stdlib `wave` does not: besides
    integer PCM of 8 / 16 / 24 / 32 bits also IEEE float 32 / 64 (format tag 3) and WAVE_FORMAT_EXTENSIBLE (0xFFFE,
    sub-format in the first two bytes of the GUID); odd-sized chunks are padded, unknown chunks skipped, a `data` size
    of 0 / 0xFFFFFFFF (streamed writers) means "to the end of the file"."""
    import struct
    with open(str(path), "rb") as f:
        blob = f.read()
    if len(blob) < 12 or blob[:4] != b"RIFF" or blob[8:12] != b"WAVE":
        raise RuntimeError(f"{path}: not a RIFF/WAVE file")
    pos, fmt, data = 12, None, None
    while pos + 8 <= len(blob):
        cid, size = blob[pos:pos + 4], struct.unpack("<I", blob[pos + 4:pos + 8])[0]
        body = pos + 8
        if cid == b"fmt ":
            if size < 16:
                raise RuntimeError(f"{path}: short fmt chunk")
            tag, nch, sr, _, _, bits = struct.unpack("<HHIIHH", blob[body:body + 16])
            if tag == 0xFFFE and size >= 26:
                tag = struct.unpack("<H", blob[body + 24:body + 26])[0]
            fmt = (tag, nch, sr, bits)
        elif cid == b"data":
            if size in (0, 0xFFFFFFFF) or body + size > len(blob):
                size = len(blob) - body
            data = blob[body:body + size]
            break
        pos = body + size + (size & 1)
    if fmt is None or data is None:
        raise RuntimeError(f"{path}: missing fmt or data chunk")
    tag, nch, sr, bits = fmt
    if nch < 1 or sr < 1:
        raise RuntimeError(f"{path}: invalid channel count / sample rate")
    width = (bits + 7) // 8
    data = data[: len(data) // (width * nch) * (width * nch)]
    if tag == 1 and bits == 16:
        x = np.frombuffer(data, dtype="<i2").astype(np.float32) / 32768.0
    elif tag == 1 and bits == 32:
        x = (np.frombuffer(data, dtype="<i4").astype(np.float64) / 2147483648.0).astype(np.float32)
    elif tag == 1 and bits == 8:
        x = (np.frombuffer(data, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    elif tag == 1 and bits == 24:
        b = np.frombuffer(data, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
        v = np.where(v >= 1 << 23, v - (1 << 24), v)
        x = v.astype(np.float32) / 8388608.0
    elif tag == 3 and bits == 32:
        x = np.frombuffer(data, dtype="<f4").astype(np.float32)
    elif tag == 3 and bits == 64:
        x = np.frombuffer(data, dtype="<f8").astype(np.float32)
    else:
        raise RuntimeError(f"{path}: unsupported WAVE format (tag {tag}, {bits} bits); PCM 8/16/24/32 and float 32/64 are read")
    return x.reshape(-1, nch), sr


def _resample(x, sr_in, sr_out):
    if sr_in == sr_out:
        return x
    from math import gcd
    from scipy.signal import resample_poly
    g = gcd(sr_in, sr_out)
    return resample_poly(x, sr_out // g, sr_in // g, axis=0).astype(np.float32)


def load_native(path):
    """(x, sr): the file's samples as float32 (L, C), one column per channel, at its own rate sr."""
    return _read_pcm(path)


def load_mono_native(path):
    """(x, sr): the file's mono mix (mean over channels), float32, at its own rate sr."""
    x, sr = load_native(path)
    return x.mean(axis=1).astype(np.float32), sr


def load_mono(path, sample_rate=44100):
    """librosa.load(path, sr=sample_rate): mono mix (mean over channels), float32."""
    return _resample(*load_mono_native(path), sample_rate)


def read_wave(path, sample_rate):
    """tools/wav.py:116-149: -> [samples, channels] float32."""
    x, sr = _read_pcm(path)
    return _resample(x, sr, sample_rate)


def pcm16(frames):
    """tools/wav.py:9-37's quantiser: float frames -> int16 (L, C).  A last axis of 3 or more is the samples axis
    ((C, L) and (1, C, L) arrays are transposed); float32 frames with max <= 1 over every sample (NaN: not <= 1) are
    scaled by 2^15, float16 / float64 frames always; then cast to int16 as C truncates on x86 (toward zero, to int32,
    the low 16 bits kept; 0 outside int32's range).  (1, N) or (1, 1, N) arrays give one channel."""
    frames = np.array(frames, copy=True)
    shape = list(frames.shape)
    if len(shape) == 1:
        frames = frames[..., None]
        shape = list(frames.shape)
    in_channels = shape[-1]
    if in_channels >= 3:
        if len(shape) == 2:
            frames = np.transpose(frames, (1, 0))
        elif len(shape) == 3:
            frames = np.transpose(frames, (0, 2, 1))
    if (np.max(frames) <= 1 and frames.dtype == np.float32) or frames.dtype in (np.float16, np.float64):
        frames = frames * 2 ** 15
    frames = frames.astype(np.short)
    if len(frames.shape) >= 3:
        frames = frames[0, ...]
    if frames.ndim == 1:
        frames = frames[:, None]
    return frames


def write_pcm16(pcm, fname, sample_rate=44100):
    """Writes int16 (L, C) samples to fname: FLAC for a .flac name (at most 8 channels), WAV otherwise."""
    if str(fname).lower().endswith(".flac"):         # soundfile.write picks the container from the extension
        from . import _hostio
        with open(str(fname), "wb") as f:
            f.write(_hostio.flac_encode_int16(pcm, sample_rate))
        return
    with wave.open(str(fname), "wb") as f:
        f.setnchannels(pcm.shape[1])
        f.setsampwidth(2)
        f.setframerate(sample_rate)
        f.writeframes(np.ascontiguousarray(pcm, dtype="<i2").tobytes())


def save_wave(frames, fname, sample_rate=44100):
    """tools/wav.py:9-37 semantics: write_pcm16(pcm16(frames)); (1, N) or (1, 1, N) arrays are written as mono, (C, N)
    arrays (N >= 3) as C channels."""
    write_pcm16(pcm16(frames), fname, sample_rate)


_MEL_BASIS = None


def slaney_htk_mel_basis():
    """librosa.filters.mel(sr=44100, n_fft=2048, htk=True, n_mels=128, fmin=0, fmax=22050) with
    its default norm='slaney' (vocoder/model/util.py:115-123); float64 build, float32 result."""
    global _MEL_BASIS
    if _MEL_BASIS is None:
        n_mels, fmax, sr, n_fft = 128, 22050.0, 44100, 2048
        fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
        mels = np.linspace(0.0, 2595.0 * np.log10(1.0 + fmax / 700.0), n_mels + 2)
        mel_f = 700.0 * (10.0 ** (mels / 2595.0) - 1.0)
        fdiff = np.diff(mel_f)
        ramps = np.subtract.outer(mel_f, fftfreqs)
        lower = -ramps[:-2] / fdiff[:-1, None]
        upper = ramps[2:] / fdiff[1:, None]
        weights = np.maximum(0, np.minimum(lower, upper))
        weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
        _MEL_BASIS = weights.astype(np.float32)
    return _MEL_BASIS
