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


def probe(path):
    """(frames, channels, rate) of an audio file from its headers, without decoding it: load_native(path)'s
    (x.shape[0], x.shape[1], sr).  WAV: the RIFF chunks are walked with seeks by _read_riff's rules (padding, extensible
    format, a `data` size of 0 / 0xFFFFFFFF or past the end meaning "to the end of the file").  FLAC: STREAMINFO's total
    samples; a stream that leaves it 0 (length unknown) is measured from its last frame's header, or, if no frame header
    is found there, estimated from the file size as if uncompressed.  Raises RuntimeError for a file that is not one."""
    import os
    import struct
    path = str(path)
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        if path.lower().endswith(".flac"):
            return _probe_flac(f, size)
        head = f.read(12)
        if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
            raise RuntimeError(f"{path}: not a RIFF/WAVE file")
        pos, fmt = 12, None
        while pos + 8 <= size:
            f.seek(pos)
            cid, csize = struct.unpack("<4sI", f.read(8))
            body = pos + 8
            if cid == b"fmt ":
                if csize < 16:
                    raise RuntimeError(f"{path}: short fmt chunk")
                _, nch, sr, _, _, bits = struct.unpack("<HHIIHH", f.read(16))
                fmt = (nch, sr, bits)
            elif cid == b"data":
                if fmt is None:
                    break
                if csize in (0, 0xFFFFFFFF) or body + csize > size:
                    csize = size - body
                nch, sr, bits = fmt
                if nch < 1 or sr < 1:
                    raise RuntimeError(f"{path}: invalid channel count / sample rate")
                return csize // ((bits + 7) // 8 * nch), nch, sr
            pos = body + csize + (csize & 1)
    raise RuntimeError(f"{path}: missing fmt or data chunk")


def _probe_flac(f, size):
    from . import _hostio
    n = 1 << 14
    while True:                                          # the metadata chain, read until STREAMINFO's block is whole
        f.seek(0)
        try:
            info = _hostio.flac_info(f.read(n))
            break
        except RuntimeError:
            if n >= size:
                raise
            n *= 8
    ch, rate, total = int(info.channels), int(info.sample_rate), int(info.total_samples)
    if total == 0:
        audio = size - int(info.audio_offset)
        tail = min(audio, int(info.max_blocksize or 65535) * ch * 5 + 4096)      # more than one frame can take
        f.seek(size - tail)
        total = _flac_last_sample(f.read(tail), info)
        if total is None:
            total = audio * 8 // (ch * int(info.bits_per_sample))
    return total, ch, rate


def _crc8(data):
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


_CRC16 = []


def _crc16(data):
    """FLAC's frame CRC-16 (polynomial 0x8005, initial 0); 0 over a whole frame, footer included."""
    if not _CRC16:
        for v in range(256):
            c = v << 8
            for _ in range(8):
                c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
            _CRC16.append(c)
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


def _flac_frame_header(h):
    """(number, blocksize, header bytes) of the FLAC frame header at the start of h, number being the frame number of
    a fixed-blocksize stream or the first sample's of a variable one; None if h does not start with a valid one."""
    if len(h) < 6 or h[0] != 0xFF or h[1] not in (0xF8, 0xF9):
        return None
    bs_code, sr_code, ch_code = h[2] >> 4, h[2] & 0x0F, h[3] >> 4
    if bs_code == 0 or sr_code == 0x0F or ch_code > 10 or h[3] & 1:
        return None
    k = 0                                                # the number's UTF-8-style coding: k leading ones, k - 1 more bytes
    while k < 8 and h[4] & (0x80 >> k):
        k += 1
    if k == 1 or k > 7 or 5 + max(k - 1, 0) > len(h):
        return None
    number, q = h[4] & (0x7F >> k), 5
    for _ in range(k - 1):
        if h[q] & 0xC0 != 0x80:
            return None
        number, q = number << 6 | h[q] & 0x3F, q + 1
    if bs_code in (6, 7):
        bs, q = int.from_bytes(h[q:q + bs_code - 5], "big") + 1, q + bs_code - 5
    else:
        bs = 192 if bs_code == 1 else (576 << (bs_code - 2) if bs_code < 6 else 256 << (bs_code - 8))
    q += {12: 1, 13: 2, 14: 2}.get(sr_code, 0)
    if q >= len(h) or _crc8(h[:q]) != h[q]:
        return None
    return number, bs, q + 1


def _flac_last_sample(tail, info):
    """One past the last sample of the FLAC frame that ends `tail` (the end of the file): the last offset that holds a
    frame header (CRC-8 checked) from which the frame's CRC-16 checks to the end; None if there is none."""
    p = len(tail)
    while p > 0:
        p = max(tail.rfind(b"\xff\xf8", 0, p), tail.rfind(b"\xff\xf9", 0, p))
        if p < 0:
            return None
        hdr = _flac_frame_header(tail[p:p + 16])
        if hdr is not None and _crc16(tail[p:]) == 0:
            number, bs, _ = hdr
            return number + bs if tail[p + 1] & 1 else number * int(info.max_blocksize) + bs
    return None


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
