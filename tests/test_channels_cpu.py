"""Multichannel restores without a GPU: the quantiser / writer split of save_wave, the multichannel reader, the seeded
dropout's per-channel stream base, the wave budget's channel count, the refusals, vfx_pack_pcm16's table checks (before
any CUDA call) and the command line's --keep-channels wiring."""
import ctypes
import os
import wave

import numpy as np
import pytest

import audio_files


def _old_save_wave(frames, fname, sample_rate=44100):
    """save_wave as it was before it was split into pcm16 and write_pcm16, kept here to pin its bytes."""
    from voicefixer_b200 import _hostio
    frames = np.array(frames, copy=True)
    shape = list(frames.shape)
    if len(shape) == 1:
        frames = frames[..., None]
        shape = list(frames.shape)
    if shape[-1] >= 3:
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
    if str(fname).lower().endswith(".flac"):
        with open(str(fname), "wb") as f:
            f.write(_hostio.flac_encode_int16(frames, sample_rate))
        return
    with wave.open(str(fname), "wb") as f:
        f.setnchannels(frames.shape[1])
        f.setsampwidth(2)
        f.setframerate(sample_rate)
        f.writeframes(np.ascontiguousarray(frames, dtype="<i2").tobytes())


def _frames(layout, seed):
    rng = np.random.default_rng(seed)
    shapes = {"1d": (5000,), "(1,L)": (1, 5000), "(1,1,L)": (1, 1, 5000), "(L,2)": (5000, 2), "(2,L)": (2, 5000),
              "(3,L)": (3, 5000), "(8,L)": (8, 5000), "loud": (2, 5000)}
    x = (0.9 * rng.uniform(-1, 1, shapes[layout])).astype(np.float32)
    return x * 3 if layout == "loud" else x                       # max > 1: written unscaled


@pytest.mark.parametrize("ext", [".wav", ".flac"])
@pytest.mark.parametrize("layout", ["1d", "(1,L)", "(1,1,L)", "(L,2)", "(2,L)", "(3,L)", "(8,L)", "loud"])
def test_save_wave_is_write_pcm16_of_pcm16_with_the_old_bytes(tmp_path, ext, layout):
    from voicefixer_b200 import wavio
    x = _frames(layout, seed=len(layout))
    wavio.save_wave(x, tmp_path / f"a{ext}")
    wavio.write_pcm16(wavio.pcm16(x), tmp_path / f"b{ext}")
    _old_save_wave(x, tmp_path / f"c{ext}")
    a, b, c = ((tmp_path / f"{k}{ext}").read_bytes() for k in "abc")
    assert a == b == c


def test_pcm16_edge_values_follow_the_x86_cast():
    from voicefixer_b200 import wavio
    v = np.array([1e10, np.inf, np.nan, 65535.9, -65536.5, 32768], np.float32)
    with np.errstate(invalid="ignore"):
        assert wavio.pcm16(v[None]).ravel().tolist() == [0, 0, 0, -1, 0, -32768]
    x = np.array([[0.5, -1.0, 1.0, -0.99999]], np.float32)          # max <= 1: scaled by 2^15, truncated
    assert wavio.pcm16(x).ravel().tolist() == [16384, -32768, -32768, -32767]


@pytest.mark.parametrize("fmt,channels,sr", [("s16", 1, 44100), ("s24", 2, 16000), ("flac", 3, 48000),
                                             ("f32", 6, 22050), ("flac", 2, 44100)])
def test_load_native_returns_every_channel_and_its_mean_is_load_mono_native(tmp_path, fmt, channels, sr):
    from voicefixer_b200 import wavio
    p = audio_files.write(tmp_path / ("a.flac" if fmt == "flac" else "a.wav"), 4001, sr, channels, fmt, seed=channels)
    x, r = wavio.load_native(p)
    assert r == sr and x.shape == (4001, channels) and x.dtype == np.float32
    m, r2 = wavio.load_mono_native(p)
    assert r2 == sr and m.dtype == np.float32 and np.array_equal(m, x.mean(axis=1).astype(np.float32))
    # restore(channels="keep") reads with read_wave: its columns are each column resampled alone
    y = wavio.read_wave(p, 44100)
    for c in range(channels):
        assert np.array_equal(y[:, c], wavio._resample(np.ascontiguousarray(x[:, c]), sr, 44100))


def test_drop_key_rows_base_zero_is_the_old_rows_and_a_base_adds_to_the_stream():
    from voicefixer_b200.api import SEG_LENGTH, drop_key_rows
    segs = [(0, 0, 100), (1, SEG_LENGTH, SEG_LENGTH + 50), (0, 2 * SEG_LENGTH, 2 * SEG_LENGTH + 9)]
    seeds = [7, (1 << 64) - 1]
    old = np.array([(seeds[i], a // SEG_LENGTH) for i, a, _ in segs], dtype=np.uint64)
    assert np.array_equal(drop_key_rows(segs, seeds), old)
    assert np.array_equal(drop_key_rows(segs, seeds, [0, 0]), old)
    rows = drop_key_rows(segs, seeds, [3 << 32, 1 << 32])
    assert rows.dtype == np.uint64 and rows[:, 0].tolist() == [7, (1 << 64) - 1, 7]
    assert rows[:, 1].tolist() == [(3 << 32) | 0, (1 << 32) | 1, (3 << 32) | 2]


def test_plan_waves_counts_every_channel_of_a_file():
    from voicefixer_b200.api import file_samples, plan_waves
    shapes = [(44100,), (44100, 2), (22050, 3), (48000, 1)]
    rates = [44100, 44100, 22050, 48000]
    n = [file_samples(s, r, 0, f"f{k}") for k, (s, r) in enumerate(zip(shapes, rates))]
    assert n == [44100, 2 * 44100, 3 * 44100, 44100]
    assert list(plan_waves(n, 3 * 44100)) == [[0, 1], [2], [3]]


def test_file_samples_refuses_more_than_eight_channels_and_short_files():
    from voicefixer_b200.api import file_samples
    assert file_samples((44100, 8), 44100, 0, "ok.wav") == 8 * 44100
    with pytest.raises(ValueError, match=r"nine\.flac has 9 channels.*at most 8"):
        file_samples((44100, 9), 44100, 0, "nine.flac")
    with pytest.raises(ValueError, match=r"short\.wav.*at least 1025"):
        file_samples((1000, 2), 44100, 0, "short.wav")


def _vf(monkeypatch):
    from voicefixer_b200 import api

    class _Eng:
        device = 0

    monkeypatch.setattr(api, "_check_cuda", lambda cuda: None)
    return api.VoiceFixer.from_engine(_Eng())


def test_bad_channels_are_refused_before_anything_is_read(monkeypatch, tmp_path):
    from voicefixer_b200 import wavio
    vf = _vf(monkeypatch)
    for name in ("load_native", "load_mono_native", "read_wave", "_read_pcm"):
        monkeypatch.setattr(wavio, name, lambda *a, **k: pytest.fail("read before channels was checked"))
    for bad in ("stereo", None, 2, "KEEP"):
        with pytest.raises(ValueError, match='channels is .*"mix" or "keep"'):
            vf.restore_files(["a.wav"], ["x.wav"], channels=bad)
        with pytest.raises(ValueError, match='channels is .*"mix" or "keep"'):
            vf.restore("a.wav", str(tmp_path / "x.wav"), channels=bad)


def test_restore_keep_restores_each_column_and_writes_them_all(monkeypatch, tmp_path):
    from voicefixer_b200 import wavio
    vf = _vf(monkeypatch)
    calls = []

    def restore_inmem(wav, cuda=False, mode=0, your_vocoder_func=None):
        calls.append((wav.copy(), mode))
        return (0.5 * np.asarray(wav, np.float32))[None]

    monkeypatch.setattr(vf, "restore_inmem", restore_inmem)
    p = audio_files.write(tmp_path / "in.wav", 3000, 22050, 3, "s16", seed=1)
    vf.restore(p, str(tmp_path / "out.flac"), mode=1, channels="keep")
    x = wavio.read_wave(p, 44100)
    assert len(calls) == 3 and all(m == 1 for _, m in calls)
    assert all(np.array_equal(w, x[:, c]) for c, (w, _) in enumerate(calls))
    wavio.save_wave(np.stack([0.5 * x[:, c] for c in range(3)]), tmp_path / "want.flac")
    assert (tmp_path / "out.flac").read_bytes() == (tmp_path / "want.flac").read_bytes()
    got, sr = wavio.load_native(str(tmp_path / "out.flac"))
    assert got.shape == (x.shape[0], 3) and sr == 44100


# ---------------------------------------------------------------------------- vfx_pack_pcm16's table checks
def _lib():
    from voicefixer_b200 import _lib
    return _lib, _lib.load()


def _table(lib_mod, items):
    t = (lib_mod.Pcm16Item * len(items))()
    for b, (rows, n, off, C) in enumerate(items):
        for c, r in enumerate(rows):
            t[b].rows[c] = r
        t[b].n, t[b].dst_off, t[b].C = n, off, C
    return t


def test_pack_pcm16_item_layout_and_workspace():
    lib_mod, lib = _lib()
    assert ctypes.sizeof(lib_mod.Pcm16Item) == 8 * 8 + 8 + 8 + 8
    assert lib.vfx_pack_pcm16_workspace_bytes(0) == 0
    assert 0 < lib.vfx_pack_pcm16_workspace_bytes(1) < lib.vfx_pack_pcm16_workspace_bytes(100)


R = [0x1000 + 0x100 * k for k in range(9)]


@pytest.mark.parametrize("case,items,match", [
    ("no_channels", [([], 10, 0, 0)], "item 0: 0 channels"),
    ("nine_channels", [(R[:8], 10, 0, 9)], "item 0: 9 channels"),
    ("null_row", [(R[:1], 10, 0, 1), ([R[0], 0], 10, 10, 2)], "item 1: channel 1's row is null"),
    ("empty", [(R[:1], 0, 0, 1)], "item 0: length 0"),
    ("past_the_end", [(R[:2], 30, 50, 2)], r"item 0: destination \[50, 110\) is not inside the 100"),
    ("negative_offset", [(R[:1], 10, -1, 1)], "item 0: destination"),
    ("overlap", [(R[:2], 10, 0, 2), (R[:1], 10, 19, 1)], "item 1: its destination overlaps item 0's"),
])
def test_pack_pcm16_refuses_a_bad_table_before_any_cuda_call(case, items, match):
    lib_mod, lib = _lib()
    rc = lib.vfx_pack_pcm16(_table(lib_mod, items), len(items), 0x2000, 100, 0x3000, 4096, None)
    assert rc == -1
    assert __import__("re").search(match, lib.vfx_last_error().decode())


# ---------------------------------------------------------------------------- the command line
class _StubFixer:
    calls = []

    def restore_files(self, inputs, outputs, mode=0, cuda=True, dropout_seed=None, channels="mix", _on_wave=None,
                      _on_wave_done=None):
        type(self).calls.append((list(inputs), list(outputs), list(mode), channels))
        _on_wave(list(range(len(inputs))))
        _on_wave_done(list(range(len(inputs))), 0.25)

    def restore_columns(self, x, cuda=False, mode=0):
        type(self).calls.append(("columns", x.shape, mode))
        return (0.25 * x.T).astype(np.float32)

    def restore_inmem(self, *a, **k):
        pytest.fail("--keep-channels ran the mono path")


def test_cli_parses_keep_channels():
    from voicefixer_b200.__main__ import build_parser
    assert build_parser().parse_args(["-i", "a.wav"]).keep_channels is False
    assert build_parser().parse_args(["-i", "a.wav", "--keep-channels"]).keep_channels is True


def test_cli_keep_channels_with_and_without_batch(tmp_path, monkeypatch, capsys):
    from voicefixer_b200 import api, wavio, __main__ as cli
    monkeypatch.setattr(api, "VoiceFixer", _StubFixer)
    _StubFixer.calls = []
    os.makedirs(tmp_path / "in")
    srcs = [audio_files.write(tmp_path / "in" / n, 3000, 22050, ch, "s16", seed=ch) for n, ch in (("a.wav", 2),
                                                                                              ("b.wav", 1))]
    argv = ["--infolder", str(tmp_path / "in"), "--outfolder", str(tmp_path / "out"), "--mode", "1", "--keep-channels"]
    assert cli.main(argv + ["--batch"]) == 0
    assert _StubFixer.calls == [(srcs, [str(tmp_path / "out" / n) for n in ("a.wav", "b.wav")], [1, 1], "keep")]
    _StubFixer.calls = []
    assert cli.main(argv) == 0
    n44 = wavio.read_wave(srcs[0], 44100).shape[0]
    assert _StubFixer.calls == [("columns", (n44, 2), 1), ("columns", (n44, 1), 1)]
    for s in srcs:
        x = wavio.read_wave(s, 44100)
        wavio.save_wave((0.25 * x.T).astype(np.float32), tmp_path / "want.wav")
        assert (tmp_path / "out" / os.path.basename(s)).read_bytes() == (tmp_path / "want.wav").read_bytes()
    out = capsys.readouterr().out
    assert all(f"Processing {s}, mode=1" in out for s in srcs)
