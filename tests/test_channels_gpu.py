"""Multichannel restores on the GPU: the 16-bit packer (vfx_pack_pcm16) against the host quantiser wavio.pcm16, bit for
bit; restore_files(channels="keep") against the per-file restore(channels="keep"), byte for byte; a dual-mono file
against its mix; mode 2's per-channel seeded masks; and --keep-channels with and without --batch."""
import gc
import os
import wave

import numpy as np
import pytest
import torch

import audio_files

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _device_memory_back():
    """Hands the device memory of each test's VoiceFixer instances back, before and after it (an engine keeps the
    workspace of its largest batch until the cycle collector frees it)."""
    def release():
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    release()
    yield
    release()


@pytest.fixture()
def home(tmp_path, monkeypatch):
    from voicefixer_b200 import synthetic
    monkeypatch.setenv("HOME", str(tmp_path))
    synthetic.write_checkpoints(str(tmp_path), seed=0)
    return tmp_path


# ============================================================================ the packer
def _pack(engine, files):
    """engine.pack_pcm16 on host arrays: files = [(C, n) float32 array] -> [int16 (n, C)]."""
    dev = [[torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in f] for f in files]
    y, offs = engine.pack_pcm16(dev)
    y = y.cpu().numpy()
    return [y[offs[k]:offs[k + 1]].reshape(-1, f.shape[0]) for k, f in enumerate(files)]


def _want(f):
    from voicefixer_b200 import wavio
    with np.errstate(invalid="ignore", over="ignore"):
        return wavio.pcm16(f)


def test_pack_pcm16_edge_values(engine):
    edge = np.array([[1e10, np.inf, np.nan, 65535.9, -65536.5, 32768]], np.float32)
    [got] = _pack(engine, [edge])
    assert got.ravel().tolist() == [0, 0, 0, -1, 0, -32768] == _want(edge).ravel().tolist()
    # no NaN, maximum > 1: not scaled; the int32 range's edges; a NaN of either sign; -0.0 and 1.0 in a scaled file
    files = [np.array([[2.0, -2147483648.0, 2147483520.0, 2147483648.0, -3e9, 70000.7, -1.9, -np.inf]], np.float32),
             np.array([[0.5, -np.nan, 0.25], [0.1, 0.2, 0.3]], np.float32),
             np.array([[-0.0, 1.0, -1.0, 0.999999, -0.99999, 3e-5, -3e-5, 0.0]], np.float32),
             np.array([[1.0000001, 0.5, -0.5]] * 3, np.float32)]
    for got, f in zip(_pack(engine, files), files):
        assert got.dtype == np.int16 and np.array_equal(got, _want(f)), f


def test_pack_pcm16_on_ragged_tables(engine):
    rng = np.random.default_rng(0)
    files = []
    for k in range(40):
        C, n = 1 + k % 8, int(rng.integers(3, 300000 if k % 5 == 0 else 5000))
        f = rng.uniform(-1, 1, (C, n)).astype(np.float32)
        if k % 7 == 3:
            f *= 1.5                                          # maximum > 1 in most of these
        if k % 11 == 4:
            f[rng.integers(C), rng.integers(n)] = np.nan
        if k % 13 == 5:
            f[0, 0] = 1.0                                     # maximum exactly 1: scaled
        files.append(f)
    for k, (got, f) in enumerate(zip(_pack(engine, files), files)):
        assert got.shape == (f.shape[1], f.shape[0]) and np.array_equal(got, _want(f)), f"file {k}"


def test_pack_pcm16_refuses_a_bad_table_and_writes_nothing(engine):
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import _ptr, _stream
    x = torch.full((2, 64), 0.5, device=DEV)
    y = torch.full((256,), 7, dtype=torch.int16, device=DEV)
    table = (_lib.Pcm16Item * 2)()
    for b in range(2):
        table[b].rows[0], table[b].n, table[b].C = x[b].data_ptr(), 64, 1
    table[1].dst_off = 32                                     # overlaps item 0's [0, 64)
    ws = torch.empty(engine.pack_pcm16_workspace_bytes(2), dtype=torch.uint8, device=DEV)
    rc = engine.lib.vfx_pack_pcm16(table, 2, _ptr(y), y.numel(), _ptr(ws), ws.numel(), _stream())
    torch.cuda.synchronize()
    assert rc == -1 and "overlaps" in engine.lib.vfx_last_error().decode()
    assert (y == 7).all()
    with pytest.raises(ValueError, match="9 channels"):
        engine.pack_pcm16([[x[0]] * 9])


# ============================================================================ restore_files(channels="keep")
# (name, seconds, rate, channels, format): WAV and FLAC, 16 / 44.1 / 48 kHz, one to three channels, two files over 30 s
FILES = [("a.wav", 2.0, 16000, 2, "s16"), ("b.flac", 3.0, 48000, 3, "flac"), ("c.wav", 31.5, 44100, 2, "s24"),
         ("d.flac", 1.5, 44100, 1, "flac"), ("e.wav", 4.0, 48000, 1, "f32"), ("f.flac", 32.0, 16000, 3, "flac"),
         ("g.wav", 2.5, 48000, 3, "s16"), ("h.flac", 5.0, 16000, 2, "flac")]


def _folder(root, files=FILES):
    os.makedirs(root, exist_ok=True)
    return [audio_files.write(root / name, int(sec * sr), sr, ch, fmt, seed=k)
            for k, (name, sec, sr, ch, fmt) in enumerate(files)]


def _bytes(paths):
    return [open(p, "rb").read() for p in paths]


def _differ(got, want):
    return [os.path.basename(str(g)) for g, w in zip(got, want) if _bytes([g]) != _bytes([w])]


@pytest.mark.timeout(1500)
def test_restore_files_keep_writes_what_restore_keep_writes(home):
    from voicefixer_b200 import wavio
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    srcs = _folder(home / "in")
    for mode, budget in ((0, None), (1, 44100 * 20)):          # the default budget, and many waves
        os.makedirs(home / f"ref{mode}")
        os.makedirs(home / f"got{mode}")
        ref = [str(home / f"ref{mode}" / os.path.basename(p)) for p in srcs]
        got = [str(home / f"got{mode}" / os.path.basename(p)) for p in srcs]
        for s, r in zip(srcs, ref):
            vf.restore(s, r, mode=mode, channels="keep")
        waves = []
        vf.restore_files(srcs, got, mode=mode, channels="keep", _budget=budget, _on_wave=waves.append)
        assert [i for w in waves for i in w] == list(range(len(srcs)))
        if budget is not None:
            assert len(waves) >= 4
        assert not _differ(got, ref), f"mode {mode}, waves {waves}: {_differ(got, ref)} differ"
        for s, g in zip(srcs, got):
            assert wavio.load_native(g)[0].shape[1] == wavio.load_native(s)[0].shape[1]


@pytest.mark.timeout(900)
def test_a_dual_mono_file_keeps_the_mix_in_both_channels(home):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    x = audio_files.speechlike(44100 * 3, 1, seed=5)
    src = str(home / "dual.wav")
    with open(src, "wb") as f:
        f.write(audio_files.encode(np.concatenate([x, x], 1), 22050, "s16"))
    vf.restore(src, str(home / "mix.wav"), mode=0)
    vf.restore(src, str(home / "keep.wav"), mode=0, channels="keep")
    vf.restore_files([src], [str(home / "keep_many.wav")], mode=0, channels="keep")
    mix, keep = _pcm(home / "mix.wav"), _pcm(home / "keep.wav")
    assert mix.shape[1] == 1 and keep.shape[1] == 2
    assert np.array_equal(keep[:, 0], mix[:, 0]) and np.array_equal(keep[:, 1], mix[:, 0])
    assert _bytes([home / "keep_many.wav"]) == _bytes([home / "keep.wav"])


def _pcm(path):
    with wave.open(str(path), "rb") as f:
        return np.frombuffer(f.readframes(f.getnframes()), "<i2").reshape(-1, f.getnchannels())


@pytest.mark.timeout(900)
def test_mode2_seeds_give_each_channel_its_own_stream(home):
    from voicefixer_b200 import philox, wavio
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    src = audio_files.write(home / "st.wav", 35 * 44100, 44100, 2, "s16", seed=9)      # segments k = 0 and 1
    seed = 12345
    vf.restore_files([src], [str(home / "out.wav")], mode=2, dropout_seed=seed, channels="keep")
    x = wavio.read_wave(src, 44100)
    y0 = vf.restore_inmem(x[:, 0], cuda=True, mode=2, dropout_seed=seed)
    ks = iter(range(2))                       # the plan runs segment 0 (30 s) before segment 1 (the 5 s tail)

    def masks(B, T):
        return np.stack([philox.seeded_masks(seed, (1 << 32) | next(ks), T) for _ in range(B)], 1)

    y1 = vf.restore_many([x[:, 1]], mode=2, drop_masks_fn=masks)[0]
    assert next(ks, None) is None
    got = _pcm(home / "out.wav")
    assert np.array_equal(got, wavio.pcm16(np.concatenate([y0, y1])))
    assert not np.array_equal(got[:, 0], got[:, 1])
    mono = vf.restore_inmem(x[:, 1], cuda=True, mode=2, dropout_seed=seed)          # channel 1 with channel 0's keys
    assert not np.array_equal(mono, y1)


@pytest.mark.timeout(900)
def test_cli_keep_channels_with_and_without_batch(home, monkeypatch):
    from voicefixer_b200.__main__ import main
    from voicefixer_b200.api import VoiceFixer
    monkeypatch.setenv("VFX_PRECISION", "tf32")
    files = [f for f in FILES if f[0].endswith(".wav") and f[1] <= 5.0]
    _folder(home / "in", files)
    names = sorted(f[0] for f in files)
    for out, extra in (("per_file", []), ("batch", ["--batch"])):
        assert main(["--infolder", str(home / "in"), "--outfolder", str(home / out), "--keep-channels", "--silent",
                     *extra]) == 0
    assert sorted(os.listdir(home / "batch")) == names
    assert _bytes([home / "batch" / n for n in names]) == _bytes([home / "per_file" / n for n in names])
    vf = VoiceFixer(precision="tf32")
    vf.restore(str(home / "in" / "a.wav"), str(home / "ref.wav"), channels="keep")
    assert _bytes([home / "batch" / "a.wav"]) == _bytes([home / "ref.wav"])
    assert _pcm(home / "ref.wav").shape[1] == 2
