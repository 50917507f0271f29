"""VoiceFixer.restore_files and `python -m voicefixer_b200 --batch` on the GPU, with synthetic checkpoints: every file
they write is byte for byte the file restore() (or, in seeded mode 2, the seeded restore_inmem) writes for it, in one
wave or many, and a file that cannot be read stops the run after the files before it."""
import gc
import os

import numpy as np
import pytest
import torch

import audio_files

pytestmark = pytest.mark.gpu

# (name, seconds, rate, channels, format): 0.5 s .. 65 s, so that some files have several 30 s segments and the 65 s
# one a short tail; every reader format, mono to six channels, four rates
FILES = [("a.wav", 0.5, 44100, 1, "s16"), ("b.wav", 1.2, 16000, 1, "u8"), ("c.wav", 2.0, 22050, 2, "s24"),
         ("d.flac", 3.0, 48000, 2, "flac"), ("e.wav", 65.0, 44100, 1, "s16"), ("f.wav", 4.0, 48000, 6, "s32"),
         ("g.wav", 1.0, 44100, 2, "f32"), ("h.flac", 31.0, 16000, 1, "flac"), ("i.wav", 6.0, 22050, 1, "f64"),
         ("j.wav", 0.8, 48000, 2, "s16"), ("k.flac", 12.0, 44100, 2, "flac"), ("l.wav", 45.0, 48000, 2, "s16")]


@pytest.fixture(autouse=True)
def _device_memory_back():
    """Hands the device memory of each test's VoiceFixer instances back, before and after it: an engine keeps the
    workspace of its largest batch, and a VoiceFixer and its model shim form a cycle that keeps the engine alive until
    the cycle collector runs, so without this the tests after these would find the device full."""
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


def _folder(root, files=FILES):
    os.makedirs(root, exist_ok=True)
    return [audio_files.write(root / name, int(sec * sr), sr, ch, fmt, seed=k)
            for k, (name, sec, sr, ch, fmt) in enumerate(files)]


def _bytes(paths):
    return [open(p, "rb").read() for p in paths]


def _differ(got, want):
    """The files of got whose bytes are not those of the file at the same place in want."""
    return [os.path.basename(str(g)) for g, w in zip(got, want) if _bytes([g]) != _bytes([w])]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_restore_files_writes_what_restore_writes(home, monkeypatch, precision):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision=precision)
    srcs = _folder(home / "in")
    for mode in (0, 1):
        ref = [str(home / "ref" / f"{mode}-{os.path.basename(p)}") for p in srcs]
        os.makedirs(home / "ref", exist_ok=True)
        for s, r in zip(srcs, ref):
            vf.restore(s, r, mode=mode)
        # the default budget: how many waves it makes depends on the device memory that is free
        dflt = [str(home / "default" / os.path.basename(r)) for r in ref]
        os.makedirs(home / "default", exist_ok=True)
        waves = []
        vf.restore_files(srcs, dflt, mode=mode, _on_wave=waves.append)
        assert [i for w in waves for i in w] == list(range(len(srcs)))
        assert not _differ(dflt, ref), f"mode {mode}, default budget, waves {waves}: {_differ(dflt, ref)} differ"
        # every file in one wave
        one = [str(home / "one" / os.path.basename(r)) for r in ref]
        os.makedirs(home / "one", exist_ok=True)
        waves = []
        vf.restore_files(srcs, one, mode=mode, _budget=1 << 40, _on_wave=waves.append)
        assert waves == [list(range(len(srcs)))]
        assert not _differ(one, ref), f"mode {mode}, one wave: {_differ(one, ref)} differ"
    # several waves, and batches of two segments, so that the 65 s file's three segments are split across batches
    monkeypatch.setattr(vf._engine, "max_batch", lambda L, **k: 2)
    many = [str(home / "many" / os.path.basename(p)) for p in srcs]
    os.makedirs(home / "many", exist_ok=True)
    modes = [k % 2 for k in range(len(srcs))]
    waves = []
    vf.restore_files(srcs, many, mode=modes, _budget=44100 * 20, _on_wave=waves.append)
    assert len(waves) >= 5 and [i for w in waves for i in w] == list(range(len(srcs)))
    assert [4] in waves                                                          # 65 s: a wave of its own
    want = [str(home / "ref" / f"{m}-{os.path.basename(p)}") for p, m in zip(srcs, modes)]
    assert not _differ(many, want), f"waves {waves}: {_differ(many, want)} differ"


@pytest.mark.timeout(900)
def test_restore_files_mode2(home):
    from voicefixer_b200 import wavio, resample
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    files = [f for f in FILES if f[1] >= 1.0]                                   # mode 2 needs more than 64 frames
    srcs = _folder(home / "in", files)
    seeds = [1000 + 7 * k for k in range(len(srcs))]
    os.makedirs(home / "out")
    ref = [str(home / "out" / f"ref-{os.path.basename(p)}") for p in srcs]
    for s, r, seed in zip(srcs, ref, seeds):
        wavio.save_wave(vf.restore_inmem(wavio.load_mono(s), cuda=True, mode=2, dropout_seed=seed), r)
    got = [str(home / "out" / f"got-{os.path.basename(p)}") for p in srcs]
    vf.restore_files(srcs, got, mode=2, dropout_seed=seeds)
    assert _bytes(got) == _bytes(ref)
    vf.restore_files(srcs, got, mode=2, _budget=44100 * 20)                      # random masks
    for s, g in zip(srcs, got):
        x, sr = wavio.load_mono_native(s)
        y = wavio.load_mono(g)
        assert y.shape == (resample.out_len(x.shape[0], sr),) and np.isfinite(y).all() and np.abs(y).max() > 0


@pytest.mark.timeout(900)
def test_cli_batch_writes_what_the_cli_writes(home, monkeypatch, capsys):
    from voicefixer_b200.__main__ import main
    monkeypatch.setenv("VFX_PRECISION", "tf32")
    wav_files = [f for f in FILES if f[0].endswith(".wav") and f[1] <= 12.0]    # the command line reads .wav only
    _folder(home / "in", wav_files)
    names = sorted(f[0] for f in wav_files)
    for mode in ("0", "1"):
        for out, extra in (("per_file", []), ("batch", ["--batch"])):
            assert main(["--infolder", str(home / "in"), "--outfolder", str(home / f"{out}{mode}"), "--mode", mode,
                         *extra]) == 0
        assert sorted(os.listdir(home / f"batch{mode}")) == names
        assert _bytes([home / f"batch{mode}" / n for n in names]) == _bytes([home / f"per_file{mode}" / n for n in names])
    out = capsys.readouterr().out
    assert all(f"Processing {home / 'in' / n}, mode=1" in out for n in names)
    assert main(["--infile", str(home / "in" / "g.wav"), "--outfile", str(home / "r.flac"), "--mode", "all", "--batch",
                 "--silent"]) == 0
    from voicefixer_b200 import wavio
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    for m in (0, 1):
        vf.restore(str(home / "in" / "g.wav"), str(home / f"ref-mode{m}.flac"), mode=m)
        assert _bytes([home / f"r-mode{m}.flac"]) == _bytes([home / f"ref-mode{m}.flac"])
    assert wavio.load_mono(str(home / "r-mode2.flac")).shape == (44100,)


@pytest.mark.timeout(900)
def test_restore_files_stops_at_a_truncated_file(home):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    srcs = _folder(home / "in", FILES[:6])
    with open(srcs[2], "r+b") as f:
        f.truncate(20)                                                           # inside the fmt chunk
    os.makedirs(home / "out")
    outs = [str(home / "out" / os.path.basename(p)) for p in srcs]
    with pytest.raises(RuntimeError, match="c.wav"):
        vf.restore_files(srcs, outs, mode=0)
    assert [os.path.exists(o) for o in outs] == [True, True, False, False, False, False]
    os.makedirs(home / "ref")
    for s in srcs[:2]:
        vf.restore(s, str(home / "ref" / os.path.basename(s)))
    assert _bytes(outs[:2]) == _bytes([home / "ref" / os.path.basename(s) for s in srcs[:2]])
