"""restore_files over several GPUs, the parts that need none: wavio.probe against load_native on every reader format,
plan_devices' assignment, parallel.run_on_devices with fake targets in spawned processes, restore_files' refusals of
a bad gpus, and the command line's --gpus."""
import multiprocessing
import os
import pickle
import struct
import time

import numpy as np
import pytest
import torch

import audio_files


# ---------------------------------------------------------------------------- wavio.probe
@pytest.mark.parametrize("fmt", audio_files.FORMATS)
@pytest.mark.parametrize("channels,sr,n", [(1, 16000, 12345), (2, 44100, 70001), (3, 48000, 4097), (1, 22050, 1)])
def test_probe_is_load_native_shape_and_rate(tmp_path, fmt, channels, sr, n):
    from voicefixer_b200 import wavio
    p = audio_files.write(tmp_path / f"x.{'flac' if fmt == 'flac' else 'wav'}", n, sr, channels, fmt, seed=n)
    x, rate = wavio.load_native(p)
    assert wavio.probe(p) == (x.shape[0], x.shape[1], rate) == (n, channels, sr)


def _wav_with(tmp_path, name, data_size=None, junk=None, extensible=False):
    """A 16-bit stereo WAV of 5001 frames, its data size field replaced, an odd-sized chunk before `data`, or its fmt
    chunk WAVE_FORMAT_EXTENSIBLE."""
    blob = bytearray(audio_files.encode(audio_files.speechlike(5001, 2, 3), 32000, "s16"))
    if extensible:
        fmt = bytes(blob[20:36])
        ext = struct.pack("<HHIIHH", 0xFFFE, *struct.unpack("<HIIHH", fmt[2:])) + struct.pack("<HHI", 22, 16, 3) + \
            struct.pack("<H", 1) + bytes(14)
        blob = blob[:16] + struct.pack("<I", len(ext)) + ext + blob[36:]
    if junk is not None:
        at = blob.index(b"data")
        blob = blob[:at] + b"LIST" + struct.pack("<I", len(junk)) + junk + b"\x00" * (len(junk) & 1) + blob[at:]
    if data_size is not None:
        at = blob.index(b"data")
        blob[at + 4:at + 8] = struct.pack("<I", data_size)
    p = tmp_path / name
    p.write_bytes(bytes(blob))
    return str(p)


def _flac_without_total(tmp_path, n, channels, sr):
    """A FLAC stream whose STREAMINFO leaves the total samples 0 (length unknown, as a streaming encoder writes)."""
    blob = bytearray(audio_files.encode(audio_files.speechlike(n, channels, 5), sr, "flac"))
    info = 8                                             # "fLaC", then the STREAMINFO block's 4-byte header
    blob[info + 13] &= 0xF0
    blob[info + 14:info + 18] = bytes(4)
    p = tmp_path / f"unknown{n}.flac"
    p.write_bytes(bytes(blob))
    return str(p)


def test_probe_follows_the_riff_rules_and_measures_a_flac_of_unknown_length(tmp_path):
    from voicefixer_b200 import wavio
    paths = [_wav_with(tmp_path, "ffff.wav", data_size=0xFFFFFFFF), _wav_with(tmp_path, "zero.wav", data_size=0),
             _wav_with(tmp_path, "long.wav", data_size=1 << 30), _wav_with(tmp_path, "odd.wav", junk=b"abc"),
             _wav_with(tmp_path, "ext.wav", extensible=True)]
    paths += [_flac_without_total(tmp_path, n, ch, sr) for n, ch, sr in ((70001, 2, 48000), (4096, 1, 16000),
                                                                         (300, 3, 44100), (123457, 1, 22050))]
    for p in paths:
        x, rate = wavio.load_native(p)
        assert wavio.probe(p) == (x.shape[0], x.shape[1], rate), p
    with open(paths[-1], "rb") as f:                     # its STREAMINFO really says "unknown"
        from voicefixer_b200 import _hostio
        assert _hostio.flac_info(f.read(4096)).total_samples == 0


def test_probe_reads_headers_only_and_refuses_what_is_not_audio(tmp_path, monkeypatch):
    from voicefixer_b200 import wavio
    p = audio_files.write(tmp_path / "big.wav", 44100 * 20, 44100, 2, "s16", seed=0)
    f = tmp_path / "big.flac"
    audio_files.write(f, 44100 * 20, 44100, 2, "flac", seed=0)
    reads = []
    real_open = open

    class Counting:
        def __init__(self, fh):
            self.fh = fh

        def __enter__(self):
            return self

        def __exit__(self, *a):
            self.fh.close()

        def read(self, n=-1):
            data = self.fh.read(n)
            reads.append(len(data))
            return data

        def seek(self, *a):
            return self.fh.seek(*a)

    monkeypatch.setattr("builtins.open", lambda *a, **k: Counting(real_open(*a, **k)))
    assert wavio.probe(p) == (44100 * 20, 2, 44100) and sum(reads) < 100
    reads.clear()
    assert wavio.probe(str(f)) == (44100 * 20, 2, 44100) and sum(reads) < 1 << 15
    monkeypatch.undo()
    (tmp_path / "no.wav").write_bytes(b"RIFX" + bytes(40))
    (tmp_path / "no.flac").write_bytes(b"OggS" + bytes(60))
    for bad in ("no.wav", "no.flac"):
        with pytest.raises(RuntimeError):
            wavio.probe(str(tmp_path / bad))


# ---------------------------------------------------------------------------- plan_devices
def _check_plan(weights, sources, n, shards):
    assert len(shards) == n
    assert sorted(i for s in shards for i in s) == list(range(len(weights)))
    assert all(s == sorted(s) for s in shards)
    where = {}
    for d, s in enumerate(shards):
        for i in s:
            assert where.setdefault(sources[i], d) == d, "one input on two devices"
    groups = {}
    for w, src in zip(weights, sources):
        groups[src] = groups.get(src, 0) + w
    loads = [sum(weights[i] for i in s) for s in shards]
    assert max(loads) <= max(groups.values()) + sum(weights) / n


def test_plan_devices_balances_keeps_order_and_keeps_an_input_on_one_device():
    from voicefixer_b200.api import plan_devices
    rng = np.random.default_rng(0)
    for trial in range(200):
        m = int(rng.integers(1, 40))
        n = int(rng.integers(1, 9))
        weights = [int(w) for w in rng.integers(0, 10 ** 6, m)]
        sources = [f"f{int(k)}.wav" for k in rng.integers(0, max(1, m // 2 if trial % 3 == 0 else m), m)]
        shards = plan_devices(weights, sources, n)
        _check_plan(weights, sources, n, shards)
        assert shards == plan_devices(list(weights), list(sources), n)           # deterministic
    # longest first onto the least-loaded device, ties to the lower index; more devices than files
    assert plan_devices([5, 9, 1, 4], ["a", "b", "c", "d"], 2) == [[1, 2], [0, 3]]
    assert plan_devices([3, 3, 3], ["a", "b", "c"], 5) == [[0], [1], [2], [], []]
    # --mode all: every input three times in a row, each triple on one device
    assert plan_devices([2, 2, 2, 1, 1, 1, 3, 3, 3], list("aaabbbccc"), 2) == [[6, 7, 8], [0, 1, 2, 3, 4, 5]]
    assert plan_devices([0, 0], ["a", "b"], 2) == [[0, 1], []]                    # weight 0 adds no load


def test_probe_samples_weighs_channels_restored_and_unprobeable_files_zero(tmp_path):
    from voicefixer_b200.api import _probe_samples
    from voicefixer_b200 import resample
    a = audio_files.write(tmp_path / "a.wav", 16000, 16000, 2, "s16", seed=1)
    (tmp_path / "bad.wav").write_bytes(b"nothing")
    n44 = resample.out_len(16000, 16000)
    assert _probe_samples([a, str(tmp_path / "bad.wav"), a, "missing.flac"], [0, 0, 1, 0], False) == [n44, 0, n44, 0]
    assert _probe_samples([a], [0], True) == [2 * n44]


# ---------------------------------------------------------------------------- parallel.run_on_devices
def _fake_target(device, shard, args):
    """Writes one marker file per index, after args["sleep"][device] seconds; fails at args["fail"].get(device) (an
    index of its shard) with ValueError, or exits with code 3 on args["exit"]."""
    time.sleep(args.get("sleep", {}).get(device, 0))
    if args.get("exit") == device:
        os._exit(3)
    for i in shard:
        if args.get("fail", {}).get(device) == i:
            return i, ValueError(f"file {i} failed on device {device}")
        with open(os.path.join(args["dir"], f"{i}-{device}"), "w") as f:
            f.write(str(os.getpid()))
    return None


def _markers(d):
    return sorted(os.listdir(d))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n", [2, 3])
def test_run_on_devices_collects_every_shard(tmp_path, n):
    from voicefixer_b200.parallel import run_on_devices
    shards = [(d, [i for i in range(10) if i % n == d]) for d in range(n)]
    assert run_on_devices(shards, _fake_target, {"dir": str(tmp_path), "sleep": {0: 0.5}}) is None
    assert _markers(tmp_path) == sorted(f"{i}-{i % n}" for i in range(10))
    pids = {d: {open(tmp_path / f"{i}-{d}").read() for i in s} for d, s in shards}
    assert pids[0] == {str(os.getpid())} and len({p for d in pids for p in pids[d]}) == n     # the caller runs shard 0
    assert multiprocessing.active_children() == []


@pytest.mark.timeout(300)
@pytest.mark.parametrize("slow", [1, 2])
def test_run_on_devices_raises_the_lowest_failing_index_whoever_finishes_last(tmp_path, slow):
    from voicefixer_b200.parallel import run_on_devices
    shards = [(0, [0, 3, 6, 9]), (1, [1, 4, 7]), (2, [2, 5, 8])]
    args = {"dir": str(tmp_path), "fail": {0: 9, 1: 7, 2: 5}, "sleep": {slow: 2.0}}
    with pytest.raises(ValueError, match="^file 5 failed on device 2$"):
        run_on_devices(shards, _fake_target, args)
    assert _markers(tmp_path) == ["0-0", "1-1", "2-2", "3-0", "4-1", "6-0"]        # every shard ran to its failure
    assert multiprocessing.active_children() == []
    # the caller's own failure, when it is the lowest, is raised as the very exception
    args = {"dir": str(tmp_path), "fail": {0: 3, 1: 4}}
    with pytest.raises(ValueError, match="^file 3 failed on device 0$") as e:
        run_on_devices(shards[:2], _fake_target, args)
    assert e.value.__traceback__ is not None
    assert multiprocessing.active_children() == []


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n", [2, 3])
def test_run_on_devices_names_a_worker_that_dies(tmp_path, n):
    from voicefixer_b200.parallel import run_on_devices
    shards = [(d, [d, d + n]) for d in range(n)]
    with pytest.raises(RuntimeError, match="device 1 exited with code 3"):
        run_on_devices(shards, _fake_target, {"dir": str(tmp_path), "exit": 1})
    assert _markers(tmp_path) == sorted(f"{i}-{d}" for d, s in shards if d != 1 for i in s)
    assert multiprocessing.active_children() == []


# ---------------------------------------------------------------------------- restore_files(gpus=)
class _Eng:
    device = 0
    precision = "tf32"
    table = [("a.w", 0, 10)]
    arena = torch.arange(64, dtype=torch.uint8)


def _vf(monkeypatch, count=1):
    from voicefixer_b200 import api, wavio
    monkeypatch.setattr(api, "_check_cuda", lambda cuda: None)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: count)
    for name in ("load_native", "load_mono_native", "read_wave", "_read_pcm", "probe"):
        monkeypatch.setattr(wavio, name, lambda *a, **k: pytest.fail("a file was opened"))
    return api.VoiceFixer.from_engine(_Eng())


def test_restore_files_refuses_a_bad_gpus_before_any_file_is_opened(monkeypatch):
    from voicefixer_b200 import parallel
    vf = _vf(monkeypatch, count=2)
    monkeypatch.setattr(parallel, "run_on_devices", lambda *a: pytest.fail("workers started"))
    for bad in (0, -1, 2.5, 3, "2", True, 2.0):
        with pytest.raises(ValueError, match="gpus"):
            vf.restore_files(["a.wav", "b.wav"], ["x.wav", "y.wav"], gpus=bad)
    with pytest.raises(ValueError, match="mode must be 0, 1 or 2"):               # the existing checks come first
        vf.restore_files(["a.wav"], ["x.wav"], mode=3, gpus=0)
    with pytest.raises(ValueError, match="no file is restored in mode 2"):
        vf.restore_files(["a.wav"], ["x.wav"], dropout_seed=1, gpus=2)


def test_restore_files_hands_each_device_its_shard_and_the_arena(monkeypatch, tmp_path):
    from voicefixer_b200 import api, parallel, wavio
    vf = _vf(monkeypatch, count=4)
    lengths = {"a.wav": 44100 * 9, "b.wav": 44100 * 5, "c.wav": 44100 * 4}
    monkeypatch.setattr(wavio, "probe", lambda p: (lengths[p], 2, 44100))
    seen = []
    monkeypatch.setattr(parallel, "run_on_devices", lambda shards, target, args: seen.append((shards, target, args)))
    _Eng.device = 3
    try:
        vf.restore_files(["a.wav", "b.wav", "c.wav", "a.wav"], ["w", "x", "y", "z"], mode=[0, 2, 2, 1], dropout_seed=7,
                         gpus=3, _messages=("took",))
    finally:
        _Eng.device = 0
    [(shards, target, args)] = seen
    assert target is api._restore_shard and shards == [(3, [0, 3]), (0, [1]), (1, [2])]
    assert args.modes == [0, 2, 2, 1] and args.seeds == [7, 7, 7, 7] and args.messages == ("took",)
    assert torch.equal(args.arena, _Eng.arena) and args.arena.is_shared() and args.table == _Eng.table
    assert args.vf is vf and pickle.loads(pickle.dumps(args)).vf is None               # the instance stays here


# ---------------------------------------------------------------------------- the command line
class _StubFixer:
    calls = []

    def restore_files(self, inputs, outputs, mode=0, cuda=True, dropout_seed=None, channels="mix", gpus=None,
                      _messages=()):
        type(self).calls.append((list(inputs), list(outputs), list(mode), channels, gpus, _messages))


def test_cli_passes_gpus_to_restore_files(tmp_path, monkeypatch):
    from voicefixer_b200 import api, __main__ as cli
    assert cli.build_parser().parse_args(["-i", "a.wav"]).gpus == 1
    assert cli.build_parser().parse_args(["-i", "a.wav", "--gpus", "4"]).gpus == 4
    monkeypatch.setattr(api, "VoiceFixer", _StubFixer)
    os.makedirs(tmp_path / "in")
    srcs = [audio_files.write(tmp_path / "in" / n, 3000, 22050, 1, "s16", seed=0) for n in ("a.wav", "b.wav")]
    argv = ["--infolder", str(tmp_path / "in"), "--outfolder", str(tmp_path / "out"), "--gpus", "2"]
    _StubFixer.calls = []
    assert cli.main(argv) == 0
    assert cli.main(argv + ["--mode", "all", "--keep-channels", "--silent"]) == 0
    outs = [str(tmp_path / "out" / n) for n in ("a.wav", "b.wav")]
    alls = [cli._mode_name(o, m) for o in outs for m in (0, 1, 2)]
    assert _StubFixer.calls == [(srcs, outs, [0, 0], "mix", 2, ("processing", "took")),
                                ([s for s in srcs for _ in range(3)], alls, [0, 1, 2] * 2, "keep", 2, ("took",))]
