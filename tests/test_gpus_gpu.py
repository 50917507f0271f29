"""VoiceFixer.restore_files(..., gpus=2) and `python -m voicefixer_b200 --gpus 2` on the GPU, with synthetic checkpoints:
every file they write is byte for byte the file the single-device restore_files writes, a truncated file stops its
own device's shard only, and no worker process outlives a call.

Each case runs on two GPUs when the machine has them ("gpus2", gpus=2 as a user calls it; skipped on one GPU) and as two
processes on device 0 ("one_gpu_two_procs", the tests' _devices=[0, 0]), which takes the same path through the worker
process, the shared-memory weights and the per-shard restore, so it runs on a one-GPU machine too."""
import gc
import multiprocessing
import os

import pytest
import torch

from test_restore_files_gpu import FILES, _bytes, _differ, _folder

pytestmark = pytest.mark.gpu

TWO_GPUS = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices; this machine has "
                              f"{torch.cuda.device_count()}")
PLACES = [pytest.param("gpus2", marks=TWO_GPUS), "one_gpu_two_procs"]


def _kw(place):
    return {"gpus": 2} if place == "gpus2" else {"gpus": 2, "_devices": [0, 0]}


@pytest.fixture(autouse=True)
def _device_memory_back():
    """Hands the device memory of each test's VoiceFixer instances back, before and after it, and checks that no
    worker process is left."""
    def release():
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    release()
    yield
    release()
    assert multiprocessing.active_children() == []


@pytest.fixture()
def home(tmp_path, monkeypatch):
    from voicefixer_b200 import synthetic
    monkeypatch.setenv("HOME", str(tmp_path))
    synthetic.write_checkpoints(str(tmp_path), seed=0)
    return tmp_path


def _outs(root, name, srcs, tag=""):
    os.makedirs(root / name, exist_ok=True)
    return [str(root / name / f"{tag}{k}-{os.path.basename(p)}") for k, p in enumerate(srcs)]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("place", PLACES)
def test_two_devices_write_what_one_writes(home, place):
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine
    vf = VoiceFixer(precision="tf32")
    srcs = _folder(home / "in")
    cases = {                                            # name -> (inputs, restore_files keywords)
        "mode0": (srcs, dict(mode=0)),
        "mode1_waves": (srcs, dict(mode=1, _budget=44100 * 20)),
        "mode2_seeded": ([p for p, f in zip(srcs, FILES) if f[1] >= 1.0], dict(mode=2, dropout_seed=12345)),
        "repeats": ([srcs[k] for k in (1, 1, 3, 4, 3, 7, 3, 9)], dict(mode=[0, 1, 2, 0, 1, 1, 2, 0],
                                                                        dropout_seed=[5, 6, 7, 8, 9, 10, 11, 12])),
        "keep": (srcs, dict(mode=[k % 2 for k in range(len(srcs))], channels="keep")),
    }
    for name, (ins, kw) in cases.items():
        one = _outs(home, name + "-one", ins)
        vf.restore_files(ins, one, **kw)
        two = _outs(home, name + "-two", ins)
        vf.restore_files(ins, two, **kw, **_kw(place))
        assert not _differ(two, one), f"{name}: {_differ(two, one)} differ"
    # an instance made by from_engine (no checkpoint behind it) hands on its engine's weights the same way
    fe = VoiceFixer.from_engine(Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1),
                                       precision="bf16"))
    one, two = _outs(home, "fe-one", srcs), _outs(home, "fe-two", srcs)
    fe.restore_files(srcs, one, mode=1)
    fe.restore_files(srcs, two, mode=1, **_kw(place))
    assert not _differ(two, one), f"from_engine: {_differ(two, one)} differ"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("place", PLACES)
def test_cli_gpus_writes_what_batch_writes(home, monkeypatch, capfd, place):
    from voicefixer_b200 import api
    from voicefixer_b200.__main__ import main
    monkeypatch.setenv("VFX_PRECISION", "tf32")
    if place != "gpus2":                                  # --gpus 2 as two processes on device 0
        real = api.VoiceFixer.restore_files
        monkeypatch.setattr(api.VoiceFixer, "restore_files",
                            lambda self, *a, gpus=None, **k: real(self, *a, gpus=gpus, **k,
                                                                  **({"_devices": [0, 0]} if gpus == 2 else {})))
    wav_files = [f for f in FILES if f[0].endswith(".wav") and 1.0 <= f[1] <= 12.0]  # .wav only; mode 2 needs >= 1 s
    _folder(home / "in", wav_files)
    names = sorted(f[0] for f in wav_files)
    for out, extra in (("batch", ["--batch"]), ("gpus", ["--gpus", "2"])):
        assert main(["--infolder", str(home / "in"), "--outfolder", str(home / out), "--mode", "all", *extra]) == 0
    got = sorted(os.listdir(home / "gpus"))
    assert got == sorted(os.listdir(home / "batch")) and len(got) == 3 * len(names)
    same = [n for n in got if "-mode2" not in n]                                # mode 2 without a seed: random masks
    assert _bytes([home / "gpus" / n for n in same]) == _bytes([home / "batch" / n for n in same])
    out = capfd.readouterr().out
    for n in names:
        for m in (0, 1, 2):
            assert out.count(f"Processing {home / 'in' / n}, mode={m}\n") == 2, (n, m)
    assert out.rstrip().splitlines()[-1].startswith("Done: ")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("place", PLACES)
def test_a_truncated_file_stops_its_own_shard_only(home, place):
    from voicefixer_b200.api import VoiceFixer, plan_devices, _probe_samples
    vf = VoiceFixer(precision="tf32")
    srcs = _folder(home / "in", FILES[:8])
    with open(srcs[2], "r+b") as f:
        f.truncate(20)                                                           # inside the fmt chunk
    outs = _outs(home, "out", srcs)
    shards = plan_devices(_probe_samples(srcs, [0] * len(srcs), False), srcs, 2)
    bad = 0 if 2 in shards[0] else 1
    assert 2 in shards[bad] and shards[1 - bad] and shards[bad].index(2) > 0, shards   # the case this test is about
    with pytest.raises(RuntimeError, match="c.wav"):
        vf.restore_files(srcs, outs, mode=0, **_kw(place))
    written = [i for i in range(len(srcs)) if os.path.exists(outs[i])]
    assert written == sorted(shards[1 - bad] + [i for i in shards[bad] if i < 2]), (shards, written)
    ref = _outs(home, "ref", srcs)
    vf.restore_files([srcs[i] for i in written], [ref[i] for i in written], mode=0)
    assert _bytes([outs[i] for i in written]) == _bytes([ref[i] for i in written])


@pytest.mark.timeout(600)
def test_one_gpu_is_the_default_path_and_more_gpus_than_devices_are_refused(home):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer(precision="tf32")
    srcs = _folder(home / "in", FILES[:4])
    one, dflt = _outs(home, "one", srcs), _outs(home, "default", srcs)
    vf.restore_files(srcs, dflt, mode=1)
    vf.restore_files(srcs, one, mode=1, gpus=1)
    assert _bytes(one) == _bytes(dflt)
    n = torch.cuda.device_count()
    with pytest.raises(ValueError, match=f"gpus={n + 1}, but {n} CUDA device"):
        vf.restore_files(srcs, one, gpus=n + 1)
