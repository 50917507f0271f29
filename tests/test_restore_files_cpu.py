"""VoiceFixer.restore_files and `--batch` without a GPU: the wave planner, the native-rate reader it decodes with, the
reader -> GPU -> writer pipeline with fake stages, and the command line's wiring."""
import os
import threading
import time

import numpy as np
import pytest

import audio_files


# ---------------------------------------------------------------------------- plan_waves
def _waves(lengths, budget):
    from voicefixer_b200.api import plan_waves
    return list(plan_waves(lengths, budget))


@pytest.mark.parametrize("seed", range(6))
def test_plan_waves_keeps_order_covers_every_file_and_respects_the_budget(seed):
    rng = np.random.default_rng(seed)
    lengths = [int(v) for v in rng.integers(1, 5000, size=int(rng.integers(1, 60)))]
    budget = int(rng.integers(1000, 20000))
    waves = _waves(lengths, budget)
    assert [i for w in waves for i in w] == list(range(len(lengths)))           # in order, each file exactly once
    for k, w in enumerate(waves):
        assert w == list(range(w[0], w[-1] + 1))                                # consecutive runs
        total = sum(lengths[i] for i in w)
        assert total <= budget or len(w) == 1                                   # over budget only alone
        if k + 1 < len(waves):                                                  # greedy: the next file did not fit
            assert total + lengths[waves[k + 1][0]] > budget


def test_plan_waves_puts_an_oversize_file_alone():
    assert _waves([10, 100, 10, 10], 50) == [[0], [1], [2, 3]]
    assert _waves([100], 50) == [[0]]
    assert _waves([60, 60, 60], 50) == [[0], [1], [2]]


def test_plan_waves_budget_edges():
    assert _waves([], 100) == []
    assert _waves([25, 25, 25, 25], 100) == [[0, 1, 2, 3]]                      # exactly the budget
    assert _waves([25, 25, 25, 26], 100) == [[0, 1, 2], [3]]                    # one sample over
    assert _waves([1, 1, 1], 0) == [[0], [1], [2]]                              # no budget: one file per wave
    assert _waves([5, 5, 5], 10 ** 12) == [[0, 1, 2]]


def test_plan_waves_reads_lengths_lazily():
    """A wave is yielded once the first length past it is known, so the reader decodes at most one file ahead."""
    from voicefixer_b200.api import plan_waves
    seen = []

    def lengths():
        for n in (40, 40, 40, 40):
            seen.append(n)
            yield n

    gen = plan_waves(lengths(), 80)
    assert next(gen) == [0, 1] and len(seen) == 3
    assert next(gen) == [2, 3] and len(seen) == 4


# ---------------------------------------------------------------------------- load_mono_native
CASES = ([(fmt, 2, 44100) for fmt in audio_files.FORMATS] + [("s16", 1, 44100), ("s16", 6, 44100), ("flac", 6, 48000)]
         + [(fmt, ch, sr) for sr in (16000, 22050, 48000) for fmt, ch in (("s16", 1), ("f32", 2), ("flac", 2))])


@pytest.mark.parametrize("fmt,channels,sr", CASES)
def test_load_mono_native_then_resample_is_load_mono(tmp_path, fmt, channels, sr):
    from voicefixer_b200 import wavio
    ext = ".flac" if fmt == "flac" else ".wav"
    p = audio_files.write(tmp_path / f"a{ext}", 3001, sr, channels, fmt, seed=channels + sr)
    x, got_sr = wavio.load_mono_native(p)
    assert got_sr == sr and x.dtype == np.float32 and x.shape == (3001,)
    pcm, _ = wavio._read_pcm(p)
    assert np.array_equal(x, pcm.mean(axis=1).astype(np.float32))              # the mix load_mono always made
    y = wavio._resample(x, got_sr, 44100)
    want = wavio.load_mono(p)
    assert y.dtype == want.dtype and np.array_equal(y, want)


# ---------------------------------------------------------------------------- run_waves with fake stages
def _pipeline(srcs, budget, fail_load=None, fail_restore=None, fail_write=None, delay=0.0):
    """run_waves with fake stages; returns (log, result or exception)."""
    from voicefixer_b200.api import run_waves
    log, lock = [], threading.Lock()

    def rec(*a):
        with lock:
            log.append(a)

    def load(i, prev):
        if prev is None:
            time.sleep(delay)
            if srcs[i] == fail_load:
                raise RuntimeError(f"restore_files: {srcs[i]}: cannot read")
            rec("read", srcs[i])
            prev = srcs[i] + ":pcm"
        return prev, 10

    def restore(wave):
        time.sleep(delay)
        if any(srcs[i] == fail_restore for i, _ in wave):
            raise RuntimeError("device fault")
        rec("gpu", [i for i, _ in wave])
        return {i: item + ":restored" for i, item in wave}

    def write(ids, result):
        time.sleep(delay)
        for i in ids:
            if f"out{i}" == fail_write:
                raise RuntimeError(f"restore_files: out{i}: disk full")
            rec("write", f"out{i}", result[i])

    try:
        return log, run_waves(srcs, budget, load, restore, write)
    except Exception as e:                                                  # noqa: BLE001
        return log, e


def _written(log):
    return [e[1] for e in log if e[0] == "write"]


def test_run_waves_overlaps_stages_and_keeps_order():
    srcs = [f"in{i}" for i in range(6)] + ["in5"]                              # in5 twice (two modes)
    for budget, gpu in ((20, [[0, 1], [2, 3], [4, 5], [6]]),
                        (0, [[i] for i in range(7)])):                          # the command line's one file per wave
        t0 = time.time()
        log, waves = _pipeline(srcs, budget, delay=0.05)
        wall = time.time() - t0
        assert waves == len(gpu)
        assert [e[1] for e in log if e[0] == "gpu"] == gpu
        assert _written(log) == [f"out{i}" for i in range(7)]
        assert ("write", "out6", "in5:pcm:restored") in log
        assert [e[1] for e in log if e[0] == "read"] == srcs[:6]                # in5 decoded once
        assert wall < 0.85 * (6 + 2 * len(gpu)) * 0.05                          # the stages overlap


def test_run_waves_decodes_an_input_once_per_wave():
    log, waves = _pipeline(["a", "a", "a", "b", "b", "a"], budget=30)
    assert waves == 2                                                           # [0, 1, 2] [3, 4, 5]
    assert [e[1] for e in log if e[0] == "read"] == ["a", "b", "a"]
    assert _written(log) == [f"out{i}" for i in range(6)]
    log, waves = _pipeline(["a", "a", "b"], budget=0)                          # one job per wave: the reader still
    assert waves == 3                                                           # holds the job before when it loads
    assert [e[1] for e in log if e[0] == "read"] == ["a", "b"]


@pytest.mark.parametrize("budget", [0, 10, 30, 1000])
def test_run_waves_failing_read_keeps_the_files_before_it(budget):
    srcs = [f"in{i}" for i in range(7)]
    log, err = _pipeline(srcs, budget, fail_load="in4")
    assert isinstance(err, RuntimeError) and "in4" in str(err)
    assert _written(log) == ["out0", "out1", "out2", "out3"]                   # its wave is cut short, not dropped
    assert "in5" not in [e[1] for e in log if e[0] == "read"]                  # nothing after it is started


def test_run_waves_failing_restore_fails_its_wave_only():
    srcs = [f"in{i}" for i in range(7)]
    for budget, written in ((20, ["out0", "out1"]),                            # waves [0, 1] [2, 3] ...
                            (0, ["out0", "out1", "out2"])):                     # one file per wave
        log, err = _pipeline(srcs, budget, fail_restore="in3")
        assert isinstance(err, RuntimeError) and "device fault" in str(err)
        assert _written(log) == written
        assert not any(e[0] == "gpu" and 4 in e[1] for e in log)


@pytest.mark.parametrize("budget", [0, 10, 1000])
def test_run_waves_failing_write_keeps_the_files_before_it(budget):
    srcs = [f"in{i}" for i in range(7)]
    log, err = _pipeline(srcs, budget, fail_write="out3")
    assert isinstance(err, RuntimeError) and "out3" in str(err)
    assert _written(log) == ["out0", "out1", "out2"]


def test_run_waves_threads_exit():
    before = {t.ident for t in threading.enumerate()}
    for budget in (0, 20):
        for kw in ({}, {"fail_load": "in2"}, {"fail_restore": "in2"}, {"fail_write": "out2"}):
            _pipeline([f"in{i}" for i in range(5)], budget, **kw)
    assert not [t for t in threading.enumerate() if t.ident not in before and t.name.startswith("vfx-wave")]


# ---------------------------------------------------------------------------- restore_files' own checks
def _vf(monkeypatch):
    from voicefixer_b200 import api

    class _Eng:
        device = 0

    monkeypatch.setattr(api, "_check_cuda", lambda cuda: None)
    return api.VoiceFixer.from_engine(_Eng())


def test_restore_files_refuses_bad_lists_before_reading(monkeypatch, tmp_path):
    from voicefixer_b200 import wavio
    vf = _vf(monkeypatch)
    monkeypatch.setattr(wavio, "load_mono_native", lambda p: pytest.fail("read before the arguments were checked"))
    with pytest.raises(ValueError, match="non-empty"):
        vf.restore_files([], [])
    with pytest.raises(ValueError, match="2 inputs and 1 outputs"):
        vf.restore_files(["a.wav", "b.wav"], ["x.wav"])
    with pytest.raises(ValueError, match="mode has 3 entries for 2 files"):
        vf.restore_files(["a.wav", "b.wav"], ["x.wav", "y.wav"], mode=[0, 1, 2])
    with pytest.raises(ValueError, match="file 1 has mode 3"):
        vf.restore_files(["a.wav", "b.wav"], ["x.wav", "y.wav"], mode=[0, 3])
    with pytest.raises(ValueError, match="no file is restored in mode 2"):
        vf.restore_files(["a.wav"], ["x.wav"], mode=1, dropout_seed=5)
    with pytest.raises(ValueError, match="recording 1 has dropout_seed -1"):
        vf.restore_files(["a.wav", "b.wav"], ["x.wav", "y.wav"], mode=2, dropout_seed=[3, -1])


# ---------------------------------------------------------------------------- the command line
class _StubFixer:
    calls = []

    def restore_files(self, inputs, outputs, mode=0, cuda=True, dropout_seed=None, _on_wave=None, _on_wave_done=None):
        type(self).calls.append((list(inputs), list(outputs), list(mode), cuda))
        _on_wave(list(range(len(inputs))))
        _on_wave_done(list(range(len(inputs))), 0.25)

    def restore_inmem(self, *a, **k):
        pytest.fail("--batch ran the per-file path")


@pytest.mark.parametrize("mode", ["0", "1", "all"])
def test_cli_batch_passes_plan_jobs_list_to_restore_files(tmp_path, monkeypatch, capsys, mode):
    from voicefixer_b200 import api, __main__ as cli
    monkeypatch.setattr(api, "VoiceFixer", _StubFixer)
    _StubFixer.calls = []
    os.makedirs(tmp_path / "in")
    for name in ("b.wav", "a.wav", "c.flac"):
        (tmp_path / "in" / name).write_bytes(b"")
    argv = ["--infolder", str(tmp_path / "in"), "--outfolder", str(tmp_path / "out"), "--mode", mode]
    jobs = cli.plan_jobs(cli.build_parser().parse_args(argv))
    assert cli.main(argv + ["--batch"]) == 0
    assert _StubFixer.calls == [([j[0] for j in jobs], [j[1] for j in jobs], [j[2] for j in jobs], True)]
    assert len(jobs) == (6 if mode == "all" else 2)
    out = capsys.readouterr().out
    for src, _, m in jobs:
        assert "Processing {}, mode={}".format(src, m) in out
    assert out.count("Restoration took 0.2 s") == 1 and "Done: {} job(s)".format(len(jobs)) in out
    assert os.path.isdir(tmp_path / "out")                                      # output folder made, as without --batch


def test_cli_batch_infile_mode_all(tmp_path, monkeypatch):
    from voicefixer_b200 import api, __main__ as cli
    monkeypatch.setattr(api, "VoiceFixer", _StubFixer)
    _StubFixer.calls = []
    (tmp_path / "a.wav").write_bytes(b"")
    assert cli.main(["-i", str(tmp_path / "a.wav"), "-o", str(tmp_path / "r.flac"), "--mode", "all", "--batch",
                     "--disable-cuda", "--silent"]) == 0
    [(ins, outs, modes, cuda)] = _StubFixer.calls
    assert ins == [str(tmp_path / "a.wav")] * 3 and modes == [0, 1, 2] and cuda is False
    assert outs == [str(tmp_path / f"r-mode{m}.flac") for m in (0, 1, 2)]


def test_cli_batch_on_an_empty_folder_runs_nothing(tmp_path, monkeypatch):
    from voicefixer_b200 import api, __main__ as cli
    monkeypatch.setattr(api, "VoiceFixer", _StubFixer)
    _StubFixer.calls = []
    os.makedirs(tmp_path / "in")
    assert cli.main(["--infolder", str(tmp_path / "in"), "--outfolder", str(tmp_path / "o"), "--batch"]) == 0
    assert _StubFixer.calls == []
