"""CPU tests of the host logic and of the C-ABI surface (no compute calls without a GPU)."""
import os
import re
import wave
import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from voicefixer_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vfx_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(vfx_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/vfx_b200.h but not exported"
    assert declared == set(_lib.SIGNATURES), "ctypes signatures out of sync with the header"
    assert lib.vfx_version() >= 100


def test_conv_desc_layout_matches_header():
    """ctypes mirror of struct vfx_conv_desc has the same field order as the header."""
    from voicefixer_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vfx_b200.h")).read()
    body = re.search(r"typedef struct vfx_conv_desc \{(.*?)\} vfx_conv_desc;", hdr, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for stmt in body.split(";"):
        stmt = stmt.strip()
        if not stmt:
            continue
        decl = re.sub(r"^(const\s+)?(void|float|int|long long)\s*\*?", "", stmt).strip()
        for part in decl.split(","):
            names.append(re.sub(r"\[.*\]", "", part).replace("*", "").strip())
    assert names == [f[0] for f in _lib.ConvDesc._fields_]


def test_engine_refuses_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from voicefixer_b200.engine import Engine
    with pytest.raises(RuntimeError, match="no CPU path"):
        Engine({}, {})


def test_weight_packing_shapes(states):
    from voicefixer_b200 import weights
    from voicefixer_b200.engine import Engine
    pa = weights.pack_analysis(states[0], "fp32")
    pv = weights.pack_vocoder(states[1], "bf16")
    assert tuple(pa["unet.enc1.b1.conv1.w"].shape) == (9, 32, 2)
    pb = weights.pack_analysis(states[0], "bf16")              # bf16: Cin 2 zero-padded to 32 operand channels
    assert tuple(pb["unet.enc1.b1.conv1.w"].shape) == (9, 32, 32) and tuple(pb["unet.enc1.b1.sc.w"].shape) == (32, 32)
    assert float(pb["unet.enc1.b1.conv1.w"][:, :, 2:].abs().max()) == 0.0
    assert tuple(pa["unet.dec1.up.w"].shape) == (9, 384, 384)
    assert tuple(pa["dn.g7.l0.whh_t"].shape) == (2, 256, 768)
    assert tuple(pv["voc.up0.w"].shape) == (14, 512, 1024) and pv["voc.up0.w"].dtype == torch.bfloat16
    assert tuple(pv["voc.rs3.l7.c2.w"].shape) == (3, 64, 64)
    assert tuple(pv["voc.post.w"].shape) == (7, 64) and pv["voc.post.w"].dtype == torch.float32
    # mel filterbank band table covers every non-zero
    fbT = pa["fe.fbT"]
    for m in (0, 1, 64, 127):
        s, n = int(pa["fe.fb_start"][m]), int(pa["fe.fb_len"][m])
        mask = torch.zeros(1025, dtype=torch.bool); mask[s:s + n] = True
        assert torch.all(fbT[m][~mask] == 0)
    table, total = Engine.layout({**pa, **pv})
    assert all(off % 256 == 0 for _, off, _ in table) and total > 3e8
    # weight-norm fold and both key layouts agree
    from voicefixer_b200 import synthetic
    old = synthetic.make_vocoder_state(1, old_style_keys=True)
    pv2 = weights.pack_vocoder(old, "fp32")
    pv1 = weights.pack_vocoder(states[1], "fp32")
    assert torch.equal(pv1["voc.rs0.l3.c1.w"], pv2["voc.rs0.l3.c1.w"])
    w = pv1["voc.up2.w"]        # ConvTranspose1d: norm over dims (1,2) per IN channel == g
    g = states[1]["generator.9.layer.parametrizations.weight.original0"].reshape(-1)
    assert torch.allclose(w.permute(2, 1, 0).pow(2).sum((1, 2)).sqrt(), g, rtol=1e-4)


def test_stft_kernel_check_rejects_foreign_window(states):
    from voicefixer_b200 import weights
    bad = dict(states[0])
    bad["f_helper.stft.conv_real.weight"] = torch.ones(1025, 1, 2048)
    with pytest.raises(ValueError, match="Hann"):
        weights.check_stft_kernels(bad)


def test_missing_checkpoints_raise_reference_errors(tmp_path, monkeypatch):
    monkeypatch.setenv("HOME", str(tmp_path))
    from voicefixer_b200 import api
    with pytest.raises(RuntimeError, match="Error 1"):
        api.VoiceFixer()
    with pytest.raises(RuntimeError, match="Error 1"):
        api.Vocoder(44100)
    with pytest.raises(RuntimeError, match="only support 44100"):
        api.Vocoder(16000)
    os.makedirs(tmp_path / ".cache/voicefixer/synthesis_module/44100")
    torch.save({"generator": {}}, tmp_path / api.VOCODER_CKPT)
    with pytest.raises(RuntimeError, match="Error 0"):
        api.VoiceFixer()


def test_wav_io_roundtrip_and_int16_truncation(tmp_path):
    from voicefixer_b200 import wavio
    x = np.array([[0.0, 0.5, -0.5, 0.99997, -1.0, 1.5 / 32768, -1.5 / 32768]], dtype=np.float32)
    p = tmp_path / "a.wav"
    wavio.save_wave(x, str(p), 44100)
    with wave.open(str(p), "rb") as f:
        assert f.getnchannels() == 1 and f.getframerate() == 44100 and f.getsampwidth() == 2
        pcm = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2")
    assert pcm.tolist() == [0, 16384, -16384, 32767, -32768, 1, -1]      # astype(np.short): toward zero
    y = wavio.load_mono(str(p), 44100)
    assert y.dtype == np.float32 and y.shape == (7,) and abs(y[1] - 0.5) < 1e-4
    with pytest.raises(RuntimeError, match="not a readable FLAC stream"):
        (tmp_path / "x.flac").write_bytes(b"RIFF....WAVEfmt " + bytes(64))
        wavio.load_mono(str(tmp_path / "x.flac"))


def test_segmentation_matches_reference_loop():
    """The while-loop at voicefixer/base.py:117-137 cuts [0,30s), [30s,60s), ... + ragged tail."""
    from voicefixer_b200.api import SEG_LENGTH
    for n in (1, SEG_LENGTH - 1, SEG_LENGTH, SEG_LENGTH + 1, 3 * SEG_LENGTH + 5):
        segs, bp = [], SEG_LENGTH
        while bp < n + SEG_LENGTH:
            segs.append((max(bp - SEG_LENGTH, 0), min(bp, n)))
            bp += SEG_LENGTH
        assert segs[0][0] == 0 and segs[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(segs, segs[1:]))
        assert len(segs) == (n + SEG_LENGTH - 1) // SEG_LENGTH


def test_oracle_conditions_match_oracle_module():
    from voicefixer_b200.api import oracle_conditions
    from oracle import vf_oracle as O
    wav = (np.random.RandomState(5).randn(9000) * 0.1).astype(np.float32)
    a = oracle_conditions(wav)                                  # (1, Tc, 128) channels-last
    b = O.oracle_cond(wav).numpy()                              # (1, 128, Tc)
    assert a.shape == (1, b.shape[2], 128)
    assert np.max(np.abs(a - b.transpose(0, 2, 1))) < 1e-4


def test_cli_job_planning_matches_reference_naming(tmp_path):
    """voicefixer/__main__.py:13-19,147-213: `--mode all` -> <name>-mode<k><ext>; only .wav inputs; folder mode."""
    from voicefixer_b200.__main__ import build_parser, plan_jobs
    (tmp_path / "in").mkdir()
    for n in ("a.wav", "b.wav", "c.txt"):
        (tmp_path / "in" / n).write_bytes(b"")
    args = build_parser().parse_args(["-i", str(tmp_path / "in" / "a.wav"), "-o", str(tmp_path / "o" / "r.wav"), "--mode", "all"])
    jobs = plan_jobs(args)
    assert [os.path.basename(j[1]) for j in jobs] == ["r-mode0.wav", "r-mode1.wav", "r-mode2.wav"] and [j[2] for j in jobs] == [0, 1, 2]
    args = build_parser().parse_args(["--infolder", str(tmp_path / "in"), "--outfolder", str(tmp_path / "out"), "--mode", "1"])
    jobs = plan_jobs(args)
    assert [os.path.basename(j[0]) for j in jobs] == ["a.wav", "b.wav"] and all(j[2] == 1 for j in jobs)
    assert os.path.basename(jobs[0][1]) == "a.wav"
    with pytest.raises(AssertionError, match="--infile"):
        plan_jobs(build_parser().parse_args([]))
    with pytest.raises(AssertionError, match="not found"):
        plan_jobs(build_parser().parse_args(["-i", str(tmp_path / "nope.wav")]))
    with pytest.raises(AssertionError, match="Unsupported output format"):
        plan_jobs(build_parser().parse_args(["-i", str(tmp_path / "in" / "a.wav"), "-o", "x.mp3"]))
    jobs = plan_jobs(build_parser().parse_args(["-i", str(tmp_path / "in" / "a.wav"), "-o", "x.flac"]))   # soundfile format
    assert jobs == [(str(tmp_path / "in" / "a.wav"), "x.flac", 0)]
    with pytest.raises(ValueError, match="only support the .wav"):
        plan_jobs(build_parser().parse_args(["-i", str(tmp_path / "in" / "c.txt"), "-o", "x.wav"]))


def test_header_is_valid_c99():
    """include/vfx_b200.h is the C ABI: it must compile as plain C, not only as C++."""
    import shutil, subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    r = subprocess.run([gcc, "-std=c99", "-fsyntax-only", "-x", "c", os.path.join(ROOT, "include", "vfx_b200.h")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_voicefixer_alias_package_resolves_to_b200_classes():
    import voicefixer
    from voicefixer_b200 import api
    assert voicefixer.VoiceFixer is api.VoiceFixer and voicefixer.Vocoder is api.Vocoder
    with pytest.raises(AttributeError):
        voicefixer.NoSuchThing


def test_wav_loader_mono_mix_and_resample(tmp_path):
    """librosa.load(path, sr=44100) semantics used by VoiceFixer._load_wav: mean over channels, resample to 44.1 kHz."""
    from voicefixer_b200 import wavio
    sr = 22050
    t = np.arange(sr // 2) / sr
    left, right = 0.5 * np.sin(2 * np.pi * 440 * t), 0.25 * np.sin(2 * np.pi * 440 * t)
    pcm = (np.stack([left, right], 1) * 32767).astype("<i2")
    with wave.open(str(tmp_path / "st.wav"), "wb") as f:
        f.setnchannels(2); f.setsampwidth(2); f.setframerate(sr); f.writeframes(pcm.tobytes())
    y = wavio.load_mono(str(tmp_path / "st.wav"), 44100)
    assert y.dtype == np.float32 and abs(len(y) - 22050) <= 2
    t2 = np.arange(len(y)) / 44100.0
    ref = 0.375 * np.sin(2 * np.pi * 440 * t2)
    assert np.max(np.abs(y[500:-500] - ref[500:-500])) < 5e-3
    x2 = wavio.read_wave(str(tmp_path / "st.wav"), 44100)
    assert x2.shape[1] == 2 and abs(x2.shape[0] - 22050) <= 2


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_planning_only_engine_validates_weight_sets_and_sizes_workspace(states, precision):
    """vfx_engine_create(device=-1): finalize + workspace planning without a GPU.  The 20 x 30 s bf16 figure is the
    workspace a GPU run of the same batch allocates (17.168495616 GB): a change to the launch sequence's buffers shows here."""
    import ctypes
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import Planner
    from voicefixer_b200.weights import pack_analysis, pack_vocoder
    voc = pack_vocoder(states[1], precision)
    full = dict(pack_analysis(states[0], precision), **voc)
    pl = Planner(full, precision)
    if precision == "bf16":
        assert pl.workspace_bytes(20, 44100 * 30) == 17168495616
    small, big = pl.workspace_bytes(1, 44100), pl.workspace_bytes(8, 441000)
    assert 0 < small < big and pl.workspace_bytes(8, 441000) == big            # deterministic
    assert pl.workspace_bytes(1, 1024) == 0 and pl.workspace_bytes(0, 44100) == 0
    # the reference's stand-alone Vocoder (vocoder/base.py:10-40) loads the synthesis checkpoint only
    pv = Planner(voc, precision)
    assert pv.workspace_bytes(1, 44100) == 0                                   # restore() needs the analysis module
    assert 0 < pv.workspace_bytes_frames(2, 101) <= pl.workspace_bytes_frames(2, 101)
    # incomplete or inconsistent weight sets are named, not guessed at
    bad = dict(full); del bad["unet.head.w"]
    with pytest.raises(_lib.VfxError, match=r"missing weight tensors: unet\.head\.w"):
        Planner(bad, precision)
    k = sorted(voc)[5]
    bad = dict(voc); del bad[k]
    with pytest.raises(_lib.VfxError, match="missing weight tensors: " + k.replace(".", r"\.")):
        Planner(bad, precision)
    bad = dict(voc); bad[k] = voc[k].reshape(-1)[:-1]
    with pytest.raises(_lib.VfxError, match="engine expects"):
        Planner(bad, precision)
    bad = dict(voc); bad["dn.bn0.beta"] = full["dn.bn0.beta"]                  # vocoder + a stray analysis tensor
    with pytest.raises(_lib.VfxError, match="missing weight tensors: dn"):
        Planner(bad, precision)
    # a planning-only engine never launches: every compute entry point refuses before touching CUDA
    lib, one = _lib.load(), ctypes.c_void_p(4096)
    rc = lib.vfx_restore(pl.h, one, 1, 44100, 0, None, one, one, 1 << 30, None)
    assert rc == -1 and b"planning-only" in lib.vfx_last_error()
    rc = lib.vfx_vocoder(pv.h, one, 1, 8, 0, one, -1, 1.0, one, 1 << 30, None)
    assert rc == -1 and b"planning-only" in lib.vfx_last_error()


def test_cli_per_file_runs_one_job_per_wave_through_run_waves(tmp_path, monkeypatch, capsys):
    """execute(batch=False) is run_waves with budget 0: each job a wave of its own, an input that the job before also
    read (--mode all) decoded once, `Processing` through say and `Restoration took` through print (--silent keeps it),
    outputs written in job order.  The pipeline's overlap, order and error rules are tested on run_waves itself."""
    from voicefixer_b200 import api, wavio, __main__ as cli
    calls, waves = [], []
    run_waves = api.run_waves

    def spy(srcs, budget, load, restore, write):
        calls.append(("run_waves", list(srcs), budget))
        return run_waves(srcs, budget, load, restore, lambda ids, out: (waves.append(ids), write(ids, out)))

    class StubFixer:
        def _load_wav(self, path, sample_rate):
            calls.append(("load", os.path.basename(path), sample_rate))
            return wavio.load_mono(path, sample_rate)

        def restore_inmem(self, wav, cuda=False, mode=0):
            calls.append(("restore", len(wav), cuda, mode))
            return wav[None] * (0.25 * (mode + 1))

    monkeypatch.setattr(api, "run_waves", spy)
    rng = np.random.default_rng(1)
    srcs = [str(tmp_path / f"in{k}.wav") for k in range(2)]
    for k, src in enumerate(srcs):
        wavio.save_wave((0.5 * rng.standard_normal((1, 3000 + k))).clip(-1, 1).astype(np.float32), src)
    jobs = [(srcs[0], str(tmp_path / f"a{m}.wav"), m) for m in (0, 1, 2)] + [(srcs[1], str(tmp_path / "b.wav"), 1)]
    for say in (print, lambda *a: None):                                         # default, then --silent
        del calls[:], waves[:]
        cli.execute(StubFixer(), jobs, batch=False, cuda=False, say=say)
        assert calls[0] == ("run_waves", [j[0] for j in jobs], 0) and waves == [[0], [1], [2], [3]]
        assert [c for c in calls if c[0] == "load"] == [("load", "in0.wav", 44100), ("load", "in1.wav", 44100)]
        assert [c for c in calls if c[0] == "restore"] == [("restore", 3000 + (j[0] == srcs[1]), False, j[2])
                                                           for j in jobs]
        took, lines = "Restoration took 0.0 s", capsys.readouterr().out.splitlines()
        if say is print:
            assert lines == [x for src, _, m in jobs for x in ("Processing {}, mode={}".format(src, m), took)]
        else:
            assert lines == [took] * 4
        for src, dst, m in jobs:
            wavio.save_wave(wavio.load_mono(src)[None] * (0.25 * (m + 1)), tmp_path / "want.wav")
            assert open(dst, "rb").read() == (tmp_path / "want.wav").read_bytes()
    calls.clear()
    cli.execute(StubFixer(), [], batch=False)                                   # no jobs: nothing is read or restored
    assert calls == [("run_waves", [], 0)] and capsys.readouterr().out == ""


def test_cli_main_wiring_folder_mode_all_with_flac_output(tmp_path, monkeypatch, capsys):
    """`python -m voicefixer_b200` end to end on the host side (decode -> [GPU stage stubbed] -> encode): file naming of
    --mode all, FLAC / WAV by extension, messages.  The GPU stage itself is covered by the -m gpu tests."""
    from voicefixer_b200 import api, wavio, __main__ as cli

    class StubFixer:
        def _load_wav(self, path, sample_rate):
            return wavio.load_mono(path, sample_rate)

        def restore_inmem(self, wav, cuda=False, mode=0):
            return (wav[: 512 * (len(wav) // 512)] if mode == 1 else wav)[None] * 0.5      # (1, N) float32

    monkeypatch.setattr(api, "VoiceFixer", StubFixer)
    rng = np.random.default_rng(0)
    os.makedirs(tmp_path / "in")
    for name, n in (("a.wav", 5000), ("b.wav", 7000)):
        wavio.save_wave((0.5 * rng.standard_normal((1, n))).clip(-1, 1).astype(np.float32), str(tmp_path / "in" / name))
    assert cli.main(["--infolder", str(tmp_path / "in"), "--outfolder", str(tmp_path / "out"), "--mode", "all"]) == 0
    assert sorted(os.listdir(tmp_path / "out")) == [f"{s}-mode{m}.wav" for s in "ab" for m in (0, 1, 2)]
    a = wavio.load_mono(str(tmp_path / "in" / "a.wav"))
    assert np.allclose(wavio.load_mono(str(tmp_path / "out" / "a-mode0.wav")), a * 0.5, atol=1 / 32768)
    assert wavio.load_mono(str(tmp_path / "out" / "a-mode1.wav")).shape == (512 * (5000 // 512),)
    out = capsys.readouterr().out
    assert out.count("Restoration took") == 6 and "Initializing VoiceFixer" in out and "mode=2" in out
    assert cli.main(["-i", str(tmp_path / "in" / "b.wav"), "-o", str(tmp_path / "x" / "b.flac"), "--silent"]) == 0
    assert (tmp_path / "x" / "b.flac").read_bytes()[:4] == b"fLaC"
    assert wavio.load_mono(str(tmp_path / "x" / "b.flac")).shape == (7000,)


def test_wav_reader_formats_beyond_stdlib_wave(tmp_path):
    """librosa.load accepts float and WAVE_FORMAT_EXTENSIBLE files; stdlib `wave` rejects them.  All decode to the same
    float32 samples (to the format's resolution), extra chunks and odd padding are skipped."""
    import struct
    from voicefixer_b200 import wavio
    rng = np.random.default_rng(2)
    x = np.clip(0.4 * rng.standard_normal((1000, 2)), -0.999, 0.999)

    def riff(tag, bits, payload, extensible=False, extra=b"", data_size=None):
        nch, sr = 2, 44100
        block = nch * bits // 8
        if extensible:
            fmt = struct.pack("<HHIIHHHHIH14s", 0xFFFE, nch, sr, sr * block, block, bits, 22, bits, 3, tag,
                              bytes.fromhex("000000001000800000aa00389b71"))
        else:
            fmt = struct.pack("<HHIIHH", tag, nch, sr, sr * block, block, bits)
        body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + extra
        body += b"data" + struct.pack("<I", len(payload) if data_size is None else data_size) + payload
        return b"RIFF" + struct.pack("<I", len(body)) + body

    i24 = np.round(x * 8388607).astype(np.int32)
    b24 = np.stack([(i24 >> s) & 0xFF for s in (0, 8, 16)], axis=-1).astype(np.uint8).tobytes()
    cases = {
        "f32": (riff(3, 32, x.astype("<f4").tobytes()), 1e-7),
        "f64": (riff(3, 64, x.astype("<f8").tobytes()), 1e-7),
        "f32ext": (riff(3, 32, x.astype("<f4").tobytes(), extensible=True), 1e-7),
        "i16ext": (riff(1, 16, np.round(x * 32767).astype("<i2").tobytes(), extensible=True), 1e-4),
        "i24": (riff(1, 24, b24), 1e-6),
        "i32": (riff(1, 32, np.round(x * 2147483647).astype("<i4").tobytes()), 1e-6),
        "u8": (riff(1, 8, np.round(x * 127 + 128).astype(np.uint8).tobytes()), 2e-2),
        "list_chunk": (riff(3, 32, x.astype("<f4").tobytes(), extra=b"LIST" + struct.pack("<I", 5) + b"abcde\x00"), 1e-7),
        "streamed": (riff(3, 32, x.astype("<f4").tobytes(), data_size=0xFFFFFFFF), 1e-7),
    }
    for name, (blob, tol) in cases.items():
        p = tmp_path / f"{name}.wav"
        p.write_bytes(blob)
        y = wavio.read_wave(str(p), 44100)
        assert y.dtype == np.float32 and y.shape == (1000, 2) and np.abs(y - x).max() < tol, name
        assert wavio.load_mono(str(p)).shape == (1000,)
    (tmp_path / "bad.wav").write_bytes(riff(2, 4, bytes(100)))                 # ADPCM
    with pytest.raises(RuntimeError, match="unsupported WAVE format"):
        wavio.load_mono(str(tmp_path / "bad.wav"))
    (tmp_path / "junk.wav").write_bytes(b"OggS" + bytes(64))
    with pytest.raises(RuntimeError, match="not a RIFF/WAVE"):
        wavio.load_mono(str(tmp_path / "junk.wav"))


# ---------------------------------------------------------------------------- restore_stream windowing (no GPU: fake engine)
class _EchoEngine:
    """Stands in for the CUDA engine: restore() returns its input and records the window lengths."""
    device = 0
    arena = None

    def __init__(self):
        self.windows = []

    def restore(self, x, mode=0):
        self.windows.append(int(x.shape[1]))
        return x.clone()


def _stream_vf(monkeypatch):
    import torch
    from voicefixer_b200 import api
    monkeypatch.setattr(api, "_check_cuda", lambda cuda: None)
    real_to = torch.Tensor.to
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self if (a and isinstance(a[0], str) and a[0].startswith("cuda")) else real_to(self, *a, **k))
    eng = _EchoEngine()
    return api.VoiceFixer.from_engine(eng), eng


@pytest.mark.parametrize("n,blk,chunk,ctx", [(200000, 4410, 1.0, 0.5), (200000, 100000, 1.0, 0.0), (44100 * 3 + 17, 999, 0.5, 0.25),
                                             (50000, 50000, 2.0, 1.0), (1500, 700, 1.0, 1.0)])
def test_restore_stream_covers_the_input_exactly_once(monkeypatch, n, blk, chunk, ctx):
    """With an identity engine the concatenated stream output must be the input: every sample emitted exactly once, in
    order, whatever the block sizes; no window shorter than the front end's reflect pad allows."""
    vf, eng = _stream_vf(monkeypatch)
    rs = np.random.RandomState(0)
    x = rs.randn(n).astype(np.float32)
    out = list(vf.restore_stream((x[i:i + blk] for i in range(0, n, blk)), chunk_seconds=chunk, context_seconds=ctx))
    y = np.concatenate(out)
    assert y.shape == x.shape and np.array_equal(y, x)
    assert min(eng.windows) > 1024
    C, X = int(round(chunk * 44100)), int(round(ctx * 44100))
    assert max(eng.windows) <= C + 2 * X or n <= C + 2 * X
    full = [w for w in eng.windows if w == C + 2 * X]
    assert len(full) >= max(0, (n - X) // C - 2)                       # steady state: fixed-size windows


def test_restore_stream_30s_windows_are_the_reference_segments(monkeypatch):
    """chunk 30 s, no context: the windows are exactly restore_inmem's segments (voicefixer/base.py:116-119)."""
    vf, eng = _stream_vf(monkeypatch)
    n = 44100 * 65 + 123
    x = np.zeros(n, np.float32)
    out = list(vf.restore_stream([x[:1000000], x[1000000:]], chunk_seconds=30.0, context_seconds=0.0))
    assert eng.windows == [44100 * 30, 44100 * 30, 44100 * 5 + 123]
    assert [len(o) for o in out] == eng.windows
    with pytest.raises(ValueError):
        list(vf.restore_stream([x], chunk_seconds=0))
