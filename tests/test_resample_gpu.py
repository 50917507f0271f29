"""Rate conversion on the device (vfx_resample) against scipy's resample_poly (the host loader, wavio._resample), bit for
bit: one mixed-rate ragged launch, a 10-minute 48 kHz recording per 30 s segment (past the 2^31 index), and
restore_many / oracle_many with sample_rate= against the same calls on the host-resampled recordings.  Also the
refusals of a bad item or a short workspace, and that an all-44.1 kHz call launches nothing new."""
import numpy as np
import pytest
import torch

from voicefixer_b200 import _lib, wavio
from voicefixer_b200 import resample as rs
from voicefixer_b200.engine import _ptr, _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100
SEG = 30 * SR
RATES = [8000, 11025, 16000, 22050, 24000, 32000, 48000, 96000, 44056, 44100]
GAP = 7                                      # NaNs between staged windows and between tap sets: never read

_ENGINES = {}


def _engine(states, prec="tf32"):
    if prec not in _ENGINES:
        from voicefixer_b200.engine import Engine
        _ENGINES[prec] = Engine(states[0], states[1], precision=prec)
    return _ENGINES[prec]


def _x(n, seed):
    return (0.3 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def _launch(eng, jobs, L_cap, ws_bytes=None, sentinel=float("nan")):
    """jobs: [(x, rate, a, b)]: outputs [a, b) of recording x at `rate`.  Stages each window and each ratio's taps between
    NaN gaps, prefills y with `sentinel` and calls vfx_resample.  Returns (rc, y, lens_out, table)."""
    stage, taps, tap_off, table = [np.full(GAP, np.nan, np.float32)], [np.full(GAP, np.nan, np.float32)], {}, []
    off, hoff = GAP, GAP
    for x, rate, a, b in jobs:
        first, stop = rs.window(len(x), rate, a, b)
        up, down = rs.ratio(rate)
        h, rem = rs.taps(rate)
        if (up, down) not in tap_off and len(h):
            tap_off[(up, down)] = hoff
            taps += [h, np.full(GAP, np.nan, np.float32)]
            hoff += len(h) + GAP
        it = _lib.ResampleItem(x_off=off, x_first=first, n_in=len(x), y_first=a, h_off=tap_off.get((up, down), 0),
                               x_len=stop - first, y_len=b - a, up=up, down=down, rem=rem, h_len=len(h))
        table.append(it)
        stage += [x[first:stop], np.full(GAP, np.nan, np.float32)]
        off += stop - first + GAP
    xs = torch.from_numpy(np.concatenate(stage)).to(DEV)
    hs = torch.from_numpy(np.concatenate(taps)).to(DEV)
    B = len(jobs)
    arr = (_lib.ResampleItem * B)(*table)
    y = torch.full((B, L_cap), sentinel, device=DEV)
    lens = torch.full((B,), -5, dtype=torch.int32, device=DEV)
    need = eng.resample_workspace_bytes(B)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    rc = eng.lib.vfx_resample(eng.h, _ptr(xs), xs.numel(), _ptr(hs), hs.numel(), arr, B, _ptr(y), L_cap, _ptr(lens),
                              _ptr(ws), need if ws_bytes is None else ws_bytes, _stream())
    torch.cuda.synchronize()
    return rc, y.cpu().numpy(), lens.cpu().numpy(), arr


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ============================================================================ 1. the kernel against scipy
def test_mixed_rate_ragged_launch_equals_resample_poly(states):
    eng = _engine(states)
    jobs, refs = [], []
    for rate in RATES:
        rng = np.random.default_rng(rate)
        for n in [1, 2, 37, 4099] + [int(v) for v in rng.integers(5000, 48018, 2)]:
            x = _x(n, n + rate)
            ref = wavio._resample(x, rate, SR)
            jobs.append((x, rate, 0, len(ref)))
            refs.append(ref)
        x = _x(int(2.3 * rate), rate)                   # segment windows: the middle of a recording, and its tail
        ref = wavio._resample(x, rate, SR)
        for a, b in ((SR // 2, SR + 777), (len(ref) - 5000, len(ref))):
            jobs.append((x, rate, a, b))
            refs.append(ref[a:b])
    L_cap = max(len(r) for r in refs) + 3
    rc, y, lens, _ = _launch(eng, jobs, L_cap)
    assert rc == 0, eng.lib.vfx_last_error()
    for k, ref in enumerate(refs):
        assert _same_bits(y[k, :len(ref)], ref), f"item {k} ({jobs[k][1]} Hz, outputs {jobs[k][2]}..{jobs[k][3]})"
        assert (y[k, len(ref):] == 0).all() and not np.signbit(y[k, len(ref):]).any(), f"item {k}: row tail"
    assert lens.tolist() == [len(r) for r in refs]


def test_ten_minutes_at_48k_per_segment_window(states):
    """20 segments of 30 s out of 26.5 M samples at 44.1 kHz: p = (j + rem) * 160 passes 2^31 from j = 13.4 M on."""
    eng = _engine(states)
    x = _x(600 * 48000, 48)
    ref = wavio._resample(x, 48000, SR)
    assert (len(ref) + rs.taps(48000)[1]) * 160 > 2 ** 31
    bounds = [(a, min(a + SEG, len(ref))) for a in range(0, len(ref), SEG)]
    rc, y, lens, _ = _launch(eng, [(x, 48000, a, b) for a, b in bounds], SEG)
    assert rc == 0, eng.lib.vfx_last_error()
    for k, (a, b) in enumerate(bounds):
        assert _same_bits(y[k, :b - a], ref[a:b]), f"segment {k} ({a}..{b})"
    assert lens.tolist() == [b - a for a, b in bounds]


# ============================================================================ 2. refusals
def _bad(table, k, **fields):
    for f, v in fields.items():
        setattr(table[k], f, v)


@pytest.mark.parametrize("fields,match", [
    (dict(up=0), "item 1: ratio"),
    (dict(x_first=1), "read inputs [27, 736); the window holds [1, 710)"),   # shifted: no longer holds the last input
    (dict(x_len=10 ** 9), "item 1: window"),
    (dict(h_off=10 ** 6), "item 1: taps"),
    (dict(y_len=SR + 1), "item 1: y_len"),
    (dict(y_first=10 ** 7), "item 1: outputs"),
])
def test_bad_item_is_refused_before_any_launch(states, fields, match):
    eng = _engine(states)
    x = _x(20000, 3)
    jobs = [(x, 16000, 0, 1000), (x, 16000, 100, 2000)]
    rc, _, _, table = _launch(eng, jobs, SR)
    assert rc == 0
    _bad(table, 1, **fields)
    xs = torch.zeros(10 ** 6, device=DEV)
    hs = torch.from_numpy(rs.taps(16000)[0].copy()).to(DEV)
    table[0].x_off = table[1].x_off = 0
    table[0].h_off = 0
    if "h_off" not in fields:
        table[1].h_off = 0
    y = torch.full((2, SR), -1920.0, device=DEV)
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    rc = eng.lib.vfx_resample(eng.h, _ptr(xs), xs.numel(), _ptr(hs), hs.numel(), table, 2, _ptr(y), SR, None, _ptr(ws),
                              4096, _stream())
    torch.cuda.synchronize()
    assert rc == -1 and match.encode() in eng.lib.vfx_last_error(), eng.lib.vfx_last_error()
    assert eng.launch_count() == n0
    assert bool((y == -1920.0).all()), "a refused call wrote its output"


def test_short_workspace_is_refused_before_any_launch(states):
    eng = _engine(states)
    x = _x(20000, 4)
    jobs = [(x, 16000, 0, 1000)] * 5                            # 5 items: a 320-byte table
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    rc, y, lens, _ = _launch(eng, jobs, 1000, ws_bytes=256, sentinel=-1920.0)
    assert rc == -3 and b"workspace too small" in eng.lib.vfx_last_error()
    assert eng.launch_count() == n0
    assert (y == -1920.0).all() and (lens == -5).all()
    rc, y, lens, _ = _launch(eng, jobs, 1000)
    assert rc == 0 and eng.launch_count() == n0 + 1


# ============================================================================ 3. the public API
RECORDINGS = [(16000, 2.0), (48000, 31.0), (44100, 3.0), (8000, 1.5), (22050, 65.2), (96000, 4.0)]


def _recordings(seed):
    return [_x(int(s * r), seed + k) for k, (r, s) in enumerate(RECORDINGS)], [r for r, _ in RECORDINGS]


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
def test_restore_many_with_rates_equals_host_resampling(states, prec):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer.from_engine(_engine(states, prec))
    wavs, rates = _recordings(50)
    host = [wavio._resample(w, r, SR) for w, r in zip(wavs, rates)]
    for mode, fn in ((0, None), (1, None), (2, False)):
        got = vf.restore_many(wavs, mode=mode, drop_masks_fn=fn, sample_rate=rates)
        want = vf.restore_many(host, mode=mode, drop_masks_fn=fn)
        for i in range(len(wavs)):
            assert _same_bits(got[i], want[i]), f"{prec} mode {mode}: recording {i} ({rates[i]} Hz)"
    torch.manual_seed(51)
    got = vf.restore_many(wavs, mode=2, sample_rate=rates)                 # default masks: the same draws
    after = torch.rand(3)
    torch.manual_seed(51)
    want = vf.restore_many(host, mode=2)
    assert torch.equal(torch.rand(3), after), "the device path drew from torch's generator"
    for i in range(len(wavs)):
        assert _same_bits(got[i], want[i]), f"{prec} mode 2 with masks: recording {i}"


def test_oracle_many_with_rates_equals_host_resampling(states):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer.from_engine(_engine(states, "tf32"))
    wavs, rates = _recordings(60)
    got = vf._vocoder.oracle_many(wavs, sample_rate=rates)
    want = vf._vocoder.oracle_many([wavio._resample(w, r, SR) for w, r in zip(wavs, rates)])
    for i in range(len(wavs)):
        assert _same_bits(got[i], want[i]), f"recording {i} ({rates[i]} Hz)"
    one = vf._vocoder.oracle_many(wavs[:1], sample_rate=16000)[0]
    assert _same_bits(one, want[0])


def test_16k_wav_file_restores_like_the_file_path(states, tmp_path):
    from voicefixer_b200.api import VoiceFixer
    vf = VoiceFixer.from_engine(_engine(states, "tf32"))
    path = str(tmp_path / "x16k.wav")
    wavio.save_wave(_x(3 * 16000, 70)[None] / 3, path, sample_rate=16000)        # peak below 1: scaled to int16
    pcm, sr = wavio._read_pcm(path)
    assert sr == 16000 and pcm.shape[1] == 1
    got = vf.restore_many([pcm[:, 0]], sample_rate=16000)[0]
    want = vf.restore_inmem(vf._load_wav(path, 44100), cuda=True)
    assert _same_bits(got, want)


def test_default_rate_launches_nothing_new(states):
    from voicefixer_b200.api import VoiceFixer
    eng = _engine(states, "tf32")
    vf = VoiceFixer.from_engine(eng)
    wavs = [_x(n, n) for n in (3 * SR, 31 * SR)]
    counts = []
    for kw in ({}, {"sample_rate": 44100}, {"sample_rate": [44100, 44100]}):
        n0 = eng.launch_count()
        vf.restore_many(wavs, **kw)
        counts.append(eng.launch_count() - n0)
    assert counts[0] == counts[1] == counts[2] > 0
    n0 = eng.launch_count()
    vf.restore_many(wavs, sample_rate=[44100, 16000])
    assert eng.launch_count() - n0 > counts[0]                              # one resampling launch per batch


@pytest.mark.parametrize("kw,match", [
    (dict(sample_rate=16000.5), "restore_many: recording 0 has sample_rate 16000.5"),
    (dict(sample_rate=[16000]), "restore_many: sample_rate has 1 entries for 2 recordings"),
    (dict(sample_rate=[16000, 0]), "restore_many: recording 1 has sample_rate 0"),
])
def test_bad_rates_raise_before_launching(states, kw, match):
    from voicefixer_b200.api import VoiceFixer
    eng = _engine(states, "tf32")
    vf = VoiceFixer.from_engine(eng)
    n0 = eng.launch_count()
    with pytest.raises(ValueError, match=match):
        vf.restore_many([_x(SR, 1), _x(SR, 2)], **kw)
    with pytest.raises(ValueError, match=match.replace("restore_many", "oracle_many")):
        vf._vocoder.oracle_many([_x(SR, 1), _x(SR, 2)], **kw)
    assert eng.launch_count() == n0
