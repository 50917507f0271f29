"""Rate conversion to 44.1 kHz without a GPU: the device kernel's loop restated in numpy from resample.taps / out_len /
window equals scipy's resample_poly (the host loader, wavio._resample) bit for bit, whole and per 30 s segment window;
the rate validation of restore_many / oracle_many; and the C ABI of vfx_resample (bindings, struct layout, workspace
size, refusal on a planning-only engine)."""
import ctypes
import os
import re
import numpy as np
import pytest

from voicefixer_b200 import resample as rs
from voicefixer_b200 import wavio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATES = [8000, 11025, 16000, 22050, 24000, 32000, 48000, 96000, 44056]
SEG = 44100 * 30


def restate(xw, first, n_in, rate, a, b):
    """Outputs [a, b) of a recording of n_in samples at `rate` as resample.cu computes them, reading only the window
    xw = recording[first : first + len(xw)] (an index outside it raises)."""
    up, down = rs.ratio(rate)
    if up == down == 1:
        assert first <= a and b - first <= len(xw)
        return xw[a - first:b - first].copy()
    h, rem = rs.taps(rate)
    p = (np.arange(a, b, dtype=np.int64) + rem) * down
    num = p - len(h) + 1
    lo = np.maximum(0, -(-num // up))
    hi = np.minimum(n_in - 1, p // up)
    acc = np.zeros(b - a, np.float32)
    for k in range(int((hi - lo).max()) + 1 if b > a else 0):
        i = lo + k
        live = i <= hi
        i = np.where(live, i, lo)
        assert (i[live] >= first).all() and (i[live] < first + len(xw)).all(), "read outside the window"
        prod = xw[i - first] * h[np.where(live, p - i * up, 0)]       # float32 product, then a float32 sum: no FMA
        acc = np.where(live, acc + prod, acc)
    return acc


def _x(n, seed):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32)


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _lengths(rate):
    return [1, 2, 37, 4099] + [int(n) for n in np.random.default_rng(rate).integers(5000, 48018, 2)]


@pytest.mark.parametrize("rate", RATES)
def test_restated_kernel_equals_resample_poly_on_whole_recordings(rate):
    for n in _lengths(rate):
        x = _x(n, n + rate)
        ref = wavio._resample(x, rate, 44100)
        assert len(ref) == rs.out_len(n, rate)
        first, stop = rs.window(n, rate, 0, len(ref))
        assert (first, stop) == (0, n)
        assert _bits_equal(restate(x[first:stop], first, n, rate, 0, len(ref)), ref), f"{rate} Hz, {n} samples"


@pytest.mark.parametrize("rate", RATES)
def test_segment_windows_reproduce_the_whole_stream(rate):
    """30 s segments of a 44.1 kHz stream computed from their own input windows: the first and last 3000 samples of every
    segment (the halo is all at the edges), for a recording of three segments and one shorter than a segment."""
    for seconds in (65.3, 7.0):
        n = int(seconds * rate)
        x = _x(n, rate)
        ref = wavio._resample(x, rate, 44100)
        n_out = rs.out_len(n, rate)
        bounds = [(a, min(a + SEG, n_out)) for a in range(0, n_out, SEG)]
        assert len(bounds) == (3 if seconds > 60 else 1)
        for a, b in bounds:
            first, stop = rs.window(n, rate, a, b)
            assert stop - first <= rs.staging_bound(b - a, rate)
            for lo, hi in ((a, min(b, a + 3000)), (max(a, b - 3000), b)):
                y = restate(x[first:stop], first, n, rate, lo, hi)
                assert _bits_equal(y, ref[lo:hi]), f"{rate} Hz, segment {a}..{b}, samples {lo}..{hi}"
            # the window is tight: one sample less on either side and the segment reads outside it
            if first > 0:
                with pytest.raises(AssertionError, match="outside the window"):
                    restate(x[first + 1:stop], first + 1, n, rate, a, a + 1)
            if stop < n:
                with pytest.raises(AssertionError, match="outside the window"):
                    restate(x[first:stop - 1], first, n, rate, b - 1, b)


def test_taps_and_ratios():
    assert rs.ratio(16000) == (441, 160) and rs.ratio(48000) == (147, 160) and rs.ratio(44100) == (1, 1)
    h, rem = rs.taps(16000)
    half = 10 * 441
    assert h.dtype == np.float32 and len(h) == (160 - half % 160) + 2 * half + 1 and rem == (half + 160 - half % 160) // 160
    assert not h.flags.writeable and rs.taps(16000)[0] is h                  # cached per ratio
    assert len(rs.taps(44100)[0]) == 0 and rs.out_len(12345, 44100) == 12345
    assert rs.out_len(16000, 16000) == 44100 and rs.out_len(1, 48000) == 1
    assert rs.window(100, 16000, 5, 5) == (0, 0)


@pytest.mark.parametrize("sample_rate,n,match", [
    (16000.0, 2, "recording 0 has sample_rate 16000.0"),
    (0, 1, "recording 0 has sample_rate 0"),
    (-8000, 3, "recording 0 has sample_rate -8000"),
    (True, 1, "recording 0 has sample_rate True"),
    ("16000", 1, "recording 0 has sample_rate '16000'"),
    ([16000, 44100, None], 3, "recording 2 has sample_rate None"),
    ([16000, 2 ** 31], 2, "recording 1 has sample_rate 2147483648"),
    ([16000, 44100], 3, "sample_rate has 2 entries for 3 recordings"),
    ((), 1, "sample_rate has 0 entries for 1 recordings"),
])
def test_rate_validation_messages(sample_rate, n, match):
    with pytest.raises(ValueError, match="restore_many: " + re.escape(match)):
        rs.rates(sample_rate, n, "restore_many")


def test_rates_accepts_ints_lists_and_arrays():
    assert rs.rates(16000, 3, "x") == [16000] * 3
    assert rs.rates([8000, np.int64(48000)], 2, "x") == [8000, 48000]
    assert rs.rates(np.array([22050, 44100]), 2, "x") == [22050, 44100]
    assert all(type(r) is int for r in rs.rates(np.array([22050]), 1, "x"))


def _header():
    return open(os.path.join(ROOT, "include", "vfx_b200.h")).read()


@pytest.mark.parametrize("name", ["vfx_resample", "vfx_resample_workspace_bytes"])
def test_entry_points_bound_like_the_header(name):
    from voicefixer_b200 import _lib
    m = re.search(r"^(?:int|size_t) " + name + r"\((.*?)\);", _header(), flags=re.S | re.M)
    assert m and name in _lib.SIGNATURES and hasattr(_lib.load(), name)
    args = [a.strip() for a in m.group(1).split(",")]
    sig = _lib.SIGNATURES[name][1]
    assert len(sig) == len(args)
    want = {"int ": _lib._i, "long long ": _lib._ll, "size_t ": _lib._sz}
    for a, t in zip(args, sig):
        for prefix, ct in want.items():
            if a.startswith(prefix):
                assert t is ct, (name, a)
        if "*" in a and "vfx_resample_item" not in a:
            assert t is _lib._vp, (name, a)


def test_item_struct_matches_the_header():
    from voicefixer_b200 import _lib
    body = re.search(r"typedef struct vfx_resample_item \{(.*?)\} vfx_resample_item;", _header(), flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype = _lib._ll if decl.startswith("long long ") else _lib._i
        assert decl.startswith(("long long ", "int ")), decl
        fields += [(nm.strip(), ctype) for nm in decl.split(" ", 2 if ctype is _lib._ll else 1)[-1].split(",")]
    assert [(f, t) for f, t in _lib.ResampleItem._fields_] == fields
    assert ctypes.sizeof(_lib.ResampleItem) == 64


def test_workspace_is_sized_without_a_gpu():
    from voicefixer_b200.engine import Engine
    assert [Engine.resample_workspace_bytes(B) for B in (0, -1, 1, 4, 5, 64)] == [0, 0, 64, 256, 320, 4096]   # the staged item table


def test_planning_only_engine_refuses_resample(states):
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import Planner
    from voicefixer_b200.weights import pack_vocoder
    pv = Planner(pack_vocoder(states[1], "tf32"), "tf32")
    item = (_lib.ResampleItem * 1)()
    item[0].n_in, item[0].x_len, item[0].y_len, item[0].up, item[0].down = 4, 4, 4, 1, 1
    fake = ctypes.c_void_p(256)                                         # never dereferenced
    rc = pv.lib.vfx_resample(pv.h, fake, 4, None, 0, item, 1, fake, 4, None, fake, 256, None)
    assert rc == -1 and b"planning-only" in pv.lib.vfx_last_error()


def test_oracle_plan_packs_by_the_resampled_lengths():
    from voicefixer_b200.api import plan_vocoder_many
    wavs, rates = [np.ones(16000, np.float32), np.ones(44100, np.float32), np.ones(48000, np.float32)], [16000, 44100, 48000]
    lens = [rs.out_len(w.shape[0], r) for w, r in zip(wavs, rates)]
    assert lens == [44100, 44100, 44100]
    assert plan_vocoder_many(wavs, "wav", lambda L: 2, pack_lengths=lens) == [(44100, [0, 1]), (44100, [2])]
    with pytest.raises(ValueError, match="item 1 is all zeros"):                 # the recordings themselves are checked
        plan_vocoder_many([wavs[0], np.zeros(10, np.float32)], "wav", lambda L: 2, pack_lengths=[44100, 28])
