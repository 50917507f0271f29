"""The window schedule that VoiceFixer.restore_stream and StreamPool share, and the pool's bookkeeping, without a GPU: the
schedule against a literal copy of restore_stream's former loop, the availability prefix of a stream at another rate,
and the pool against a stub engine whose "restore" is a position- and length-dependent element-wise map and whose
resampler is scipy on the staged window."""
import numpy as np
import pytest
import torch

from voicefixer_b200 import api, resample, wavio

SR = 44100


# ============================================================================ 1. the schedule
def _old_loop(block_sizes, chunk, ctx):
    """restore_stream's window loop as it stood before the schedule was shared, written out: yields (lo, hi, keep_lo,
    keep_hi) where the old code ran a window, and tracks the same buffer of received samples."""
    buf_len = 0
    base = 0
    pos = 0
    for n in block_sizes:
        buf_len += n
        while base + buf_len >= pos + chunk + ctx:
            lo = max(0, pos - ctx)
            yield (lo, pos + chunk + ctx, pos, pos + chunk)
            pos += chunk
            drop = max(0, pos - ctx) - base
            if drop > 0:
                buf_len, base = buf_len - drop, base + drop
    end = base + buf_len
    while pos < end:
        hi = min(end, pos + chunk + ctx)
        keep_hi = min(end, pos + chunk)
        if end - keep_hi <= 1024 and end - keep_hi > 0 and ctx == 0:
            keep_hi = hi = end
        lo = max(0, pos - ctx)
        if hi - lo <= 1024:
            lo = max(0, hi - 1025 - ctx)
            if hi - lo <= 1024:
                raise RuntimeError("restore_stream: fewer than 1025 samples in total; the front end reflect-pads 1024")
        yield (lo, hi, pos, keep_hi)
        pos = keep_hi


def _new_loop(block_sizes, chunk, ctx):
    """The same stream through StreamSchedule, as restore_stream drives it: (windows, emit position after each)."""
    sched = api.StreamSchedule(chunk, ctx)
    avail, pos, wins, emitted = 0, 0, [], []
    for n in block_sizes:
        avail += n
        w, pos = sched.due(pos, avail, ended=False)
        wins += w
        emitted += [k for _, _, _, k in w]
        assert not w or pos == w[-1][3]
    w, pos = sched.due(pos, avail, ended=True)
    wins += w
    emitted += [k for _, _, _, k in w]
    assert pos == avail
    return wins, emitted


def _outcome(fn):
    try:
        return fn(), None
    except RuntimeError as e:
        return None, str(e)


def _blocks(rng, total, lo, hi):
    """Seeded block sizes log-uniform in [lo, hi] samples, summing to total."""
    sizes = []
    while sum(sizes) < total:
        sizes.append(int(min(total - sum(sizes), np.exp(rng.uniform(np.log(lo), np.log(hi))))))
    return sizes


CONFIGS = [(SR, SR // 2), (SR // 4, SR // 10), (2 * SR, SR), (SR, 0), (30 * SR, 0), (3000, 0), (2000, 100), (1500, 2000)]
TAILS = [1, 2, 511, 1023, 1024, 1025]


@pytest.mark.parametrize("chunk,ctx", CONFIGS)
@pytest.mark.parametrize("seed", range(4))
def test_schedule_equals_the_old_loop(chunk, ctx, seed):
    rng = np.random.default_rng(seed)
    sched = api.StreamSchedule(chunk, ctx)
    totals = [0, 1, 1024, 1025, 1026] + [k * chunk + t for k in (0, 1, 3) for t in TAILS] + [int(rng.integers(1, 8 * SR))]
    for total in totals:
        for lo, hi in ((1, 3 * SR), (1, 64), (SR // 10, SR // 10)):
            if total > 200_000 and hi < 1000:
                continue                       # 1-sample blocks: short streams only
            sizes = _blocks(rng, total, lo, hi)
            old, old_err = _outcome(lambda: list(_old_loop(sizes, chunk, ctx)))
            new, new_err = _outcome(lambda: _new_loop(sizes, chunk, ctx))
            assert old_err == new_err, (total, sizes[:5])
            if old_err is None:
                wins, emitted = new
                assert wins == old, (total, sizes[:5])
                assert emitted == [w[3] for w in old]
                assert all(h - l <= sched.capacity for l, h, _, _ in wins)


def test_capacity_is_reached():
    """The bound is the rule's: full windows reach chunk + 2 ctx, short flush windows 1025 + ctx."""
    for chunk, ctx in [(SR, SR // 2), (500, 1000)]:
        sched = api.StreamSchedule(chunk, ctx)
        longest = 0
        for total in range(1025, 4 * (chunk + ctx)):
            wins, _ = sched.due(0, total, ended=True)
            longest = max([longest] + [h - l for l, h, _, _ in wins])
        assert longest == sched.capacity == max(chunk + 2 * ctx, 1025 + ctx)
    assert api.StreamSchedule(SR, 0).capacity == SR + 1024
    assert api.StreamSchedule(100, 0).capacity == 1124


# ============================================================================ 2. availability at other rates
@pytest.mark.parametrize("rate", [8000, 16000, 48000, 22050, 44100])
def test_available_prefix_by_brute_force(rate):
    big = 10 ** 9                              # a recording far longer than any prefix here: window() does not clip
    stops = [resample.window(big, rate, j, j + 1)[1] for j in range(resample.out_len(1400, rate) + 10)]
    for n in list(range(0, 600)) + [997, 1400]:
        m = 0
        while m < len(stops) and stops[m] <= n:
            m += 1
        assert m < len(stops)
        assert resample.available(n, rate) == m, n
        assert resample.available(n, rate) <= resample.out_len(n, rate)


# ============================================================================ 3. the pool against a stub engine
def _fake_restore(row):
    """Stands in for the restore of one window: depends on each sample, its place in the window and the window's length."""
    n = row.shape[0]
    return (row * np.float32(0.5) + np.arange(n, dtype=np.float32) * np.float32(1e-4) + np.float32(n * 1e-6)).astype(np.float32)


class _Graph:
    def __init__(self, eng, wav, out, lens):
        self.eng, self.wav, self.out, self.lens = eng, wav, out, lens

    def replay(self):
        lens = self.lens.tolist()
        self.eng.launches.append((self.wav.shape[0], lens))
        for b, n in enumerate(lens):
            assert 1025 <= n <= self.wav.shape[1]
            self.out[b, :n] = torch.from_numpy(_fake_restore(self.wav[b, :n].numpy()))


class _StubEngine:
    device = 0

    def __init__(self, fit=64):
        self.fit, self.launches, self.resamples, self.captures = fit, [], [], []

    def max_batch(self, L, extra_per_item=0):
        return self.fit

    def workspace_bytes(self, B, L):
        return 64

    def make_graph(self, wav, out, mode=0, lens=None, ws=None):
        assert mode == 0 and lens is not None and ws is not None and wav.shape == out.shape
        self.captures.append(wav.shape[0])
        return _Graph(self, wav, out, lens)

    def resample(self, x, items, L_cap):
        """scipy on each item's staged window, zero elsewhere: output samples whose inputs all lie in the window are
        wavio._resample's on the whole recording."""
        self.resamples.append(len(items))
        y = torch.zeros(len(items), L_cap)
        for b, (rate, n_in, x_off, x_first, x_len, y_first, y_len) in enumerate(items):
            full = np.zeros(n_in, np.float32)
            full[x_first:x_first + x_len] = x[x_off:x_off + x_len].numpy()
            y[b, :y_len] = torch.from_numpy(wavio._resample(full, rate, SR)[y_first:y_first + y_len])
        return y, torch.tensor([it[6] for it in items], dtype=torch.int32)


def _pool(chunk=0.25, ctx=0.1, max_windows=3, fit=64):
    eng = _StubEngine(fit)
    return eng, api.StreamPool(eng, chunk, ctx, max_windows, device="cpu")


def _want(x, rate, sizes, chunk, ctx):
    """restore_stream's output on the stream alone: the old loop, windows through _fake_restore."""
    y = wavio._resample(x, rate, SR)
    out = [_fake_restore(y[lo:hi])[kl - lo:kh - lo] for lo, hi, kl, kh in _old_loop(sizes, chunk, ctx)]
    return np.concatenate(out) if out else np.zeros(0, np.float32)


def _split(rng, n, lo, hi):
    cuts = np.cumsum(_blocks(rng, n, lo, hi))
    return [0] + cuts.tolist()


@pytest.mark.parametrize("chunk_s,ctx_s", [(0.25, 0.1), (0.1, 0.0)])
@pytest.mark.parametrize("seed", range(3))
def test_pool_equals_each_stream_alone(seed, chunk_s, ctx_s):
    rng = np.random.default_rng(seed)
    eng, pool = _pool(chunk_s, ctx_s, max_windows=3)
    chunk, ctx = int(round(chunk_s * SR)), int(round(ctx_s * SR))
    specs = []
    for k, rate in enumerate([44100, 8000, 16000, 48000, 44100, 16000]):
        n = int(rng.integers(rate // 40 + 1, int(1.6 * rate)))
        n = max(n, -(-1100 * rate // SR))
        x = (0.3 * rng.standard_normal(n)).astype(np.float32)
        cuts = _split(rng, n, rate // 1000, rate // 3)
        specs.append(dict(x=x, rate=rate, cuts=cuts, k=0, sid=None, start=int(rng.integers(0, 6)), got=[]))
    t = 0
    while any(s["sid"] is None or s["sid"] in pool.streams for s in specs) or pool.pending:
        for s in specs:
            if s["sid"] is None and t >= s["start"]:
                s["sid"] = pool.open(s["rate"])
            elif s["sid"] is not None and not s.get("closed"):
                for _ in range(int(rng.integers(0, 4))):
                    if s["k"] < len(s["cuts"]) - 1:
                        pool.push(s["sid"], s["x"][s["cuts"][s["k"]]:s["cuts"][s["k"] + 1]])
                        s["k"] += 1
                if s["k"] == len(s["cuts"]) - 1:
                    pool.close(s["sid"])
                    s["closed"] = True
        if rng.random() < 0.7:
            out = pool.step()
            for s in specs:
                s["got"] += out.get(s["sid"], []) if s["sid"] is not None else []
        t += 1
        assert t < 10_000
    assert pool.streams == [] and pool.pending == 0
    for s in specs:
        y44 = wavio._resample(s["x"], s["rate"], SR)
        sizes = np.diff(_split(np.random.default_rng(0), len(y44), 1, SR // 3)).tolist()
        want = _want(s["x"], s["rate"], sizes, chunk, ctx)
        got = np.concatenate(s["got"])
        assert got.shape[0] == resample.out_len(len(s["x"]), s["rate"])
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), s["rate"]
    assert all(B in pool.buckets for B, _ in eng.launches)
    assert sorted(set(eng.captures)) == sorted(set(B for B, _ in eng.launches)) == sorted(set(eng.captures))
    assert len(eng.captures) == pool.graph_count


def test_oldest_first_and_the_cap():
    eng, pool = _pool(chunk=0.25, ctx=0.0, max_windows=2)
    chunk = int(0.25 * SR)
    a, b = pool.open(), pool.open()
    xa = np.arange(3 * chunk, dtype=np.float32)
    xb = -np.arange(2 * chunk, dtype=np.float32)
    pool.push(a, xa[:2 * chunk])                # a's windows 0, 1 fall due
    pool.push(b, xb[:chunk])                    # then b's window 0
    pool.push(a, xa[2 * chunk:])                # then a's window 2
    assert pool.pending == 4
    out = pool.step()
    assert list(out) == [a] and len(out[a]) == 2 and eng.launches[-1] == (2, [chunk, chunk])
    out = pool.step()
    assert list(out) == [b, a] and len(out[a]) == 1 and len(out[b]) == 1
    assert pool.step() == {} and len(eng.launches) == 2
    np.testing.assert_array_equal(out[b][0], _fake_restore(xb[:chunk]))


def test_bucket_choice():
    eng, pool = _pool(chunk=0.1, ctx=0.0, max_windows=5)
    assert pool.buckets == [1, 2, 4, 5]
    chunk = int(0.1 * SR)
    sids = [pool.open() for _ in range(5)]
    for n in [1, 2, 3, 4, 5, 1, 3]:
        for sid in sids[:n]:
            pool.push(sid, np.ones(chunk, np.float32))
        pool.step()
        B, lens = eng.launches[-1]
        assert B == {1: 1, 2: 2, 3: 4, 4: 4, 5: 5}[n]
        assert lens[:n] == [chunk] * n and lens[n:] == [1025] * (B - n)
    assert eng.captures == [1, 2, 4, 5] and pool.graph_count == 4
    _, pool = _pool(max_windows=8)
    assert pool.buckets == [1, 2, 4, 8]
    _, pool = _pool(max_windows=None, fit=12)
    assert pool.max_windows == 12 and pool.buckets == [1, 2, 4, 8, 12]
    _, pool = _pool(max_windows=40, fit=12)
    assert pool.max_windows == 12


def test_windows_wait_for_their_input_at_other_rates():
    for rate in (8000, 16000, 48000):
        eng, pool = _pool(chunk=0.25, ctx=0.1)
        chunk, ctx = int(round(0.25 * SR)), int(round(0.1 * SR))
        sid = pool.open(rate)
        x = np.ones(2 * rate, np.float32)
        n = 0
        while pool.pending == 0:
            pool.push(sid, x[n:n + 7])
            n += 7
        # the first window falls due with the first push after which its last sample's inputs have all arrived
        assert resample.available(n, rate) >= chunk + ctx > resample.available(n - 7, rate)


def test_a_step_at_44100_launches_no_resampler():
    eng, pool = _pool(chunk=0.1, ctx=0.0)
    a, b = pool.open(44100), pool.open(16000)
    pool.push(a, np.ones(SR // 10, np.float32))
    pool.step()
    assert eng.resamples == [] and len(eng.launches) == 1
    pool.push(b, np.ones(16000, np.float32))
    pool.push(a, np.ones(SR // 10, np.float32))
    pool.step()
    assert eng.resamples == [3]                  # a mixed step resamples every row, the 44.1 kHz ones as copies


def _no_launch(eng):
    assert eng.launches == [] and eng.resamples == [] and eng.captures == []


def test_refusals_name_the_stream_and_launch_nothing():
    eng, pool = _pool()
    a = pool.open()
    with pytest.raises(ValueError, match=r"stream_pool.push: stream 7 is not open"):
        pool.push(7, np.ones(10, np.float32))
    with pytest.raises(ValueError, match=r"stream_pool.close: stream 'x' is not open"):
        pool.close("x")
    for bad in (0, -8000, 44100.0, True, "16k"):
        with pytest.raises(ValueError, match=r"stream_pool.open: stream 1 has sample_rate .* positive integer"):
            pool.open(bad)
    with pytest.raises(ValueError, match=r"stream_pool.push: stream 0: a block has shape \(2, 3\)"):
        pool.push(a, np.ones((2, 3), np.float32))
    pool.push(a, np.ones(20000, np.float32))
    pool.close(a)
    with pytest.raises(ValueError, match=r"stream_pool.push: stream 0 is closed"):
        pool.push(a, np.ones(10, np.float32))
    with pytest.raises(ValueError, match=r"stream_pool.close: stream 0 is closed"):
        pool.close(a)
    for chunk, ctx in ((0, 0.5), (-1, 0.5), (0.5, -0.1)):
        with pytest.raises(ValueError, match="chunk_seconds must be positive and context_seconds non-negative"):
            api.StreamPool(eng, chunk, ctx, device="cpu")
    with pytest.raises(ValueError, match="at least 1025"):
        api.StreamPool(eng, 0.01, 0.01, device="cpu")
    for bad in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match="max_windows"):
            api.StreamPool(eng, 1.0, 0.5, max_windows=bad, device="cpu")
    _no_launch(eng)
    assert pool.open(16000) == 1                 # refused opens did not use up an id


@pytest.mark.parametrize("rate,n", [(44100, 1024), (44100, 1), (16000, 371), (8000, 185)])
def test_a_short_stream_is_refused_at_close(rate, n):
    eng, pool = _pool(chunk=1.0, ctx=0.5)
    other = pool.open()
    short = pool.open(rate)
    pool.push(other, np.ones(5000, np.float32))
    pool.push(short, np.ones(n, np.float32))
    with pytest.raises(RuntimeError, match=r"stream_pool.close: stream 1: restore_stream: fewer than 1025 samples in "
                                           r"total; the front end reflect-pads 1024"):
        pool.close(short)
    assert resample.out_len(n, rate) <= 1024
    _no_launch(eng)
    assert pool.streams == [other]
    with pytest.raises(ValueError, match="stream 1 is not open"):
        pool.push(short, np.ones(10, np.float32))
    pool.close(other)
    out = pool.step()
    assert list(out) == [other] and np.concatenate(out[other]).shape == (5000,)
    assert pool.streams == []


def test_an_empty_stream_is_forgotten_without_output():
    eng, pool = _pool()
    sid = pool.open()
    pool.close(sid)
    assert pool.step() == {} and pool.streams == []
    _no_launch(eng)


def test_old_input_is_dropped():
    eng, pool = _pool(chunk=0.25, ctx=0.1, max_windows=64)
    for rate in (44100, 16000):
        sid = pool.open(rate)
        x = np.ones(20 * rate, np.float32)
        for k in range(0, len(x), rate // 10):
            pool.push(sid, x[k:k + rate // 10])
            pool.step()
        s = pool._streams[sid]
        assert s.buf.shape[0] < rate             # about chunk + 2 ctx of input is held, not the whole 20 s
        pool.close(sid)
        pool.step()
