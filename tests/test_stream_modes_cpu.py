"""Streams in modes 1 and 2 without a GPU: the window rule (StreamSchedule) with each mode's shortest window and mode 1's
shortened output, over the chunk / context grid of the mode-0 schedule test; its 30 s / 0 s spans against
restore_inmem's segments; the refusals of restore_stream and StreamPool; restore_stream's per-window calls against a
stub engine; and StreamPool against a stub engine whose "restore" depends on the row, its length, the mode and the
dropout key, so that each stream's output must equal the stream alone, bit for bit, however the streams interleave."""
import re

import numpy as np
import pytest
import torch

from test_stream_pool_cpu import CONFIGS, TAILS, _blocks, _split
from voicefixer_b200 import api, resample, wavio

SR = 44100
MIN = {1: 1536, 2: 28224}
MSG = {1: r"mode 1's pre-filter keeps 512 \* \(L // 512\) samples of L and the front end reflect-pads 1024",
       2: r"mode 2's train-mode statistics need more than 64 frames \(1 \+ L // 441 > 64\)"}


# ============================================================================ 1. the schedule
def _drive(sched, sizes):
    """Windows of a stream fed in blocks of the given sizes and then ended, and pos after each due() call."""
    avail, pos, wins = 0, 0, []
    for n in sizes:
        avail += n
        w, pos = sched.due(pos, avail, ended=False)
        wins += w
    w, pos = sched.due(pos, avail, ended=True)
    assert pos == avail
    return wins + w


def _check_windows(sched, wins, total):
    m, mode = sched.min_len, sched.mode
    assert all(m <= hi - lo <= sched.capacity for lo, hi, _, _ in wins)
    # consecutive windows keep consecutive ranges: window j keeps from pos, the next one from where pos moved to
    starts = [kl for _, _, kl, _ in wins] + [total]
    assert starts[0] == 0 and all(a < b for a, b in zip(starts, starts[1:]))
    for (lo, hi, kl, kh), nxt in zip(wins, starts[1:]):
        assert lo <= kl <= kh <= hi
        if mode == 1:               # keep [kl, next start) cut to the pre-filter's prefix of the window
            assert kh == max(kl, min(nxt, lo + 512 * ((hi - lo) // 512)))
        else:
            assert kh == nxt
    cover = np.zeros(total, np.int32)
    for _, _, kl, kh in wins:
        cover[kl:kh] += 1
    assert cover.max() <= 1                                       # no sample emitted twice
    if mode == 2:
        assert cover.all()
    elif sched.ctx >= 511:                                        # mode 1: only the stream's last samples are lost
        lo, hi = wins[-1][:2]
        lost = (hi - lo) % 512
        assert hi == total and cover[:total - lost].all() and not cover[total - lost:].any()
    return cover


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("chunk,ctx", CONFIGS + [(SR, 511), (SR, 510), (3000, 300), (40000, 600)])
@pytest.mark.parametrize("seed", range(2))
def test_schedule_in_modes_1_and_2(mode, chunk, ctx, seed):
    m = MIN[mode]
    sched = api.StreamSchedule(chunk, ctx, mode)
    assert sched.min_len == m
    if chunk + ctx < m:
        with pytest.raises(ValueError, match=rf"stream_pool: chunk_seconds \+ context_seconds is {chunk + ctx} "
                                             rf"samples, the length of a stream's first window; {MSG[mode]}, so it "
                                             rf"needs at least {m}"):
            sched.check_first_window("stream_pool")
        return
    sched.check_first_window("stream_pool")
    rng = np.random.default_rng(seed)
    totals = [1, m - 1, m, m + 1, m + 511, 2 * m] + [k * chunk + t for k in (1, 3) for t in TAILS + [m - 1, m, 600]]
    totals += [int(rng.integers(m, 6 * max(chunk, SR)))]
    longest = 0
    for total in totals:
        sizes = _blocks(rng, total, max(1, total // 50), max(2, total // 3))
        if total < m:
            with pytest.raises(RuntimeError, match=rf"^restore_stream: fewer than {m} samples in total; {MSG[mode]}$"):
                _drive(sched, sizes)
            continue
        wins = _drive(sched, sizes)
        assert wins == _drive(sched, [total])                     # the windows depend on the total only
        _check_windows(sched, wins, total)
        longest = max([longest] + [hi - lo for lo, hi, _, _ in wins])
    if ctx > 0:                                                   # full windows mid-stream
        assert longest == sched.capacity == chunk + 2 * ctx
    else:
        # without context a flush window always reaches the stream's end (every whole chunk went out as a full
        # window first), so the bound chunk + min_len - 1 holds with room: windows reach a chunk, or min_len
        assert sched.capacity == chunk + m - 1 and longest == max(chunk, m)


def test_mode_0_keeps_its_rule():
    for chunk, ctx in CONFIGS:
        a, b = api.StreamSchedule(chunk, ctx), api.StreamSchedule(chunk, ctx, 0)
        assert a.min_len == b.min_len == 1025 and a.capacity == b.capacity
        for total in (1025, chunk + 1030, 3 * chunk + 7):
            assert _drive(a, [total]) == _drive(b, [total])


@pytest.mark.parametrize("total", [33 * SR, 60 * SR, 65 * SR + 123, 30 * SR + 1536, 95 * SR + 40000])
def test_mode_1_spans_at_30_s_are_restore_inmems_segments(total):
    """With 30 s chunks and no context, window k is segment k and emits what restore_inmem keeps of it."""
    wins = _drive(api.StreamSchedule(api.SEG_LENGTH, 0, 1), [total])
    want = [(a, a + api._net_len(b - a, 1)) for a, b in api.segment_bounds(total)]
    assert [(lo, hi) for lo, hi, _, _ in wins] == api.segment_bounds(total)
    assert [(kl, kh) for _, _, kl, kh in wins] == want
    assert sum(kh - kl for _, _, kl, kh in wins) == api.restore_out_len(total, 1)


def test_a_bad_mode_is_refused():
    for bad in (3, -1, "1"):
        with pytest.raises(ValueError, match="mode must be 0, 1 or 2"):
            api.StreamSchedule(SR, 0, bad)


# ============================================================================ 2. restore_stream against a stub engine
class _EchoEngine:
    """restore_stream's engine calls, recorded; the pre-filter keeps 512 * (L // 512) samples, restore echoes."""
    device = 0
    arena = None

    def __init__(self):
        self.calls = []

    def hf_cut(self, x):
        self.calls.append(("hf_cut", x.shape[1]))
        return x[:, :512 * (x.shape[1] // 512)].clone(), None

    def restore(self, x, mode=0, drop_keys=None):
        key = None if drop_keys is None else tuple(int(v) for v in drop_keys.numpy().view(np.uint64)[0])
        self.calls.append(("restore", x.shape[1], mode, key))
        return x.clone()


@pytest.fixture
def echo(monkeypatch):
    monkeypatch.setattr(api, "_check_cuda", lambda cuda: None)
    monkeypatch.setattr(api, "_upload_keys", lambda rows, dev: torch.from_numpy(rows.view(np.int64)))
    real_to = torch.Tensor.to
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self if (a and isinstance(a[0], str)
                                                                          and a[0].startswith("cuda"))
                        else real_to(self, *a, **k))
    eng = _EchoEngine()
    return api.VoiceFixer.from_engine(eng), eng


@pytest.mark.parametrize("mode,chunk,ctx", [(1, 1.0, 0.5), (1, 0.25, 0.0), (1, 0.5, 0.005), (2, 1.0, 0.5),
                                            (2, 30.0, 0.0)])
def test_restore_stream_runs_each_window_as_restore_inmem_does(echo, mode, chunk, ctx):
    vf, eng = echo
    n = 44100 * 4 + 999 if chunk < 30 else 44100 * 33
    x = np.random.default_rng(0).standard_normal(n).astype(np.float32)
    kw = {"dropout_seed": 2 ** 64 - 3} if mode == 2 else {}
    out = list(vf.restore_stream((x[i:i + 3000] for i in range(0, n, 3000)), chunk, ctx, mode=mode, **kw))
    wins = _drive(api.StreamSchedule(int(round(chunk * SR)), int(round(ctx * SR)), mode), [n])
    assert len(out) == len(wins)
    for y, (lo, hi, kl, kh) in zip(out, wins):
        assert np.array_equal(y, x[kl:kh])
    if mode == 1:
        want = [c for lo, hi, _, _ in wins for c in (("hf_cut", hi - lo), ("restore", 512 * ((hi - lo) // 512), 0, None))]
    else:
        want = [("restore", hi - lo, 2, (2 ** 64 - 3, k)) for k, (lo, hi, _, _) in enumerate(wins)]
    assert eng.calls == want


def test_restore_stream_draws_a_seed_from_torch(echo):
    vf, eng = echo
    x = np.zeros(2 * SR, np.float32)
    torch.manual_seed(11)
    list(vf.restore_stream([x], 1.0, 0.0, mode=2))
    torch.manual_seed(11)
    seed = api.stream_dropout_seed(2, None, "restore_stream")
    assert [c[3] for c in eng.calls] == [(seed, 0), (seed, 1)] and 0 <= seed < 2 ** 64
    assert api.stream_dropout_seed(2, None, "x") != seed          # the generator moved on


def test_restore_stream_refusals(echo):
    vf, eng = echo
    x = np.zeros(SR, np.float32)
    cases = [(dict(mode=1, dropout_seed=5), r"restore_stream: dropout_seed is mode 2's dropout; mode is 1"),
             (dict(mode=0, dropout_seed=5), r"restore_stream: dropout_seed is mode 2's dropout; mode is 0"),
             (dict(mode=2, dropout_seed=-1), r"restore_stream has dropout_seed -1; a dropout seed is an integer"),
             (dict(mode=2, dropout_seed=True), r"restore_stream has dropout_seed True"),
             (dict(mode=2, dropout_seed=2 ** 64), r"restore_stream has dropout_seed 18446744073709551616"),
             (dict(mode=2, chunk_seconds=0.5, context_seconds=0.1),
              rf"restore_stream: chunk_seconds \+ context_seconds is 26460 samples.*at least 28224"),
             (dict(mode=1, chunk_seconds=0.02, context_seconds=0.01),
              rf"restore_stream: chunk_seconds \+ context_seconds is 1323 samples.*at least 1536"),
             (dict(mode=4), "mode must be 0, 1 or 2")]
    for kw, match in cases:
        with pytest.raises(ValueError, match=match):
            list(vf.restore_stream([x], **kw))
    for mode in (1, 2):
        with pytest.raises(RuntimeError, match=rf"restore_stream: fewer than {MIN[mode]} samples in total"):
            list(vf.restore_stream([x[:MIN[mode] - 1]], 1.0, 0.5, mode=mode))
    assert eng.calls == []


# ============================================================================ 3. the pool against a stub engine
def _fake(row, n, mode, key):
    """Stands in for the restore of one window of n samples: depends on each sample, its place, n, the mode and the key;
    in mode 1 on the pre-filter's 512 * (n // 512) samples only, and zeros after them."""
    m = 512 * (n // 512) if mode == 1 else n
    seed, stream = key if key is not None else (0, 0)
    y = (row[:m] * np.float32(0.5) + np.arange(m, dtype=np.float32) * np.float32(1e-4) + np.float32(n * 1e-6)
         + np.float32(mode * 0.25) + np.float32((seed % 997) * 1e-3) + np.float32(stream * 1e-2)).astype(np.float32)
    return np.concatenate([y, np.zeros(n - m, np.float32)])


class _Graph:
    def __init__(self, eng, wav, out, mode, lens, keys):
        self.eng, self.wav, self.out, self.mode, self.lens, self.keys = eng, wav, out, mode, lens, keys

    def replay(self):
        lens = self.lens.tolist()
        keys = [tuple(int(v) for v in r) for r in self.keys.numpy().view(np.uint64)] if self.keys is not None else None
        self.eng.launches.append((self.wav.shape[0], lens, keys))
        for b, n in enumerate(lens):
            assert self.eng.min_len <= n <= self.wav.shape[1]
            y = _fake(self.wav[b, :n].numpy(), n, self.mode, keys[b] if keys else None)
            self.out[b, :n] = torch.from_numpy(y)


class _StubEngine:
    device = 0

    def __init__(self, mode, fit=64):
        self.mode, self.min_len = mode, MIN[mode]
        self.fit, self.launches, self.captures, self.fit_extra = fit, [], [], None

    def max_batch(self, L, extra_per_item=0):
        self.fit_extra = extra_per_item
        return self.fit

    def workspace_bytes(self, B, L):
        return 64

    @staticmethod
    def hf_cut_workspace_bytes(B, L):
        return 100 * B + L

    def graph_workspace_bytes(self, B, L, mode=0):
        return 128

    def make_graph(self, wav, out, mode=0, lens=None, ws=None, drop_keys=None):
        assert mode == self.mode and lens is not None and ws is not None and wav.shape == out.shape
        assert (drop_keys is not None) == (mode == 2)
        if mode == 2:
            assert drop_keys.dtype == torch.int64 and tuple(drop_keys.shape) == (wav.shape[0], 2)
        self.captures.append(wav.shape[0])
        return _Graph(self, wav, out, mode, lens, drop_keys)

    def resample(self, x, items, L_cap):
        y = torch.zeros(len(items), L_cap)
        for b, (rate, n_in, x_off, x_first, x_len, y_first, y_len) in enumerate(items):
            full = np.zeros(n_in, np.float32)
            full[x_first:x_first + x_len] = x[x_off:x_off + x_len].numpy()
            y[b, :y_len] = torch.from_numpy(wavio._resample(full, rate, SR)[y_first:y_first + y_len])
        return y, torch.tensor([it[6] for it in items], dtype=torch.int32)


def _alone(x, rate, chunk, ctx, mode, seed):
    """restore_stream on the stream alone, through the stub's restore: window k keyed (seed, k) in mode 2."""
    y = wavio._resample(x, rate, SR)
    wins = _drive(api.StreamSchedule(chunk, ctx, mode), [len(y)])
    out = [_fake(y[lo:hi], hi - lo, mode, (seed, k) if mode == 2 else None)[kl - lo:kh - lo]
           for k, (lo, hi, kl, kh) in enumerate(wins)]
    return np.concatenate(out)


@pytest.mark.parametrize("mode,chunk_s,ctx_s", [(1, 0.25, 0.1), (1, 0.1, 0.0), (1, 0.2, 0.005), (2, 0.5, 0.25),
                                                (2, 0.7, 0.0)])
@pytest.mark.parametrize("seed", range(3))
def test_pool_equals_each_stream_alone(mode, chunk_s, ctx_s, seed):
    rng = np.random.default_rng(seed)
    max_windows = [1, 2, 3, 5][seed % 4 if mode == 1 else (seed + 1) % 4]
    eng = _StubEngine(mode)
    pool = api.StreamPool(eng, chunk_s, ctx_s, max_windows, device="cpu", mode=mode)
    chunk, ctx = int(round(chunk_s * SR)), int(round(ctx_s * SR))
    specs = []
    for k, rate in enumerate([44100, 8000, 16000, 48000, 44100, 16000]):
        least = -(-(MIN[mode] + 5) * rate // SR)
        n = int(rng.integers(least, least + int(1.5 * rate)))
        x = (0.3 * rng.standard_normal(n)).astype(np.float32)
        s_seed = [2 ** 64 - 1 - k, 12345 + k, 2 ** 63 + k][k % 3]
        specs.append(dict(x=x, rate=rate, cuts=_split(rng, n, rate // 1000, rate // 3), k=0, sid=None, seed=s_seed,
                          start=int(rng.integers(0, 6)), got=[]))
    t = 0
    while any(s["sid"] is None or s["sid"] in pool.streams for s in specs) or pool.pending:
        for s in specs:
            if s["sid"] is None and t >= s["start"]:
                s["sid"] = pool.open(s["rate"], dropout_seed=s["seed"] if mode == 2 else None)
            elif s["sid"] is not None and not s.get("closed"):
                for _ in range(int(rng.integers(0, 4))):
                    if s["k"] < len(s["cuts"]) - 1:
                        pool.push(s["sid"], s["x"][s["cuts"][s["k"]]:s["cuts"][s["k"] + 1]])
                        s["k"] += 1
                if s["k"] == len(s["cuts"]) - 1:
                    pool.close(s["sid"])
                    s["closed"] = True
        if rng.random() < 0.7:
            before = len(eng.launches)
            out = pool.step()
            n = sum(len(v) for v in out.values())
            if n:
                B, lens, keys = eng.launches[-1]
                assert len(eng.launches) == before + 1 and B == pool.bucket(n)
                assert lens[n:] == [MIN[mode]] * (B - n)          # unused rows: the mode's shortest window
                if mode == 2:
                    assert keys[n:] == [(0, 0)] * (B - n)
            for s in specs:
                s["got"] += out.get(s["sid"], []) if s["sid"] is not None else []
        t += 1
        assert t < 10_000
    assert pool.streams == [] and pool.pending == 0
    for s in specs:
        want = _alone(s["x"], s["rate"], chunk, ctx, mode, s["seed"])
        got = np.concatenate(s["got"])
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), s["rate"]
    if mode == 2:                                 # every stream's keys count its windows 0, 1, 2, ... in launch order
        by_seed = {}
        for _, lens, keys in eng.launches:
            for key in keys:
                if key != (0, 0):
                    by_seed.setdefault(key[0], []).append(key[1])
        assert sorted(by_seed) == sorted(s["seed"] for s in specs)
        assert all(v == list(range(len(v))) for v in by_seed.values())
    assert sorted(set(eng.captures)) == sorted(set(B for B, _, _ in eng.launches)) and len(eng.captures) == pool.graph_count


def test_mode_1_fit_counts_the_pre_filter():
    L = api.StreamSchedule(int(0.25 * SR), int(0.1 * SR), 1).capacity
    eng = _StubEngine(1)
    api.StreamPool(eng, 0.25, 0.1, device="cpu", mode=1)
    assert eng.fit_extra == 4 * 3 * L + api.prefilter_bytes(eng, L) + 4 * L
    assert api.prefilter_bytes(eng, L) == eng.hf_cut_workspace_bytes(2, L) - eng.hf_cut_workspace_bytes(1, L) + 4 * L
    eng = _StubEngine(2)
    api.StreamPool(eng, 0.5, 0.25, device="cpu", mode=2)
    assert eng.fit_extra == 4 * 3 * api.StreamSchedule(int(0.5 * SR), int(0.25 * SR), 2).capacity


def test_the_seed_is_per_stream_and_drawn_from_torch_when_not_given():
    pool = api.StreamPool(_StubEngine(2), 0.5, 0.25, device="cpu", mode=2)
    torch.manual_seed(3)
    a = pool.open()
    b = pool.open(16000, dropout_seed=7)
    torch.manual_seed(3)
    assert pool._streams[a].seed == api.stream_dropout_seed(2, None, "x") and pool._streams[b].seed == 7


def _state(pool):
    return ([(sid, s.n, s.pos, s.seed, s.restored, list(s.pending), s.closed) for sid, s in pool._streams.items()],
            list(pool._queue), pool._next_sid)


def test_pool_refusals_name_the_stream_and_change_nothing():
    for mode, (chunk, ctx) in ((1, (0.02, 0.01)), (2, (0.5, 0.1))):
        n = int(round(chunk * SR)) + int(round(ctx * SR))
        with pytest.raises(ValueError, match=rf"stream_pool: chunk_seconds \+ context_seconds is {n} samples, the "
                                             rf"length of a stream's first window; {MSG[mode]}, so it needs at least "
                                             rf"{MIN[mode]}"):
            api.StreamPool(_StubEngine(mode), chunk, ctx, device="cpu", mode=mode)
    with pytest.raises(ValueError, match="mode must be 0, 1 or 2"):
        api.StreamPool(_StubEngine(1), 1.0, 0.5, device="cpu", mode=3)
    for mode in (0, 1):
        if mode:
            pool = api.StreamPool(_StubEngine(1), 1.0, 0.5, device="cpu", mode=1)
        else:
            pool = api.StreamPool(_Mode0Stub(), 1.0, 0.5, device="cpu")
        a = pool.open()
        before = _state(pool)
        with pytest.raises(ValueError, match=rf"stream_pool.open: stream 1: dropout_seed is mode 2's dropout; "
                                             rf"mode is {mode}"):
            pool.open(dropout_seed=3)
        assert _state(pool) == before and pool.open() == a + 1
    eng = _StubEngine(2)
    pool = api.StreamPool(eng, 0.5, 0.25, device="cpu", mode=2)
    a = pool.open(dropout_seed=1)
    before = _state(pool)
    for bad in (-1, 2 ** 64, True, 1.5, "7"):
        with pytest.raises(ValueError, match=re.escape(f"stream_pool.open: stream 1 has dropout_seed {bad!r}; a dropout "
                                                       "seed is an integer in [0, 2^64)")):
            pool.open(dropout_seed=bad)
        assert _state(pool) == before
    assert eng.launches == [] and eng.captures == []


class _Mode0Stub:
    device = 0

    def max_batch(self, L, extra_per_item=0):
        return 4

    def workspace_bytes(self, B, L):
        return 64


@pytest.mark.parametrize("mode,rate", [(1, 44100), (1, 16000), (2, 44100), (2, 8000)])
def test_a_stream_too_short_for_the_mode_is_refused_at_close(mode, rate):
    eng = _StubEngine(mode)
    pool = api.StreamPool(eng, 1.0, 0.5, device="cpu", mode=mode)
    other = pool.open(dropout_seed=5 if mode == 2 else None)
    short = pool.open(rate)
    n = (MIN[mode] - 1) * rate // SR                                     # its 44.1 kHz length stays below the minimum
    assert resample.out_len(n, rate) == MIN[mode] - 1 or rate != SR
    assert resample.out_len(n, rate) < MIN[mode]
    pool.push(other, np.ones(MIN[mode] + 100, np.float32))
    pool.push(short, np.ones(n, np.float32))
    with pytest.raises(RuntimeError, match=rf"stream_pool.close: stream {short}: restore_stream: fewer than {MIN[mode]} "
                                           rf"samples in total; {MSG[mode]}"):
        pool.close(short)
    assert pool.streams == [other] and eng.launches == []
    pool.close(other)
    out = pool.step()
    got = np.concatenate(out[other])
    want = _alone(np.ones(MIN[mode] + 100, np.float32), SR, SR, SR // 2, mode, 5)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)) and pool.streams == []
