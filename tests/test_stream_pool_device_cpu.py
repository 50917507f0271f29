"""The pure half of a device StreamPool, without a GPU: the rows one step gathers (vfx_resample_src items on each
stream's held input, rebased to a multiple of down) read exactly the inputs and taps the host path reads, and the rows
it emits (vfx_scatter_rows items with a source offset) tile each window's kept span once; a device stream drops its
old input as the host stream does, rounded down to a multiple of down; vfx_scatter_rows refuses a bad source offset
before any CUDA call; and a pool refuses a block of the wrong kind, or a CUDA block it cannot take, naming the stream
and changing nothing (fake tensor-like blocks stand in for CUDA tensors)."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from voicefixer_b200 import api, resample

SR = 44100
RATES = [8000, 11025, 16000, 22050, 44100, 48000, 96000]


def _reads(n_in, rate, J):
    """For outputs J (array) of a recording of n_in samples at rate: (first input, last input, tap of the first input),
    the scalar restatement of the resampler's sum (resample.py): inputs i = first .. last, ascending, tap p - i * up."""
    up, down = resample.ratio(rate)
    h, rem = resample.taps(rate)
    p = (J + rem) * down
    first = np.maximum(0, -(-(p - len(h) + 1) // up))
    last = np.minimum(n_in - 1, p // up)
    return first, last, p - first * up


def _check_rebased(rate, base, n, window):
    """The gather item of one window against the whole-stream arithmetic, output by output."""
    (n_in, y_first, y_len), (src_off, k) = [t[0] for t in api.stream_rows([(rate, base, n, window)])]
    lo, hi, keep_lo, keep_hi = window
    assert n_in == n - base and y_len == hi - lo and src_off == keep_lo - lo and k == keep_hi - keep_lo
    assert 0 <= y_first and y_first + y_len <= resample.out_len(n_in, rate)       # what vfx_resample_src validates
    if resample.ratio(rate) == (1, 1):
        assert y_first == lo - base and lo >= base                              # a copy of the held samples
        return
    J = np.arange(lo, hi, dtype=np.int64)
    f, l, t = _reads(n, rate, J)                                                # the stream as one recording
    f2, l2, t2 = _reads(n_in, rate, J - lo + y_first)                           # the held input as one recording
    assert (f >= base).all() or base == 0
    assert np.array_equal(f2 + base, f) and np.array_equal(l2 + base, l) and np.array_equal(t2, t)
    first, stop = resample.window(n, rate, lo, hi)                              # the staged path's window
    live = l >= f
    assert first == f[live].min() and stop == l[live].max() + 1


@pytest.mark.parametrize("rate", RATES)
def test_rebased_rows_read_the_same_inputs_and_taps(rate):
    """Random stream extents and due windows; base is what the pool's trim keeps: the first input of a point at or
    before the window's start, rounded down to a multiple of down."""
    rng = np.random.default_rng(rate)
    up, down = resample.ratio(rate)
    for _ in range(30):
        n = int(rng.integers(5 * rate, 120 * rate))
        avail = resample.available(n, rate)
        L = int(rng.integers(1025, 3 * SR))
        lo = int(rng.integers(0, avail - L))
        keep = int(rng.integers(max(0, lo - 2 * SR), lo + 1))
        first, stop = resample.window(n, rate, keep, keep + 1)
        base = first - first % down if stop > first else 0
        keep_lo = int(rng.integers(lo, lo + L))
        _check_rebased(rate, base, n, (lo, lo + L, keep_lo, int(rng.integers(keep_lo + 1, lo + L + 1))))
    if down > 1:
        with pytest.raises(ValueError, match=f"base 1 is not a multiple of down = {down}"):
            api.stream_rows([(rate, 1, 10 ** 6, (SR, 2 * SR, SR, 2 * SR))])


class _Stub:
    """The engine half the pool's bookkeeping reads."""
    device = 0

    def max_batch(self, L, extra_per_item=0):
        return 64

    def workspace_bytes(self, B, L):
        return 64


def _drive(rate, seed, chunk=0.5, ctx=0.25, seconds=30.0):
    """One stream through the pool's schedule and trim twice, as a host _Stream and as a _DevStream on CPU tensors, with
    the same blocks and steps (each step restores a random number of the oldest pending windows).  Checks the drop
    accounting and the rows of every window as it is restored; returns the kept spans in emit order."""
    rng = np.random.default_rng(seed)
    pool = api.StreamPool(_Stub(), chunk, ctx, max_windows=4, device="cpu")
    host, dev = api._Stream(rate), api._DevStream(rate, "cpu")
    down = resample.ratio(rate)[1]
    x = rng.standard_normal(int(seconds * rate)).astype(np.float32)
    spans, k, ended = [], 0, False
    while not ended or host.pending:
        if k < len(x):
            m = int(rng.integers(1, rate // 3))
            for s in (host, dev):
                s.append(x[k:k + m] if s is host else torch.from_numpy(x[k:k + m]))
            k += m
            for s in (host, dev):
                pool._schedule(0, s, resample.available(s.n, rate), ended=False)
        elif not ended:
            for s in (host, dev):
                pool._schedule(0, s, resample.out_len(s.n, rate), ended=True)
            ended = True
        assert list(host.pending) == list(dev.pending)
        for _ in range(int(rng.integers(0, 3))):
            if not host.pending:
                break
            w = host.pending[0]
            _check_rebased(rate, dev.base, dev.n, w)
            (_, y_first, y_len), (src_off, n_keep) = [t[0] for t in api.stream_rows([(rate, dev.base, dev.n, w)])]
            spans.append((w[0] + src_off, w[0] + src_off + n_keep))
            for s in (host, dev):
                s.pending.popleft()
                pool._trim(s)
        # the drop accounting: the device stream holds the host stream's input from a multiple of down before it
        assert dev.base == host.base - host.base % down and dev.base % down == 0
        assert dev.n == host.n and dev.buf.shape[0] - host.buf.shape[0] == host.base - dev.base <= down - 1
        assert np.array_equal(dev.buf.numpy(), x[dev.base:dev.n])
        assert dev.pending == host.pending
    return spans, resample.out_len(len(x), rate)


@pytest.mark.parametrize("rate", RATES)
def test_device_streams_drop_like_host_streams_and_emit_every_sample_once(rate):
    for seed, (chunk, ctx) in enumerate([(0.5, 0.25), (0.1, 0.0), (1.0, 0.5)]):
        spans, total = _drive(rate, seed, chunk, ctx, seconds=12.0 if chunk < 0.5 else 30.0)
        cover = np.zeros(total, np.int32)
        for a, b in spans:
            cover[a:b] += 1
        assert (cover == 1).all() and [a for a, _ in spans[1:]] == [b for _, b in spans[:-1]]


def test_held_input_stays_bounded():
    """Twenty minutes at 48 kHz in 0.1 s blocks: the held input and its buffer stay a few seconds long."""
    rate, block = 48000, 4800
    pool = api.StreamPool(_Stub(), 1.0, 0.5, max_windows=4, device="cpu")
    dev = api._DevStream(rate, "cpu")
    z = torch.zeros(block)
    for _ in range(20 * 600):
        dev.append(z)
        pool._schedule(0, dev, resample.available(dev.n, rate), ended=False)
        while dev.pending:
            dev.pending.popleft()
            pool._trim(dev)
        assert dev.buf.shape[0] < 3 * rate and dev._data.shape[0] < 8 * rate


# ============================================================================ vfx_scatter_rows' source offset
def test_scatter_item_keeps_its_size_and_a_zero_source_offset_by_default():
    from voicefixer_b200 import _lib
    assert ctypes.sizeof(_lib.ScatterItem) == 32 and _lib.ScatterItem.src_off.offset == 28
    assert (_lib.ScatterItem * 3)()[2].src_off == 0


# Device pointers are never dereferenced by a refused call: fake addresses stand in for them.
@pytest.mark.parametrize("src_off,n,match", [
    (-1, 1100, "item 1: source columns [-1, 1099) are not inside its row of ldx = 4096"),
    (3000, 1100, "item 1: source columns [3000, 4100) are not inside its row of ldx = 4096"),
    (0, 4097, "item 1: len 4097 is not in [0, ldx = 4096]"),
    (2996, 1100, None),
])
def test_scatter_rows_refuses_a_bad_source_offset_before_any_cuda_call(src_off, n, match):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    table = (_lib.ScatterItem * 2)()
    for b, (off, k, so) in enumerate([(0, 1000, 5), (5000, n, src_off)]):
        table[b].dst, table[b].dst_elems, table[b].dst_off, table[b].len, table[b].src_off = 0x100000, 10000, off, k, so
    if match is None:                            # in range: only the source offset of item 0 is then made bad
        table[0].src_off = 3097
        match = "item 0: source columns [3097, 4097)"
    rc = lib.vfx_scatter_rows(0x1000, 2, 4096, table, 0x2000, 4096, None)
    assert rc == -1 and match.encode() in lib.vfx_last_error(), lib.vfx_last_error()


# ============================================================================ the pool's kind and its refusals
def _fake(shape=(4410,), dtype=torch.float32, device="cuda:0", stride=1):
    """Stands in for a CUDA tensor: the pool reads only is_cuda, device, dtype, shape and stride before taking it."""
    return SimpleNamespace(is_cuda=True, device=torch.device(device), dtype=dtype, shape=shape, stride=lambda d: stride)


def _state(pool):
    return ([(sid, s.n, s.base, s.pos, list(s.pending), s.closed, type(s)) for sid, s in pool._streams.items()],
            list(pool._queue), pool._kind)


BAD_CUDA = [
    (_fake(dtype=torch.float64), "a CUDA block has dtype torch.float64; CUDA blocks must be torch.float32"),
    (_fake((4410, 2)), r"a CUDA block has shape \(4410, 2\); blocks are 1-D"),
    (_fake(()), r"a CUDA block has shape \(\)"),
    (_fake(device="cuda:1"), "a CUDA block is on cuda:1; this pool runs on cuda:0"),
    (_fake(stride=0), r"a CUDA block has element stride 0 \(an expanded tensor\)"),
]


@pytest.mark.parametrize("block,match", BAD_CUDA)
def test_a_cuda_block_that_cannot_be_taken_is_refused_and_fixes_nothing(block, match):
    pool = api.StreamPool(_Stub(), 0.25, 0.1, max_windows=3, device="cuda:0")
    a, b = pool.open(), pool.open(16000)
    before = _state(pool)
    with pytest.raises(ValueError, match=rf"stream_pool.push: stream {b}: " + match):
        pool.push(b, block)
    assert _state(pool) == before and pool._kind is None
    pool.push(a, np.ones(20000, np.float32))     # the pool is still free to become a host pool
    assert pool._kind == "host" and pool.pending == 1


def test_a_cuda_block_in_a_host_pool_is_refused_and_changes_nothing():
    pool = api.StreamPool(_Stub(), 0.25, 0.1, max_windows=3, device="cuda:0")
    a, b = pool.open(), pool.open(48000)
    pool.push(a, np.ones(20000, np.float32))
    pool.push(b, np.ones(3000, np.float32))
    before = _state(pool)
    for sid in (a, b):
        with pytest.raises(ValueError, match=rf"stream_pool.push: stream {sid}: a CUDA block in a pool of host "
                                             "blocks; the first block pushed fixes a pool's kind for its lifetime"):
            pool.push(sid, _fake())
    assert _state(pool) == before
    with pytest.raises(ValueError, match=r"stream_pool.push: stream 9 is not open"):   # an unknown stream comes first
        pool.push(9, _fake())
