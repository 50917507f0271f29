"""A device StreamPool: CUDA blocks in, CUDA blocks out.  The 14-stream mix at 8 / 16 / 44.1 / 48 kHz (some streams
pushed as strided channel views, which stay unchanged) gives blocks bit-identical, block by block, to a host pool
driven by the same calls, in three precisions; after a warm-up nothing waits on the host (torch's sync debug mode, and a
step queued behind a spinning kernel returns while it spins); each step launches the library exactly twice and
captures nothing new; steps and pushes on two CUDA streams give the same blocks, and a stream buffer replaced on a busy
side stream is not handed out early; bad blocks are refused naming the stream, leaving the other streams' outputs
unchanged; and a ten-minute stream holds at most down - 1 samples more input than the host pool does."""
import numpy as np
import pytest
import torch

from test_stream_pool_gpu import CHUNK, CTX, _streams
from voicefixer_b200 import api, resample

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100

_VF = {}


def _vf(states, prec):
    if prec not in _VF:
        from voicefixer_b200.engine import Engine
        _VF[prec] = api.VoiceFixer.from_engine(Engine(states[0], states[1], precision=prec))
    return _VF[prec]


def _sources(specs):
    """{k: the device copy of stream k}: odd streams as column 1 of an interleaved (n, 2) tensor (element stride 2)."""
    out = {}
    for s in specs:
        x = torch.from_numpy(s["x"]).to(DEV)
        if s["k"] % 2:
            x = torch.stack([-x, x], 1)[:, 1]
            assert x.stride(0) == 2
        out[s["k"]] = x
    return out


def _drive_both(host, dev, specs, srcs, rng, tick=None):
    """Opens, feeds, closes and steps both pools with the same calls, in an interleaved order, until every stream is
    done: the host pool gets numpy blocks, the device pool the same samples of srcs as CUDA views.  tick(t), if given,
    runs at the start of every tick.  Returns ({k: [host blocks]}, {k: [device blocks]})."""
    got_h = {s["k"]: [] for s in specs}
    got_d = {s["k"]: [] for s in specs}
    state = {s["k"]: dict(sid=None, off=0, closed=False) for s in specs}
    t = 0
    while not all(st["closed"] for st in state.values()) or host.pending or host.streams:
        if tick is not None:
            tick(t)
        for s in specs:
            st = state[s["k"]]
            if st["sid"] is None:
                if t >= s["start"]:
                    st["sid"] = host.open(s["rate"])
                    assert dev.open(s["rate"]) == st["sid"]
                continue
            if st["closed"]:
                continue
            budget = int(rng.integers(1, 4)) * max(s["block"], s["rate"] // 4)
            fed = 0
            while fed < budget and st["off"] < len(s["x"]):
                a, b = st["off"], st["off"] + s["block"]
                host.push(st["sid"], s["x"][a:b])
                dev.push(st["sid"], srcs[s["k"]][a:b])
                st["off"], fed = b, fed + s["block"]
            if st["off"] >= len(s["x"]):
                host.close(st["sid"])
                dev.close(st["sid"])
                st["closed"] = True
        out_h, out_d = host.step(), dev.step()
        assert {k: len(v) for k, v in out_h.items()} == {k: len(v) for k, v in out_d.items()}
        for s in specs:
            sid = state[s["k"]]["sid"]
            got_h[s["k"]] += out_h.get(sid, [])
            got_d[s["k"]] += out_d.get(sid, [])
        t += 1
        assert t < 5000
    assert dev.pending == 0 and dev.streams == []
    return got_h, got_d


def _same_blocks(h, d, what):
    assert len(h) == len(d), what
    for j, (a, b) in enumerate(zip(h, d)):
        assert b.is_cuda and b.dtype == torch.float32 and b.dim() == 1 and b.is_contiguous(), what
        assert np.array_equal(b.cpu().numpy().view(np.uint32), a.view(np.uint32)), f"{what}: block {j}"


@pytest.mark.parametrize("prec", ["tf32", "fp32", "bf16"])
def test_device_pool_blocks_equal_the_host_pools(states, prec):
    vf = _vf(states, prec)
    specs = _streams(1)
    srcs = _sources(specs)
    keep = {k: x.clone() for k, x in srcs.items()}
    host, dev = vf.stream_pool(CHUNK, CTX, max_windows=5), vf.stream_pool(CHUNK, CTX, max_windows=5)
    got_h, got_d = _drive_both(host, dev, specs, srcs, np.random.default_rng(2))
    assert dev._kind == "device" and host._kind == "host" and dev.graph_count <= len(dev.buckets)
    for s in specs:
        _same_blocks(got_h[s["k"]], got_d[s["k"]], f"{prec}: stream {s['k']} ({s['rate']} Hz)")
        assert sum(b.shape[0] for b in got_d[s["k"]]) == resample.out_len(len(s["x"]), s["rate"])
    torch.cuda.synchronize()
    for k, x in srcs.items():
        assert torch.equal(x, keep[k]), "a pushed tensor was written"


# ============================================================================ no host wait, launches, graphs
def _warm(pool, rates=(SR, 16000)):
    """A step of every bucket size at each rate (the bucket's graph and the rates' taps), then the flush."""
    for rate in rates:
        for B in pool.buckets:
            sids = [pool.open(rate) for _ in range(B)]
            for sid in sids:
                pool.push(sid, torch.full((int(1.6 * rate),), 0.1, device=DEV))
            assert pool.pending == B
            pool.step()
            for sid in sids:
                pool.close(sid)
            while pool.pending:
                pool.step()
    assert pool.graph_count == len(pool.buckets) and pool.streams == []


def _round(pool, rate, each=None):
    """Fresh streams at rate, one window each for every bucket size, then their flush; each(step) wraps every step.
    The blocks are drawn on the device, so that making them does not wait either."""
    outs = []
    for B in pool.buckets:
        sids = [pool.open(rate) for _ in range(B)]
        for sid in sids:
            pool.push(sid, 0.3 * torch.randn(int(1.6 * rate), device=DEV))
        for sid in sids:
            pool.close(sid)
        while pool.pending:
            outs.append(each(pool.step) if each else pool.step())
    return outs


def test_no_host_synchronisation_after_the_warm_up(states):
    vf = _vf(states, "tf32")
    pool = vf.stream_pool(CHUNK, CTX, max_windows=4)
    _warm(pool)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = _round(pool, SR) + _round(pool, 16000)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert pool.graph_count == len(pool.buckets)
    assert all(bool(torch.isfinite(b).all()) for o in outs for bs in o.values() for b in bs)


@pytest.mark.parametrize("rate", [SR, 16000])
def test_a_step_returns_while_earlier_work_still_runs(states, rate):
    vf = _vf(states, "tf32")
    pool = vf.stream_pool(CHUNK, CTX, max_windows=4)
    _warm(pool)
    sid = pool.open(rate)
    x = torch.from_numpy((0.3 * np.random.default_rng(4).standard_normal(5 * rate)).astype(np.float32)).to(DEV)
    torch.cuda.synchronize()
    torch.cuda._sleep(2 * 10 ** 9)                   # ~1 s at 1.98 GHz
    pool.push(sid, x)
    pool.close(sid)
    out = pool.step()
    busy = not torch.cuda.current_stream().query()
    torch.cuda.synchronize()
    assert busy, "push / close / step waited for the work queued before them"
    assert list(out) == [sid] and len(out[sid]) == 4


@pytest.mark.parametrize("rate", [SR, 16000])
def test_each_step_launches_the_library_twice_and_captures_nothing(states, rate):
    vf = _vf(states, "tf32")
    eng = vf._engine
    pool = vf.stream_pool(CHUNK, CTX, max_windows=4)
    _warm(pool)
    counts = []

    def counted(step):
        n0 = eng.launch_count()
        out = step()
        counts.append(eng.launch_count() - n0)
        return out

    outs = _round(pool, rate, each=counted)
    assert counts and counts == [2] * len(counts) and len(outs) == len(counts)
    assert pool.graph_count == len(pool.buckets)


# ============================================================================ CUDA streams
def test_steps_and_pushes_on_two_streams_give_the_same_blocks(states):
    vf = _vf(states, "tf32")
    specs = _streams(5)[4:12]
    srcs = _sources(specs)
    want_h, want_d = _drive_both(vf.stream_pool(CHUNK, CTX, max_windows=3), vf.stream_pool(CHUNK, CTX, max_windows=3),
                                 specs, srcs, np.random.default_rng(6))
    s1, s2 = torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)
    for st in (s1, s2):
        st.wait_stream(torch.cuda.current_stream())
    host, dev = vf.stream_pool(CHUNK, CTX, max_windows=3), vf.stream_pool(CHUNK, CTX, max_windows=3)
    # every tick switches stream: a tick's pushes and the step after them run on one, the next tick's on the other
    ctx = {"s": None}

    def switch(t):
        if ctx["s"] is not None:
            ctx["s"].__exit__(None, None, None)
        ctx["s"] = torch.cuda.stream(s1 if t % 2 else s2)
        ctx["s"].__enter__()

    try:
        got_h, got_d = _drive_both(host, dev, specs, srcs, np.random.default_rng(6), tick=switch)
    finally:
        ctx["s"].__exit__(None, None, None)
    for st in (s1, s2):
        torch.cuda.current_stream().wait_stream(st)
    for s in specs:
        _same_blocks(want_h[s["k"]], got_d[s["k"]], f"stream {s['k']}")
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(want_h[s["k"]], got_h[s["k"]]))


def test_a_buffer_replaced_on_a_side_stream_is_not_reused_early(states):
    """A stream's buffer is allocated on the default stream by a small push.  On a side stream queued behind a kernel
    that spins for about two seconds, a long push outgrows it (the copy out of it is still queued) and a step reads the
    new one.  A block of the old buffer's size allocated on the default stream right after must be other memory, and
    the blocks must equal a host pool's."""
    vf = _vf(states, "tf32")
    rate = 16000
    x = (0.3 * np.random.default_rng(8).standard_normal(6 * rate)).astype(np.float32)
    xd = torch.from_numpy(x).to(DEV)
    host, dev = vf.stream_pool(CHUNK, CTX, max_windows=4), vf.stream_pool(CHUNK, CTX, max_windows=4)
    _warm(dev)                                       # no capture on the side stream: capturing synchronises
    a, b = host.open(rate), dev.open(rate)
    host.push(a, x[:1000])
    dev.push(b, xd[:1000])
    torch.cuda.synchronize()
    s = dev._streams[b]
    old = (s._data.data_ptr(), s._data.numel())
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(4 * 10 ** 9)               # ~2 s at 1.98 GHz
        dev.push(b, xd[1000:])
        out_d = dev.step()
    pending = not side.query()
    fresh = torch.empty(old[1], device=DEV)
    assert fresh.data_ptr() + 4 * fresh.numel() <= old[0] or old[0] + 4 * old[1] <= fresh.data_ptr(), \
        "a replaced stream buffer was handed out early"
    fresh.view(torch.int32).fill_(-1)                # NaN bits, on memory nobody else reads
    side.synchronize()
    assert pending, "the side stream finished before the check: the test saw nothing"
    assert s._data.data_ptr() != old[0], "nothing was replaced"
    host.push(a, x[1000:])
    out_h = host.step()
    host.close(a)
    dev.close(b)
    rest_h, rest_d = [], []
    while host.pending:
        rest_h += host.step().get(a, [])
        rest_d += dev.step().get(b, [])
    _same_blocks(out_h[a] + rest_h, out_d[b] + rest_d, "the stream")


# ============================================================================ refusals and bounds
def test_refusals_name_the_stream_and_leave_the_others_unchanged(states):
    vf = _vf(states, "tf32")
    specs = _streams(3)[4:10]
    srcs = _sources(specs)
    want_h, want_d = _drive_both(vf.stream_pool(CHUNK, CTX, max_windows=3), vf.stream_pool(CHUNK, CTX, max_windows=3),
                                 specs, srcs, np.random.default_rng(7))
    host, dev = vf.stream_pool(CHUNK, CTX, max_windows=3), vf.stream_pool(CHUNK, CTX, max_windows=3)
    good = torch.ones(3000, device=DEV)
    bad = [(good.double(), "a CUDA block has dtype torch.float64"),
           (good.half(), "a CUDA block has dtype torch.float16"),
           (torch.ones(100, 2, device=DEV), r"a CUDA block has shape \(100, 2\); blocks are 1-D"),
           (good[:1].expand(3000), "a CUDA block has element stride 0"),
           (np.ones(3000, np.float32), "a host block in a pool of CUDA blocks"),
           (good.cpu(), "a host block in a pool of CUDA blocks")]
    if torch.cuda.device_count() > 1:
        bad.append((good.to("cuda:1"), "a CUDA block is on cuda:1"))
    done = []

    def refuse(t):
        if done or dev._kind != "device":            # once a CUDA block has made it a device pool
            return
        sid = host.open(16000)
        assert dev.open(16000) == sid
        for block, match in bad:
            before = (dev._streams[sid].n, dev.pending, list(dev._queue))
            with pytest.raises(ValueError, match=rf"stream_pool.push: stream {sid}: " + match):
                dev.push(sid, block)
            assert (dev._streams[sid].n, dev.pending, list(dev._queue)) == before
        with pytest.raises(ValueError, match=rf"stream_pool.push: stream {sid}: a CUDA block in a pool of host"):
            host.push(sid, good)
        for p in (host, dev):                        # a short stream is refused at close, as in the host pool
            p.push(sid, np.ones(300, np.float32) if p is host else good[:300])
            with pytest.raises(RuntimeError, match=rf"stream_pool.close: stream {sid}: restore_stream: fewer than 1025 "
                                                   "samples in total; the front end reflect-pads 1024"):
                p.close(sid)
            assert sid not in p.streams
        done.append(sid)

    got_h, got_d = _drive_both(host, dev, specs, srcs, np.random.default_rng(7), tick=refuse)
    assert len(done) == 1
    for s in specs:
        _same_blocks(want_h[s["k"]], got_d[s["k"]], f"stream {s['k']}")
        _same_blocks(want_h[s["k"]], want_d[s["k"]], f"stream {s['k']} (without refusals)")


def test_a_ten_minute_stream_holds_at_most_down_minus_one_more_samples(states):
    vf = _vf(states, "tf32")
    rate, block = 48000, 4800
    down = resample.ratio(rate)[1]
    x = (0.3 * np.random.default_rng(9).standard_normal(600 * rate)).astype(np.float32)
    xd = torch.from_numpy(x).to(DEV)
    host, dev = vf.stream_pool(CHUNK, CTX, max_windows=2), vf.stream_pool(CHUNK, CTX, max_windows=2)
    a, b = host.open(rate), dev.open(rate)
    got_h, got_d, most = [], [], 0
    for k in range(0, len(x), block):
        host.push(a, x[k:k + block])
        dev.push(b, xd[k:k + block])
        got_h += host.step().get(a, [])
        got_d += dev.step().get(b, [])
        extra = dev._streams[b].buf.shape[0] - host._streams[a].buf.shape[0]
        assert 0 <= extra <= down - 1
        most = max(most, dev._streams[b].buf.shape[0])
    host.close(a)
    dev.close(b)
    while host.pending:
        got_h += host.step().get(a, [])
        got_d += dev.step().get(b, [])
    assert most < 3 * rate                           # a few seconds, not ten minutes
    assert sum(y.shape[0] for y in got_d) == resample.out_len(len(x), rate)
    _same_blocks(got_h, got_d, "the ten-minute stream")
