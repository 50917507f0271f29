"""Streams in modes 1 and 2 on the device: restore_stream with 30 s chunks and no context equals restore_inmem in mode 1
and in seeded mode 2; host and device pools over the 14-stream mix at 8 / 16 / 44.1 / 48 kHz (each stream lengthened to
the mode's shortest window) give each stream restore_stream's bits on its own host-resampled audio with its own seed, in
tf32 and fp32, and device blocks equal host blocks in bf16 too; a seeded stream's output does not depend on its
neighbours or max_windows, and its seed matters; and after a warm-up a device step in either mode waits for nothing,
launches the library twice and captures nothing."""
import numpy as np
import pytest
import torch

from test_stream_pool_device_gpu import _round, _same_blocks, _warm
from test_stream_pool_gpu import CHUNK, CTX, _streams
from voicefixer_b200 import api, resample, wavio

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100

_VF = {}


def _vf(states, prec):
    if prec not in _VF:
        from voicefixer_b200.engine import Engine
        _VF[prec] = api.VoiceFixer.from_engine(Engine(states[0], states[1], precision=prec))
    return _VF[prec]


def _noise(n, seed):
    return (0.3 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


# ============================================================================ restore_stream against restore_inmem
@pytest.mark.parametrize("mode", [1, 2])
def test_restore_stream_at_30_s_equals_restore_inmem(states, mode):
    vf = _vf(states, "tf32")
    x = _noise(33 * SR, 1)
    kw = {"dropout_seed": 2 ** 64 - 11} if mode == 2 else {}
    want = vf.restore_inmem(x, cuda=True, mode=mode, **kw)[0]
    blocks = [x[i:i + 4410] for i in range(0, len(x), 4410)]
    got = np.concatenate(list(vf.restore_stream(blocks, chunk_seconds=30.0, context_seconds=0.0, mode=mode, **kw)))
    assert got.shape == want.shape == (api.restore_out_len(len(x), mode),)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ============================================================================ pools against restore_stream
def _mix(seed, mode):
    """The 14-stream mix, each stream at least the mode's shortest window long at 44.1 kHz, with a distinct seed."""
    m = api.StreamSchedule.MIN_LEN[mode]
    specs = _streams(seed)
    for s in specs:
        need = -(-(m + 3) * s["rate"] // SR)
        if len(s["x"]) < need:
            s["x"] = _noise(need, 100 + s["k"])
        s["seed"] = [2 ** 64 - 1 - s["k"], 7919 * s["k"], 2 ** 63 + s["k"]][s["k"] % 3]
    return specs


def _drive(pools, specs, rng, blocks):
    """Opens (with each stream's seed in mode 2), feeds, closes and steps every pool with the same calls in an
    interleaved order until every stream is done; blocks[p](s, a, b) gives pool p's block of samples [a, b) of stream s.
    Returns one {k: [blocks]} per pool."""
    got = [{s["k"]: [] for s in specs} for _ in pools]
    state = {s["k"]: dict(sid=None, off=0, closed=False) for s in specs}
    t = 0
    while not all(st["closed"] for st in state.values()) or any(p.pending or p.streams for p in pools):
        for s in specs:
            st = state[s["k"]]
            if st["sid"] is None:
                if t >= s["start"]:
                    seed = s["seed"] if pools[0].mode == 2 else None
                    sids = {p.open(s["rate"], dropout_seed=seed) for p in pools}
                    assert len(sids) == 1
                    st["sid"] = sids.pop()
                continue
            if st["closed"]:
                continue
            budget = int(rng.integers(1, 4)) * max(s["block"], s["rate"] // 4)
            fed = 0
            while fed < budget and st["off"] < len(s["x"]):
                a, b = st["off"], st["off"] + s["block"]
                for p, blk in zip(pools, blocks):
                    p.push(st["sid"], blk(s, a, b))
                st["off"], fed = b, fed + s["block"]
            if st["off"] >= len(s["x"]):
                for p in pools:
                    p.close(st["sid"])
                st["closed"] = True
        for p, g in zip(pools, got):
            out = p.step()
            for s in specs:
                g[s["k"]] += out.get(state[s["k"]]["sid"], [])
        t += 1
        assert t < 5000
    return got


def _host_and_device(vf, mode, specs, max_windows=5, seed=2):
    srcs = {s["k"]: torch.from_numpy(s["x"]).to(DEV) for s in specs}
    host = vf.stream_pool(CHUNK, CTX, max_windows=max_windows, mode=mode)
    dev = vf.stream_pool(CHUNK, CTX, max_windows=max_windows, mode=mode)
    got_h, got_d = _drive([host, dev], specs, np.random.default_rng(seed),
                          [lambda s, a, b: s["x"][a:b], lambda s, a, b: srcs[s["k"]][a:b]])
    assert host._kind == "host" and dev._kind == "device"
    assert host.graph_count <= len(host.buckets) and dev.graph_count <= len(dev.buckets)
    return got_h, got_d


def _alone(vf, s, mode):
    y = wavio._resample(s["x"], s["rate"], SR)
    kw = {"dropout_seed": s["seed"]} if mode == 2 else {}
    return np.concatenate(list(vf.restore_stream([y[i:i + 4410] for i in range(0, len(y), 4410)], CHUNK, CTX, mode=mode,
                                                 **kw)))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("prec", ["tf32", "fp32"])
def test_pools_equal_restore_stream_per_stream(states, mode, prec):
    vf = _vf(states, prec)
    specs = _mix(1, mode)
    got_h, got_d = _host_and_device(vf, mode, specs)
    for s in specs:
        want = _alone(vf, s, mode)
        g = np.concatenate(got_h[s["k"]])
        assert g.shape == want.shape and np.array_equal(g.view(np.uint32), want.view(np.uint32)), \
            f"mode {mode}, {prec}: stream {s['k']} ({s['rate']} Hz, {len(s['x'])} samples) differs from restore_stream"
        _same_blocks(got_h[s["k"]], got_d[s["k"]], f"mode {mode}, {prec}: stream {s['k']}")
        if mode == 2:
            assert g.shape[0] == resample.out_len(len(s["x"]), s["rate"])


@pytest.mark.parametrize("mode", [1, 2])
def test_device_blocks_equal_host_blocks_in_bf16(states, mode):
    vf = _vf(states, "bf16")
    specs = _mix(3, mode)
    got_h, got_d = _host_and_device(vf, mode, specs, max_windows=3, seed=4)
    for s in specs:
        _same_blocks(got_h[s["k"]], got_d[s["k"]], f"mode {mode}, bf16: stream {s['k']}")


def test_a_seeded_stream_ignores_its_neighbours_and_the_batching(states):
    vf = _vf(states, "tf32")
    specs = _mix(5, 2)
    target = dict(specs[4], k=99, start=1, seed=31337)              # 40 s at 44.1 kHz
    runs = []
    for others, max_windows in ((specs[5:8], 2), (specs[8:14], 5), ([], 1)):
        pool = vf.stream_pool(CHUNK, CTX, max_windows=max_windows, mode=2)
        srcs = {s["k"]: torch.from_numpy(s["x"]).to(DEV) for s in others + [target]}
        got = _drive([pool], others + [target], np.random.default_rng(max_windows),
                     [lambda s, a, b: srcs[s["k"]][a:b]])[0]
        runs.append(torch.cat(got[99]).cpu().numpy())
    assert all(np.array_equal(r.view(np.uint32), runs[0].view(np.uint32)) for r in runs[1:])
    pool = vf.stream_pool(CHUNK, CTX, max_windows=2, mode=2)
    other = _drive([pool], [dict(target, seed=31338)], np.random.default_rng(0), [lambda s, a, b: s["x"][a:b]])[0]
    assert not np.array_equal(np.concatenate(other[99]), runs[0])


# ============================================================================ no host wait, launches, graphs
@pytest.mark.parametrize("mode", [1, 2])
def test_device_steps_wait_for_nothing_launch_twice_and_capture_nothing(states, mode):
    vf = _vf(states, "tf32")
    eng = vf._engine
    pool = vf.stream_pool(CHUNK, CTX, max_windows=4, mode=mode)
    _warm(pool)
    counts = []

    def counted(step):
        n0 = eng.launch_count()
        out = step()
        counts.append(eng.launch_count() - n0)
        return out

    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = _round(pool, SR, each=counted) + _round(pool, 16000, each=counted)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert counts and counts == [2] * len(counts) and len(outs) == len(counts)
    assert pool.graph_count == len(pool.buckets)
    assert all(bool(torch.isfinite(b).all()) for o in outs for bs in o.values() for b in bs)
