"""VoiceFixer.stream_pool on the device: many live streams at 44.1, 8, 16 and 48 kHz, opened and closed at different
steps and restored in shared ragged graph replays, each bit-identical to restore_stream on its own (host-resampled)
audio; graph reuse and the resampler's absence on 44.1 kHz steps; and a short stream refused at close."""
import numpy as np
import pytest

from voicefixer_b200 import api, resample, wavio

pytestmark = pytest.mark.gpu
SR = 44100
CHUNK, CTX = 1.0, 0.5

_VF = {}


def _vf(states, prec):
    if prec not in _VF:
        from voicefixer_b200.engine import Engine
        _VF[prec] = api.VoiceFixer.from_engine(Engine(states[0], states[1], precision=prec))
    return _VF[prec]


def _streams(seed):
    """14 streams: (rate, samples, block size in samples, step at which it opens).  Lengths from just over 1025 samples
    at 44.1 kHz to 40 s; blocks from 1 ms to 3 s."""
    rng = np.random.default_rng(seed)
    plan = [(44100, 1026, 0.001), (16000, 373, 0.001), (8000, 187, 0.002), (48000, 1120, 0.05),
            (44100, 40 * 44100, 3.0), (48000, 40 * 48000, 0.1), (16000, 12 * 16000 + 17, 0.5), (8000, 9 * 8000 + 3, 1.0),
            (44100, 5 * 44100 + 1023, 0.02), (16000, 3 * 16000 + 5, 0.001), (48000, 7 * 48000 + 11, 3.0),
            (8000, 2 * 8000 + 1, 0.25), (44100, int(2.5 * 44100), 0.3), (16000, 20 * 16000, 0.01)]
    out = []
    for k, (rate, n, block_s) in enumerate(plan):
        x = (0.3 * rng.standard_normal(n)).astype(np.float32)
        out.append(dict(x=x, rate=rate, block=max(1, int(block_s * rate)), start=int(rng.integers(0, 8)), k=k))
    return out


def _drive(pool, specs, rng, tick=None):
    """Opens, feeds and closes the streams in an interleaved order and steps the pool until every stream is done.
    tick(pool, t), if given, runs at the start of every tick t.  Returns {k: concatenated output}."""
    got = {s["k"]: [] for s in specs}
    state = {s["k"]: dict(sid=None, off=0, closed=False) for s in specs}
    t = 0
    while not all(st["closed"] for st in state.values()) or pool.pending or pool.streams:
        if tick is not None:
            tick(pool, t)
        for s in specs:
            st = state[s["k"]]
            if st["sid"] is None:
                if t >= s["start"]:
                    st["sid"] = pool.open(s["rate"])
                continue
            if st["closed"]:
                continue
            budget = int(rng.integers(1, 4)) * max(s["block"], s["rate"] // 4)   # about 0.25-0.75 s of audio per tick
            fed = 0
            while fed < budget and st["off"] < len(s["x"]):
                pool.push(st["sid"], s["x"][st["off"]:st["off"] + s["block"]])
                st["off"] += s["block"]
                fed += s["block"]
            if st["off"] >= len(s["x"]):
                pool.close(st["sid"])
                st["closed"] = True
        out = pool.step()
        for s in specs:
            sid = state[s["k"]]["sid"]
            if sid in out:
                got[s["k"]] += out[sid]
        t += 1
        assert t < 5000
    return {k: np.concatenate(v) for k, v in got.items()}


def _alone(vf, s):
    y = wavio._resample(s["x"], s["rate"], SR)
    blocks = [y[i:i + 4410] for i in range(0, len(y), 4410)]
    return np.concatenate(list(vf.restore_stream(blocks, chunk_seconds=CHUNK, context_seconds=CTX)))


@pytest.mark.parametrize("prec", ["tf32", "fp32"])
def test_pool_equals_restore_stream_per_stream(states, prec):
    vf = _vf(states, prec)
    specs = _streams(1)
    pool = vf.stream_pool(CHUNK, CTX, max_windows=5)
    got = _drive(pool, specs, np.random.default_rng(2))
    assert pool.graph_count <= len(pool.buckets)
    for s in specs:
        want = _alone(vf, s)
        g = got[s["k"]]
        assert g.shape[0] == resample.out_len(len(s["x"]), s["rate"]), (s["k"], s["rate"])
        assert g.shape == want.shape and np.array_equal(g.view(np.uint32), want.view(np.uint32)), \
            f"stream {s['k']} ({s['rate']} Hz, {len(s['x'])} samples) differs from restore_stream on its own audio"


def test_graphs_are_reused_and_44100_steps_launch_no_resampler(states):
    vf = _vf(states, "tf32")
    eng = vf._engine
    pool = vf.stream_pool(CHUNK, CTX, max_windows=4)
    assert pool.buckets == [1, 2, 4]
    rng = np.random.default_rng(5)

    def round_(with_16k):
        """Steps of 1, 2 and 4 windows, one per fresh stream (1.6 s each: the first window is due), the last stream at
        16 kHz if with_16k; then the flush windows.  Returns the library launches of each first step."""
        launches = []
        for n in (1, 2, 4):
            rates = [44100] * (n - 1) + [16000 if with_16k else 44100]
            sids = [pool.open(r) for r in rates]
            for sid, r in zip(sids, rates):
                pool.push(sid, (0.3 * rng.standard_normal(int(1.6 * r))).astype(np.float32))
            assert pool.pending == n
            before = eng.launch_count()
            out = pool.step()
            launches.append(eng.launch_count() - before)
            assert sorted(out) == sids
            for sid in sids:
                pool.close(sid)
            while pool.pending:
                pool.step()
            assert pool.streams == []
        return launches

    round_(False)
    round_(True)                                   # warm-up: every bucket captured, the 16 kHz taps uploaded
    assert pool.graph_count == 3
    assert round_(False) == [0, 0, 0]              # a replay launches nothing through the library, nor is a resampler run
    assert round_(True) == [1, 1, 1]               # with a 16 kHz window: the resampler's one launch
    assert pool.graph_count == 3


def test_a_short_stream_refused_at_close_leaves_the_others_unchanged(states):
    vf = _vf(states, "tf32")
    specs = _streams(3)[4:10]
    want = _drive(vf.stream_pool(CHUNK, CTX, max_windows=3), specs, np.random.default_rng(7))
    refused = []

    def refuse_one(pool, t):
        if t == 3:                                 # the other streams are open and have windows in flight
            sid = pool.open(16000)
            pool.push(sid, np.ones(300, np.float32))
            with pytest.raises(RuntimeError, match=rf"stream_pool.close: stream {sid}: restore_stream: fewer than 1025 "
                                                   "samples in total; the front end reflect-pads 1024"):
                pool.close(sid)
            assert sid not in pool.streams
            refused.append(sid)

    got = _drive(vf.stream_pool(CHUNK, CTX, max_windows=3), specs, np.random.default_rng(7), tick=refuse_one)
    assert len(refused) == 1
    for s in specs:
        assert np.array_equal(got[s["k"]].view(np.uint32), want[s["k"]].view(np.uint32))
