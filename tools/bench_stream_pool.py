"""Many live streams through one StreamPool against one restore_stream generator per stream, synthetic weights, in each
mode of --mode (0, 1 or 2, one session; in mode 2 stream i has dropout seed i in the pool and in its generator).
Each stream is a seeded synthetic utterance of --seconds at 44.1 kHz, fed in --block-second blocks, restored in chunks
of --chunk seconds with --ctx seconds of context on each side.  Two pools run: a host pool (numpy blocks in and out)
and a device pool (the same blocks as CUDA tensors in and out, no host staging and no wait in a step).

  (a) throughput: all input available.  The pool is fed one block per stream in turn and steps whenever a full batch
      of windows is due (and at the end until it is empty); the generators are driven round-robin, one window each in
      turn.  Stream-audio seconds emitted per wall second, host clock around work that ends in a device synchronise.
      The run asserts that every stream's pool output is bit-identical to its generator's, and the device pool's to
      the host pool's; the device pool's wall time ends in a device synchronise.
  (b) real time: blocks arrive on a simulated clock (stream i starts at a seeded offset in [0, chunk) s and then gets
      one block per block period).  The pool steps whenever windows are due.  A window's lag is the time from the
      arrival of the block that made it due to the end of the step that emits it; N streams keep real time when no
      lag reaches one chunk (otherwise each step leaves more than it took).  Reports p50 / p99 step time, the largest
      lag and the median time to first audio (from a stream's start to the end of the step that emits its first block).
      For the device pool a step ends when its work on the device is done (a CUDA event after it, timed from an event
      recorded at the start), not when step() returns; the driver steps it again once that event has passed, so that
      windows gather into batches while the device is busy, as they do while a host pool's step waits.
  (c) host share: the share of (a)'s step time outside the graph replay (staging on the host, uploads, resampling,
      copy-back, cutting), from the summed wall time of the steps and CUDA events around each replay inside them.
      For the device pool the step time is the device time between CUDA events recorded before and after each step.

Prints the card's name, power limit and maximum SM clock, then one JSON line with the results of each mode.  Usage:
  python tools/bench_stream_pool.py [--streams 1,8,32,64,128] [--rt-streams 8,32,64,128,192,256] [--seconds 20]
                                    [--mode 0,1,2]"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import deque

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SR = 44100


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def utterances(n, seconds, seed):
    """n seeded streams: 16 synthetic utterances, each stream one of them rotated by a seeded offset."""
    from voicefixer_b200 import synthetic
    base = synthetic.make_utterances(min(n, 16), seconds=seconds, seed=seed)
    rng = np.random.default_rng(seed)
    return [np.roll(base[i % len(base)], int(rng.integers(0, base.shape[1]))) for i in range(n)]


def blocks_of(x, block):
    return [x[i:i + block] for i in range(0, len(x), block)]


def warm(pool, device=False):
    """Captures the graph of every bucket: a step of B windows, one per fresh stream, for each bucket B."""
    for B in pool.buckets:
        sids = [pool.open() for _ in range(B)]
        for sid in sids:
            x = np.zeros(int((pool._sched.chunk + pool._sched.ctx)), np.float32) + 0.1
            pool.push(sid, torch.from_numpy(x).cuda() if device else x)
        pool.step()
        for sid in sids:
            pool.close(sid)
        while pool.pending:
            pool.step()
    assert pool.graph_count == len(pool.buckets)


def seed_of(pool, i):
    """Stream i's dropout seed: i in mode 2, none otherwise."""
    return i if pool.mode == 2 else None


def run_pool(pool, streams, block, timed_steps=None, device=False):
    """(a) for the pool: returns ([output per stream], wall seconds).  device: push CUDA tensors (the streams are
    uploaded before the clock starts) and time to a device synchronise; timed_steps then gets (bucket, start event, end
    event) per step."""
    if device:
        streams = [torch.from_numpy(x).cuda() for x in streams]
        torch.cuda.synchronize()
    blocks = [blocks_of(x, block) for x in streams]
    got = [[] for _ in streams]
    t0 = time.perf_counter()
    sids = [pool.open(dropout_seed=seed_of(pool, i)) for i in range(len(streams))]
    index = {sid: i for i, sid in enumerate(sids)}

    def step():
        ts = time.perf_counter()
        n = min(pool.pending, pool.max_windows)
        if device and timed_steps is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            out = pool.step()
            ev[1].record()
            timed_steps.append((pool.bucket(n), ev[0], ev[1]))
        else:
            out = pool.step()
            if timed_steps is not None:
                timed_steps.append((pool.bucket(n), time.perf_counter() - ts))
        for sid, ys in out.items():
            got[index[sid]] += ys

    for k in range(max(len(b) for b in blocks)):
        for sid, b in zip(sids, blocks):
            if k < len(b):
                pool.push(sid, b[k])
                if k == len(b) - 1:
                    pool.close(sid)
        while pool.pending >= pool.max_windows:
            step()
    while pool.pending:
        step()
    if device:
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    if device:
        return [torch.cat(g).cpu().numpy() for g in got], wall
    return [np.concatenate(g) for g in got], wall


def run_round_robin(vf, streams, block, args, mode):
    """(a) for N restore_stream generators driven round-robin, one window each in turn."""
    gens = [vf.restore_stream(iter(blocks_of(x, block)), chunk_seconds=args.chunk, context_seconds=args.ctx, mode=mode,
                              dropout_seed=i if mode == 2 else None)
            for i, x in enumerate(streams)]
    got = [[] for _ in streams]
    t0 = time.perf_counter()
    live = list(range(len(gens)))
    while live:
        for i in list(live):
            y = next(gens[i], None)
            if y is None:
                live.remove(i)
            else:
                got[i].append(y)
    torch.cuda.synchronize()
    return [np.concatenate(g) for g in got], time.perf_counter() - t0


def time_replays(pool):
    """Wraps the replay of each of the pool's graphs in CUDA events; returns the list that receives (start, end) of
    every replay from then on, so the device time of the replays inside the steps can be summed afterwards."""
    spans = []
    for g in pool._graphs.values():
        def replay(g=g, orig=g.replay):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            orig()
            ev[1].record()
            spans.append(ev)
        g.replay = replay
    return spans


def replay_ms(pool, B, reps=10):
    g = pool._graphs[B]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    g.replay()
    ev[0].record()
    for _ in range(reps):
        g.replay()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def run_real_time(pool, streams, block, args, rng, device=False):
    """(b): returns dict(steps, p50/p99 step ms, max / p99 lag s, median time to first audio s, keeps_real_time).
    device: push CUDA tensors; a step ends when an event recorded after it completes on the device."""
    period = block / SR
    if device:
        streams = [torch.from_numpy(x).cuda() for x in streams]
    blocks = [blocks_of(x, block) for x in streams]
    start = rng.uniform(0, args.chunk, size=len(streams))
    sids = [pool.open(dropout_seed=seed_of(pool, i)) for i in range(len(streams))]
    index = {sid: i for i, sid in enumerate(sids)}
    next_k = [0] * len(streams)
    due = deque()                                   # arrival time of the push that made each pending window due
    step_ms, lags, first = [], [], [None] * len(streams)
    ends = []                                       # device pool: (end event, [(stream, arrival) per window emitted])
    torch.cuda.synchronize()
    ev0 = torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    ev0.record()
    left = len(streams)
    while left or pool.pending:
        now = time.perf_counter() - t0
        for i in range(len(streams)):
            while next_k[i] < len(blocks[i]) and start[i] + (next_k[i] + 1) * period <= now:
                before = pool.pending
                pool.push(sids[i], blocks[i][next_k[i]])
                next_k[i] += 1
                if next_k[i] == len(blocks[i]):
                    pool.close(sids[i])
                    left -= 1
                arrived = start[i] + next_k[i] * period
                due.extend([arrived] * (pool.pending - before))
        if not pool.pending or (device and ends and not ends[-1][0].query()):
            time.sleep(0.0005)                      # a device pool steps again once its previous step's work is done
            continue
        ts = time.perf_counter()
        out = pool.step()
        te = time.perf_counter()
        step_ms.append((te - ts) * 1e3)
        emitted = [(index[sid], due.popleft()) for sid, ys in out.items() for _ in ys]
        if device:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            ends.append((ev, emitted))
            continue
        for i, arrived in emitted:
            lags.append(te - t0 - arrived)
            if first[i] is None:
                first[i] = te - t0 - start[i]
    if device:
        torch.cuda.synchronize()
        for ev, emitted in ends:
            te = ev0.elapsed_time(ev) / 1e3
            for i, arrived in emitted:
                lags.append(te - arrived)
                if first[i] is None:
                    first[i] = te - start[i]
    lags = np.array(lags)
    return {"streams": len(streams), "steps": len(step_ms),
            "step_ms_p50": float(np.percentile(step_ms, 50)), "step_ms_p99": float(np.percentile(step_ms, 99)),
            "lag_s_p99": float(np.percentile(lags, 99)), "lag_s_max": float(lags.max()),
            "first_audio_s_p50": float(np.median(first)), "keeps_real_time": bool(lags.max() < args.chunk)}


def run_mode(vf, mode, args, streams, block, counts, rt_counts):
    """(a), (b) and (c) in one mode: a host and a device pool, captured once in the warm-up (as is restore_stream's
    workspace), against N restore_stream generators."""
    pool = vf.stream_pool(args.chunk, args.ctx, max_windows=args.max_windows, mode=mode)
    print(f"mode {mode}: pool window {pool.window_len} samples, buckets {pool.buckets}", flush=True)
    warm(pool)
    dpool = vf.stream_pool(args.chunk, args.ctx, max_windows=args.max_windows, mode=mode)
    warm(dpool, device=True)
    list(vf.restore_stream(blocks_of(streams[0][:3 * SR], block), args.chunk, args.ctx, mode=mode))

    table_a, host, dev_share = [], None, None
    for n in counts:
        steps, dsteps = [], []
        last = n == max(counts)
        replays, dreplays = (time_replays(pool), time_replays(dpool)) if last else ([], [])
        pool_out, pool_s = run_pool(pool, streams[:n], block, timed_steps=steps)
        dev_out, dev_s = run_pool(dpool, streams[:n], block, timed_steps=dsteps, device=True)
        torch.cuda.synchronize()
        rr_out, rr_s = run_round_robin(vf, streams[:n], block, args, mode)
        same = all(a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
                   for a, b in zip(pool_out, rr_out))
        assert same, f"N = {n}: the pool's output differs from restore_stream's"
        dev_same = all(a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
                       for a, b in zip(dev_out, pool_out))
        assert dev_same, f"N = {n}: the device pool's output differs from the host pool's"
        audio_s = sum(len(y) for y in pool_out) / SR
        row = {"mode": mode, "streams": n, "audio_s": audio_s, "pool_audio_s_per_s": audio_s / pool_s,
               "device_pool_audio_s_per_s": audio_s / dev_s, "round_robin_audio_s_per_s": audio_s / rr_s,
               "pool_s": pool_s, "device_pool_s": dev_s, "round_robin_s": rr_s, "steps": len(steps),
               "bit_identical": same and dev_same}
        table_a.append(row)
        print(json.dumps(row), flush=True)
        if last:                                    # (c) at the largest N
            # the replays inside the steps, timed by events around each: their lengths are the steps' own (a replay
            # repeated afterwards, replay_ms, reads the last step's lengths, and ragged rows cost what they hold)
            replay_s = sum(a.elapsed_time(b) for a, b in replays) / 1e3
            step_s = sum(t for _, t in steps)
            host = {"streams": n, "steps": len(steps), "step_s": step_s, "replay_s": replay_s,
                    "host_share": 1.0 - replay_s / step_s,
                    "replay_ms_per_bucket_repeated": {B: replay_ms(pool, B) for B in sorted({b for b, _ in steps})}}
            print(json.dumps(host), flush=True)
            replay_s = sum(a.elapsed_time(b) for a, b in dreplays) / 1e3
            step_s = sum(a.elapsed_time(b) for _, a, b in dsteps) / 1e3
            dev_share = {"streams": n, "steps": len(dsteps), "device_step_s": step_s, "replay_s": replay_s,
                         "outside_replay_share": 1.0 - replay_s / step_s, "wall_s": dev_s,
                         "outside_replay_share_of_wall": 1.0 - replay_s / dev_s}
            print(json.dumps({"device_pool": dev_share}), flush=True)

    table_b = {}
    for kind, p in (("host", pool), ("device", dpool)):
        rng = np.random.default_rng(args.seed + 1)
        table_b[kind] = []
        for n in rt_counts:
            row = run_real_time(p, streams[:n], block, args, rng, device=kind == "device")
            table_b[kind].append(row)
            print(json.dumps({"mode": mode, "pool": kind, **row}), flush=True)
        assert p.graph_count == len(p.buckets)      # nothing was captured after the warm-up
    largest = {kind: max([r["streams"] for r in rows if r["keeps_real_time"]], default=0)
               for kind, rows in table_b.items()}
    return {"throughput": table_a, "real_time": table_b, "largest_real_time_streams": largest, "host_share": host,
            "device_pool_share": dev_share}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,8,32,64,128")
    ap.add_argument("--rt-streams", default="8,32,64,128,192,256")
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--block-seconds", type=float, default=0.1)
    ap.add_argument("--chunk", type=float, default=1.0)
    ap.add_argument("--ctx", type=float, default=0.5)
    ap.add_argument("--max-windows", type=int, default=None)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--mode", default="0", help="comma-separated modes from 0, 1, 2, run one after the other")
    args = ap.parse_args()
    modes = [int(v) for v in args.mode.split(",") if v]
    if not modes or any(m not in (0, 1, 2) for m in modes):
        ap.error(f"--mode takes modes from 0, 1, 2; got {args.mode!r}")
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine

    info = gpu_info()
    print("gpu:", info, flush=True)
    eng = Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1), precision=args.precision)
    vf = VoiceFixer.from_engine(eng)
    block = int(round(args.block_seconds * SR))
    counts = [int(v) for v in args.streams.split(",") if v]
    rt_counts = [int(v) for v in args.rt_streams.split(",") if v]
    streams = utterances(max(counts + rt_counts), args.seconds, args.seed)

    results = {m: run_mode(vf, m, args, streams, block, counts, rt_counts) for m in modes}
    print(json.dumps({"gpu": info, "precision": args.precision, "seconds": args.seconds, "block_s": args.block_seconds,
                      "chunk_s": args.chunk, "ctx_s": args.ctx, "modes": results}))


if __name__ == "__main__":
    main()
