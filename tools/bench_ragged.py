"""Ragged batch vs. grouping by length: audio-seconds restored per second for a seeded set of utterances of different
lengths (uniform in 1 .. 10 s), mode 0, synthetic weights.

  (a) one ragged VoiceFixer.restore_batch(list) call: one CUDA-graph replay of shape (B, L_cap);
  (b) the same items grouped by exact length, one restore_batch((n, L)) call per group -- what the array form allows.
      Lengths drawn at random are almost all distinct, and restore_batch keeps the graphs of only a few shapes, so (b)
      captures a graph per group on every pass, as a caller of the array form would.

Both are timed after one untimed pass (graph capture).  The script asserts that (a) and (b) give bit-identical
results, and prints the card's name, power limit and maximum SM clock with the numbers.  Usage:
  python tools/bench_ragged.py [--items 64] [--reps 3] [--precision tf32] [--seed 0]"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine

    eng = Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1), precision=args.precision)
    vf = VoiceFixer.from_engine(eng)
    rng = np.random.default_rng(args.seed)
    lens = rng.integers(SR, 10 * SR + 1, size=args.items)
    items = [(0.3 * rng.standard_normal(int(n))).astype(np.float32) for n in lens]
    audio_s = float(lens.sum()) / SR

    def ragged():
        return vf.restore_batch(items)

    def grouped():
        groups = {}
        for i, a in enumerate(items):
            groups.setdefault(a.shape[0], []).append(i)
        out = [None] * len(items)
        for idx in groups.values():
            y = vf.restore_batch(np.stack([items[i] for i in idx]))
            for k, i in enumerate(idx):
                out[i] = y[k].copy()
        return out

    vf._batch_plans = {}
    res = {}
    for name, fn in (("ragged", ragged), ("grouped", grouped)):
        vf._batch_plans = {}                                     # release the other form's graphs and workspaces
        torch.cuda.empty_cache()
        outs = fn()                                              # capture
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            outs = fn()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        res[name] = (outs, min(times))
    a, b = res["ragged"][0], res["grouped"][0]
    identical = all(np.array_equal(x, y) for x, y in zip(a, b))
    line = {"gpu": gpu_info(), "precision": args.precision, "items": args.items, "audio_s": round(audio_s, 2),
            "L_cap_s": int(-(-int(lens.max()) // SR)), "distinct_lengths": int(len(set(lens.tolist()))),
            "ragged_s": round(res["ragged"][1], 4), "grouped_s": round(res["grouped"][1], 4),
            "ragged_audio_s_per_s": round(audio_s / res["ragged"][1], 1),
            "grouped_audio_s_per_s": round(audio_s / res["grouped"][1], 1), "bit_identical": identical}
    print(json.dumps(line))
    assert identical, "ragged and grouped results differ"


if __name__ == "__main__":
    main()
