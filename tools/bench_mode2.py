"""Mode 2's dropout masks: host-drawn against seeded, on VoiceFixer.restore_many over bench_many's workload (seeded
recordings uniform in 2 .. 45 s, a tail under 1 s lengthened by 1 s, synthetic weights), with host (numpy) and CUDA
inputs.  Three variants:

  host   : drop_masks_fn=None, the default: Bernoulli(0.5) masks drawn on torch's CPU generator and uploaded per batch;
  seeded : dropout_seed (one seed per recording): the masks are computed in the dropout kernel, only 16 bytes of key
           per segment are uploaded;
  none   : drop_masks_fn=False, no dropout at all: the floor both others stand on.

Each is timed with the host clock around calls that end in a device synchronise, after one untimed warm-up call; the
best of --reps calls is reported as audio-seconds per wall-second, with the host CPU seconds (process time, all
threads) per call averaged over the same calls.  `equal` checks in the same run that every recording's seeded output is
bit-identical to restore_inmem on that recording alone given the host restatement's masks (voicefixer_b200.philox) as
explicit masks.  The card's name, power limit and maximum SM clock are printed with the numbers, as one JSON line.
Usage:
  python tools/bench_mode2.py [--items 48] [--reps 3] [--precision tf32] [--seed 0]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_ragged import gpu_info  # noqa: E402

SR = 44100


def restated_masks_fn(n, seed):
    """drop_masks_fn for restore_inmem on one recording of n samples: the seeded masks of its segments, in the order
    restore_inmem asks for them (its groups of equal segment length in order of first appearance, each group's
    segments in order, in chunks of any size)."""
    from voicefixer_b200.api import segment_bounds
    from voicefixer_b200.philox import seeded_masks
    groups = {}
    for k, (a, b) in enumerate(segment_bounds(n)):
        groups.setdefault(b - a, []).append(k)
    order = [k for ks in groups.values() for k in ks]

    def fn(B, T):
        ks = [order.pop(0) for _ in range(B)]
        return torch.from_numpy(np.stack([seeded_masks(seed, k, T) for k in ks], 1))
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=48)
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
    lens = rng.integers(2 * SR, 45 * SR + 1, size=args.items)
    lens = np.where((lens > 30 * SR) & (lens <= 31 * SR), lens + SR, lens)    # tails under 1 s: mode 2 refuses <= 64 frames
    wavs = [(0.3 * rng.standard_normal(int(n))).astype(np.float32) for n in lens]
    dwavs = [torch.from_numpy(w).to(f"cuda:{eng.device}") for w in wavs]
    seeds = [2 * int(s) + 1 for s in rng.integers(0, 2 ** 63, size=args.items, dtype=np.int64)]   # odd, in [0, 2^64)
    audio_s = float(lens.sum()) / SR

    def timed(fn):
        fn()                                                     # warm-up
        torch.cuda.synchronize()
        best, cpu = None, 0.0
        for _ in range(args.reps):
            t0, c0 = time.perf_counter(), time.process_time()
            fn()
            torch.cuda.synchronize()
            dt, dc = time.perf_counter() - t0, time.process_time() - c0
            best = dt if best is None else min(best, dt)
            cpu += dc
        return {"wall_s": round(best, 4), "audio_s_per_s": round(audio_s / best, 1),
                "host_cpu_s_per_call": round(cpu / args.reps, 4)}

    variants = {"host": {}, "seeded": {"dropout_seed": seeds}, "none": {"drop_masks_fn": False}}
    line = {"gpu": gpu_info(), "precision": args.precision, "items": args.items, "audio_s": round(audio_s, 2),
            "segments": int(sum(-(-int(n) // (30 * SR)) for n in lens)), "torch_threads": torch.get_num_threads()}
    for inp, xs in (("host_input", wavs), ("cuda_input", dwavs)):
        line[inp] = {name: timed(lambda: vf.restore_many(xs, mode=2, **kw)) for name, kw in variants.items()}
    seeded = vf.restore_many(wavs, mode=2, dropout_seed=seeds)
    seeded_dev = vf.restore_many(dwavs, mode=2, dropout_seed=seeds)
    explicit = [vf.restore_inmem(w, cuda=True, mode=2, drop_masks_fn=restated_masks_fn(w.shape[0], s))
                for w, s in zip(wavs, seeds)]
    line["equal"] = all(np.array_equal(a.view(np.int32), b.view(np.int32)) for a, b in zip(seeded, explicit)) and all(
        np.array_equal(d.cpu().numpy().view(np.int32), b.view(np.int32)) for d, b in zip(seeded_dev, explicit))
    print(json.dumps(line))
    assert line["equal"], "seeded dropout differs from the explicit restated masks"


if __name__ == "__main__":
    main()
