"""VoiceFixer.restore_many against a loop of restore_inmem over the same recordings, in modes 0, 1 and 2: audio-seconds
restored per second for a seeded set of recordings (uniform in 2 .. 45 s, so most are shorter than one 30 s segment and
some span two; a tail under 1 s is lengthened by 1 s, since mode 2 refuses segments of 64 frames or fewer), synthetic
weights.

  (a) one restore_many(list, mode) call: every segment of every recording in ragged batches ordered by length;
  (b) restore_inmem(recording, mode) once per recording: one launch sequence per distinct segment length, B = 1 for
      most recordings.

Each is timed with the host clock around calls that end in a device synchronise, after one untimed warm-up pass; the
best of --reps passes is reported.  Mode 2 runs with random dropout masks, as restore_inmem's default does.  The script
checks in the same run that (a) and (b) give equal outputs in modes 0 and 1 (and in mode 2 without dropout), and prints
the card's name, power limit and maximum SM clock with the numbers, as one JSON line.  Usage:
  python tools/bench_many.py [--items 48] [--reps 3] [--precision tf32] [--seed 0]"""
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
    audio_s = float(lens.sum()) / SR

    def timed(fn):
        fn()                                                     # warm-up
        torch.cuda.synchronize()
        best, outs = None, None
        for _ in range(args.reps):
            t0 = time.perf_counter()
            outs = fn()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        return outs, best

    line = {"gpu": gpu_info(), "precision": args.precision, "items": args.items, "audio_s": round(audio_s, 2),
            "segments": int(sum(-(-int(n) // (30 * SR)) for n in lens))}
    for mode in (0, 1, 2):
        many, t_many = timed(lambda: vf.restore_many(wavs, mode=mode))
        loop, t_loop = timed(lambda: [vf.restore_inmem(w, cuda=True, mode=mode) for w in wavs])
        if mode == 2:                                            # equality without dropout (the masks are random)
            many = vf.restore_many(wavs, mode=2, drop_masks_fn=False)
            loop = [vf.restore_inmem(w, cuda=True, mode=2, drop_masks_fn=False) for w in wavs]
        equal = all(np.array_equal(a, b) for a, b in zip(many, loop))
        line[f"mode{mode}"] = {"many_s": round(t_many, 4), "inmem_loop_s": round(t_loop, 4),
                               "many_audio_s_per_s": round(audio_s / t_many, 1),
                               "inmem_loop_audio_s_per_s": round(audio_s / t_loop, 1), "equal": equal}
    print(json.dumps(line))
    assert all(line[f"mode{m}"]["equal"] for m in (0, 1, 2)), "restore_many and restore_inmem differ"


if __name__ == "__main__":
    main()
