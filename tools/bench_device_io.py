"""VoiceFixer.restore_many on recordings that are already CUDA tensors, against what a caller of the host-only API has
to do with them: audio-seconds restored per second for a seeded set of recordings (uniform in 2 .. 45 s, generated on
the device), at 44.1 kHz and at 16 kHz, synthetic weights.

  (a) device: restore_many(cuda_tensors, sample_rate=r): read in place, results as new CUDA tensors;
  (b) round trip: [t.cpu().numpy() for t in cuda_tensors], restore_many on the arrays, then torch.from_numpy(o).to(dev)
      for every result.

Each is timed with the host clock around calls that end in a device synchronise, after one untimed warm-up pass; the
best of --reps passes is reported.  The script checks in the same run that (a) and (b) give bit-identical outputs and
prints the card's name, power limit and maximum SM clock with the numbers, as one JSON line.  Usage:
  python tools/bench_device_io.py [--items 48] [--reps 3] [--precision tf32] [--mode 0] [--seed 0]"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_ragged import gpu_info  # noqa: E402

SR = 44100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--mode", type=int, default=0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine

    dev = "cuda:0"
    eng = Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1), precision=args.precision)
    vf = VoiceFixer.from_engine(eng)
    gen = torch.Generator(device=dev).manual_seed(args.seed)
    seconds = torch.empty(args.items).uniform_(2.0, 45.0, generator=torch.Generator().manual_seed(args.seed)).tolist()
    # a tail under 1 s is lengthened by 1 s: mode 2 refuses segments of 64 frames or fewer
    seconds = [s + 1.0 if 30.0 < s <= 31.0 else s for s in seconds]

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

    line = {"gpu": gpu_info(), "precision": args.precision, "mode": args.mode, "items": args.items,
            "audio_s": round(sum(seconds), 2)}
    kw = dict(mode=args.mode, drop_masks_fn=False if args.mode == 2 else None)
    for rate in (SR, 16000):
        wavs = [0.3 * torch.randn(int(s * rate), device=dev, generator=gen) for s in seconds]
        mb = sum(4 * w.numel() for w in wavs) / 1e6
        dev_out, t_dev = timed(lambda: vf.restore_many(wavs, sample_rate=rate, **kw))
        rt_out, t_rt = timed(lambda: [torch.from_numpy(o).to(dev) for o in
                                      vf.restore_many([w.cpu().numpy() for w in wavs], sample_rate=rate, **kw)])
        equal = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(dev_out, rt_out))
        line[f"{rate}Hz"] = {"input_MB": round(mb, 1), "output_MB": round(sum(4 * o.numel() for o in dev_out) / 1e6, 1),
                             "device_s": round(t_dev, 4), "round_trip_s": round(t_rt, 4),
                             "device_audio_s_per_s": round(sum(seconds) / t_dev, 1),
                             "round_trip_audio_s_per_s": round(sum(seconds) / t_rt, 1),
                             "speedup": round(t_rt / t_dev, 3), "equal": equal}
    print(json.dumps(line))
    assert all(line[f"{r}Hz"]["equal"] for r in (SR, 16000)), "device-resident and round-trip outputs differ"


if __name__ == "__main__":
    main()
