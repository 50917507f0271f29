"""Recordings at other sample rates than 44.1 kHz: resampling on the device (restore_many(..., sample_rate=r)) against
resampling on the host first (wavio._resample, scipy's resample_poly, then restore_many), synthetic weights.

  (a) 48 seeded recordings of 2 .. 45 s generated at 16 kHz, and the same at 48 kHz: one restore_many call with
      sample_rate=r against the host resampler on every recording followed by restore_many.  The outputs must be equal.
  (b) the resampler alone on 10 minutes of audio at 16 and 48 kHz, as 30 s segments in one launch: device time of the
      vfx_resample call (CUDA events, staged input already on the device) against resample_poly on the host.

(a) is timed with the host clock around calls that end in a device synchronise, (b) with CUDA events; both after one
untimed warm-up, best of --reps.  The card's name, power limit and maximum SM clock are printed with the numbers, as one
JSON line.  Usage:
  python tools/bench_resample.py [--reps 3] [--precision tf32] [--seed 0]"""
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
SEG = 30 * SR


def timed(fn, reps):
    fn()                                                         # warm-up
    torch.cuda.synchronize()
    best, outs = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        outs = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return outs, best


def speech_like(rng, n, rate):
    t = np.arange(n) / rate
    f0 = rng.uniform(90, 250)
    x = sum(np.sin(2 * np.pi * f0 * k * t + rng.uniform(0, 6.28)) / k for k in range(1, 8))
    return (0.3 * x * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + 0.02 * rng.standard_normal(n)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from voicefixer_b200 import resample as rs
    from voicefixer_b200 import synthetic, wavio
    from voicefixer_b200.api import VoiceFixer, _stage
    from voicefixer_b200.engine import Engine

    eng = Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1), precision=args.precision)
    vf = VoiceFixer.from_engine(eng)
    dev = f"cuda:{eng.device}"
    line = {"gpu": gpu_info(), "precision": args.precision}
    equal = True

    # (a) 48 recordings of 2 .. 45 s per rate, through restore_many
    for rate in (16000, 48000):
        rng = np.random.default_rng(args.seed + rate)
        wavs = [speech_like(rng, int(rng.uniform(2, 45) * rate), rate) for _ in range(48)]
        audio = sum(w.shape[0] for w in wavs) / rate
        dev_out, t_dev = timed(lambda: vf.restore_many(wavs, sample_rate=rate), args.reps)
        host_out, t_host = timed(lambda: vf.restore_many([wavio._resample(w, rate, SR) for w in wavs]), args.reps)
        _, t_rs = timed(lambda: [wavio._resample(w, rate, SR) for w in wavs], args.reps)
        same = all(np.array_equal(a, b) for a, b in zip(dev_out, host_out))
        equal &= same
        line[f"a_restore_many_{rate // 1000}k"] = {
            "items": len(wavs), "audio_s": round(audio, 1), "device_resample_s": round(t_dev, 4),
            "host_resample_then_restore_s": round(t_host, 4), "host_resample_alone_s": round(t_rs, 4),
            "device_audio_s_per_s": round(audio / t_dev, 1), "host_audio_s_per_s": round(audio / t_host, 1),
            "speedup": round(t_host / t_dev, 3), "bit_identical": same}
        del dev_out, host_out

    # (b) the resampler alone: 10 minutes as 30 s segments in one launch
    for rate in (16000, 48000):
        x = speech_like(np.random.default_rng(args.seed + 7), 600 * rate, rate)
        ref, t_host = timed(lambda: wavio._resample(x, rate, SR), args.reps)
        n_out = rs.out_len(x.shape[0], rate)
        segs = [(0, a, min(a + SEG, n_out)) for a in range(0, n_out, SEG)]
        xs, table = _stage([x], [rate], segs, dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        best, y = None, None
        for k in range(args.reps + 1):
            e0.record()
            y, _ = eng.resample(xs, table, SEG)
            e1.record()
            torch.cuda.synchronize()
            if k:
                best = e0.elapsed_time(e1) / 1e3 if best is None else min(best, e0.elapsed_time(e1) / 1e3)
        y = y.cpu().numpy()
        same = all(np.array_equal(y[k, :b - a], ref[a:b]) for k, (_, a, b) in enumerate(segs))
        equal &= same
        line[f"b_resampler_{rate // 1000}k"] = {
            "audio_s": 600, "outputs": n_out, "device_s": round(best, 6), "host_scipy_s": round(t_host, 4),
            "speedup": round(t_host / best, 1), "device_outputs_per_s": float(f"{n_out / best:.3e}"),
            "bit_identical": same}
    print(json.dumps(line))
    assert equal, "the device resampler and the host resampler differ"


if __name__ == "__main__":
    main()
