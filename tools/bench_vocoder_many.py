"""The stand-alone vocoder on many items: ragged batches against one call per item, synthetic weights.

  (a) 64 seeded mels with lengths uniform in 1 .. 10 s: one Vocoder.forward_many(list) call against Vocoder.forward once
      per mel.  The outputs must be bit-identical.
  (b) 16 seeded recordings of 5 .. 120 s: one Vocoder.oracle_many(list) call (front end and generator on the device, ragged
      batches) against the per-item path of Vocoder.oracle: oracle_conditions on the host, then Engine.vocoder_cond.  The
      outputs must agree within the precision's tolerance (the two front ends round differently).
  (c) the front end alone for (b)'s recordings: oracle_conditions on the host, one recording after another, against one
      vfx_oracle_cond call on the device-resident batch (Engine.oracle(..., return_cond=True)); also the largest
      difference between the two.

Each is timed with the host clock around calls that end in a device synchronise, after one untimed warm-up pass; the
best of --reps passes is reported.  The card's name, power limit and maximum SM clock are printed with the numbers, as
one JSON line.  Usage:
  python tools/bench_vocoder_many.py [--reps 3] [--precision tf32] [--seed 0]"""
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
# waveform agreement of oracle_many with the host-front-end path: the two front ends differ by ~1e-6 in the normalised
# conditions, which the operand rounding of the 16-bit / tf32 modes can amplify up to the modes' own parity bounds
TOL = {"fp32": 1e-5, "tf32": 2e-3, "fp16": 2e-3, "bf16": 3e-2}


def rel_rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(np.mean((a - b) ** 2)) / (np.sqrt(np.mean(b ** 2)) + 1e-30))


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import Vocoder, oracle_conditions
    from voicefixer_b200.engine import Engine
    from voicefixer_b200.weights import pack_vocoder

    eng = Engine(packed=pack_vocoder(synthetic.make_vocoder_state(1), args.precision), precision=args.precision)
    voc = Vocoder(44100, _engine=eng)
    rng = np.random.default_rng(args.seed)
    line = {"gpu": gpu_info(), "precision": args.precision}

    # (a) mels of 1 .. 10 s
    frames = 1 + rng.integers(SR, 10 * SR + 1, size=64) // 441
    mels = [torch.from_numpy(np.exp(rng.normal(-3.0, 2.0, size=(1, 1, int(T), 128))).astype(np.float32)) for T in frames]
    audio_a = float(sum((T + T % 2 + 4) * 441 for T in frames)) / SR
    many, t_many = timed(lambda: voc.forward_many(mels, cuda=True), args.reps)
    loop, t_loop = timed(lambda: [voc.forward(m, cuda=True) for m in mels], args.reps)
    identical = all(torch.equal(x, y) for x, y in zip(many, loop))
    line["a_forward"] = {"items": len(mels), "audio_s": round(audio_a, 1), "many_s": round(t_many, 4),
                         "per_item_s": round(t_loop, 4), "many_audio_s_per_s": round(audio_a / t_many, 1),
                         "per_item_audio_s_per_s": round(audio_a / t_loop, 1), "speedup": round(t_loop / t_many, 2),
                         "bit_identical": identical}
    del many, loop

    # (b) recordings of 5 .. 120 s through the whole oracle
    lens = rng.integers(5 * SR, 120 * SR + 1, size=16)
    wavs = []
    for n in lens:
        t = np.arange(int(n)) / SR
        f0 = rng.uniform(90, 250)
        x = sum(np.sin(2 * np.pi * f0 * k * t + rng.uniform(0, 6.28)) / k for k in range(1, 8))
        wavs.append((0.3 * x * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + 0.02 * rng.standard_normal(int(n)))
                    .astype(np.float32))
    audio_b = float(lens.sum()) / SR

    def per_item():
        return [eng.vocoder_cond(torch.from_numpy(oracle_conditions(w))).cpu().numpy() for w in wavs]

    many, t_many = timed(lambda: voc.oracle_many(wavs), args.reps)
    loop, t_loop = timed(per_item, args.reps)
    worst = max(rel_rms(x, y) for x, y in zip(many, loop))
    line["b_oracle"] = {"items": len(wavs), "audio_s": round(audio_b, 1), "many_s": round(t_many, 4),
                        "per_item_s": round(t_loop, 4), "many_audio_s_per_s": round(audio_b / t_many, 1),
                        "per_item_audio_s_per_s": round(audio_b / t_loop, 1), "speedup": round(t_loop / t_many, 2),
                        "max_rel_rms_vs_host_front_end": float(f"{worst:.3e}")}
    del many, loop

    # (c) the front end alone
    L_cap = int(lens.max())
    xb = torch.zeros(len(wavs), L_cap)
    for i, w in enumerate(wavs):
        xb[i, :w.shape[0]] = torch.from_numpy(w)
    xb = xb.to(f"cuda:{eng.device}")
    lb = torch.tensor([w.shape[0] for w in wavs], dtype=torch.int32).to(xb.device)
    host, t_host = timed(lambda: [oracle_conditions(w)[0] for w in wavs], args.reps)
    dev, t_dev = timed(lambda: eng.oracle(xb, lens=lb, return_cond=True), args.reps)
    dev = dev.cpu().numpy()
    fe_err = max(float(np.max(np.abs(dev[i, :h.shape[0]] - h))) for i, h in enumerate(host))
    line["c_front_end"] = {"host_s": round(t_host, 4), "device_s": round(t_dev, 5), "speedup": round(t_host / t_dev, 1),
                           "max_abs_diff": float(f"{fe_err:.3e}")}
    print(json.dumps(line))
    assert identical, "forward_many and forward differ"
    assert worst <= TOL[args.precision], f"oracle_many and the host-front-end path differ: rel-RMS {worst:.3e}"
    assert fe_err <= 1e-4, f"device front end differs from oracle_conditions by {fe_err:.3e}"


if __name__ == "__main__":
    main()
