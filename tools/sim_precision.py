#!/usr/bin/env python
"""CPU simulation of reduced-precision convolution operands on the oracle (test tooling; imports oracle/).

Runs the oracle's restore path under its operand-rounding model (oracle.vf_oracle.operand_rounding: every operand the
engine feeds a tensor core, rounded where the engine rounds it; accumulation in the state dicts' dtype) and reports
the waveform error against the plain oracle.  This is how the stated tolerances of the tf32 / fp16 / bf16 engine
modes were derived before the kernels were measured on the GPU:

  tf32       cvt.rna.tf32.f32 on both operands (what the engine's tf32 mode does when it writes operands)
  tf32-trunc hardware truncation of raw fp32 operands (what the tf32 tensor core does to un-rounded inputs)
  fp16       round-to-nearest fp16 operands: the same 10-bit mantissa as tf32 in 2 bytes (5-bit exponent)
  bf16       round-to-nearest bf16 operands (the engine's bf16 mode)

By default both the model and the reference compute in float64 (--sums fp64); --sums fp32 runs the model with fp32
sums against the fp32 oracle, as the engine accumulates.  The reference's own CUDA path runs its convolutions in TF32
(torch.backends.cudnn.allow_tf32 defaults to True, SURVEY D10), so the tf32 rows are also the reference GPU path's own
deviation from its CPU path.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def to_dtype(sd, dtype):
    return {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--sums", choices=("fp32", "fp64"), default="fp64")
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    dtype = torch.float64 if args.sums == "fp64" else torch.float32
    ana = to_dtype(synthetic.make_analysis_state(0), dtype)
    voc = to_dtype(synthetic.make_vocoder_state(1), dtype)
    wav = synthetic.make_utterances(1, seconds=args.seconds, seed=1234)[0]
    ref = np.asarray(O.restore_inmem(wav, ana, voc, mode=0), np.float64)
    rms = float(np.sqrt(np.mean(ref ** 2)))
    print(f"{args.sums} oracle: {args.seconds:g} s, wav rms {rms:.4f}")
    for name in ("tf32", "fp16", "tf32-trunc", "bf16"):
        with O.operand_rounding(name):
            y = np.asarray(O.restore_inmem(wav, ana, voc, mode=0), np.float64)
        err = y - ref
        print(f"{name:11s}: rel-rms {np.sqrt(np.mean(err ** 2)) / rms:.3e}  "
              f"mean-abs {np.mean(np.abs(err)):.3e}  max-abs {np.max(np.abs(err)):.3e}", flush=True)


if __name__ == "__main__":
    main()
