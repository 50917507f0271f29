#!/usr/bin/env python
"""CPU simulation of reduced-precision convolution operands on the oracle (test tooling; imports oracle/).

Rounds the activation and weight operands of every conv / conv_transpose / linear of the oracle's restore path to
a tensor-core input format (fp32 accumulate stays) and reports the waveform error against the fp32 oracle.  This is how
the stated tolerances of the tf32 / bf16 engine modes were derived before the kernels were measured on the GPU:

  tf32-rn    cvt.rna.tf32.f32 on both operands (what the engine's tf32 mode does when it writes operands)
  tf32-trunc hardware truncation of raw fp32 operands (what the tf32 tensor core does to un-rounded inputs)
  bf16       round-to-nearest bf16 operands (the engine's bf16 mode)
  fp16       round-to-nearest fp16 operands: the same 10-bit mantissa as tf32 in 2 bytes (5-bit exponent)

The reference's own CUDA path runs its convolutions in TF32 (torch.backends.cudnn.allow_tf32 defaults to True,
SURVEY D10), so the tf32 rows are also the reference GPU path's own deviation from its CPU path.
"""
import argparse
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def round_tf32_rn(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def trunc_tf32(x):
    i = x.contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32)


def round_bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


def round_fp16(x):
    return x.to(torch.float16).to(torch.float32)


MODES = {"tf32-rn": round_tf32_rn, "fp16": round_fp16, "tf32-trunc": trunc_tf32, "bf16": round_bf16}


class patched:
    """Routes the operands of the dense contractions through `rnd` (convs only, or convs + linears)."""

    def __init__(self, rnd, linears):
        self.rnd, self.linears = rnd, linears
        self.names = ["conv1d", "conv2d", "conv_transpose1d", "conv_transpose2d"] + (["linear"] if linears else [])

    def __enter__(self):
        self.saved = {n: getattr(F, n) for n in self.names}
        for n in self.names:
            f = self.saved[n]
            setattr(F, n, (lambda f: lambda x, w, *a, **k: f(self.rnd(x), self.rnd(w), *a, **k))(f))

    def __exit__(self, *a):
        for n, f in self.saved.items():
            setattr(F, n, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--threads", type=int, default=8)
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    from voicefixer_b200 import synthetic
    from oracle import vf_oracle as O
    ana, voc = synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1)
    wav = synthetic.make_utterances(1, seconds=args.seconds, seed=1234)[0]
    ref = np.asarray(O.restore_inmem(wav, ana, voc, mode=0), np.float64)
    rms = float(np.sqrt(np.mean(ref ** 2)))
    print(f"fp32 oracle: {args.seconds:g} s, wav rms {rms:.4f}")
    # the front-end DFT conv is an FFT in the engine (fp32): restore the un-rounded STFT while patched
    stft = O.stft_mag
    for name, rnd in MODES.items():
        for linears in (False, True):
            saved = {n: getattr(F, n) for n in ("conv1d",)}
            def stft_fp32(w, a, _saved=saved):
                cur = F.conv1d
                F.conv1d = _saved["conv1d"]
                try:
                    return stft(w, a)
                finally:
                    F.conv1d = cur
            O.stft_mag = stft_fp32
            with patched(rnd, linears):
                y = np.asarray(O.restore_inmem(wav, ana, voc, mode=0), np.float64)
            O.stft_mag = stft
            err = y - ref
            print(f"{name:11s} linears={'y' if linears else 'n'}: rel-rms {np.sqrt(np.mean(err ** 2)) / rms:.3e}  "
                  f"mean-abs {np.mean(np.abs(err)):.3e}  max-abs {np.max(np.abs(err)):.3e}")


if __name__ == "__main__":
    main()
