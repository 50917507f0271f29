"""The command line's two ways through a folder of files, on three seeded folders: one file at a time (`run_waves` with
a budget of 0, what `python -m voicefixer_b200 --infolder ...` runs) against many files per batch
(`VoiceFixer.restore_files`, what it runs with `--batch`), both through `__main__.execute`, in one process, alternating,
synthetic weights:

  short16k:  64 utterances of 1 .. 10 s at 16 kHz, mono 16-bit WAV;
  cli10s:    16 recordings of 10 s at 44.1 kHz, mono 16-bit WAV (bench.py's cli_folder shape);
  flac48k:   24 recordings of 2 .. 45 s at 48 kHz, stereo FLAC (the command line's folder mode reads .wav only, so
             this folder's jobs are listed here as it would list them).

Each figure is audio-seconds per second of the folder, mode 0, the best of --reps passes after one warm-up pass, timed
with the host clock around a call that returns once every output file is written.  In the same run the outputs of the
two paths are compared byte for byte in modes 0 and 1, and the card's name, power limit and maximum SM clock are read.
Everything is written under a temporary directory.  Prints one JSON line.  Usage:
  python tools/bench_files.py [--reps 3] [--precision tf32] [--seed 0]"""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.bench_ragged import gpu_info  # noqa: E402
import audio_files  # noqa: E402


def folders(rng):
    """name -> [(file name, frames, rate, channels, format)]."""
    return {
        "short16k": [(f"u{k:03d}.wav", int(rng.uniform(1, 10) * 16000), 16000, 1, "s16") for k in range(64)],
        "cli10s": [(f"r{k:03d}.wav", 10 * 44100, 44100, 1, "s16") for k in range(16)],
        "flac48k": [(f"s{k:03d}.flac", int(rng.uniform(2, 45) * 48000), 48000, 2, "flac") for k in range(24)],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from voicefixer_b200 import synthetic, __main__ as cli
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine

    vf = VoiceFixer.from_engine(Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1),
                                       precision=args.precision))
    rng = np.random.default_rng(args.seed)
    line = {"gpu": gpu_info(), "precision": args.precision, "reps": args.reps}
    with tempfile.TemporaryDirectory() as tmp:
        for name, files in folders(rng).items():
            src = os.path.join(tmp, name)
            os.makedirs(src)
            for k, (fname, n, sr, ch, fmt) in enumerate(files):
                audio_files.write(os.path.join(src, fname), n, sr, ch, fmt, seed=1000 * len(files) + k)
            audio_s = sum(n / sr for _, n, sr, _, _ in files)

            def run(batch, mode):
                dst = os.path.join(tmp, f"{name}-{'batch' if batch else 'per_file'}-{mode}")
                os.makedirs(dst, exist_ok=True)
                jobs = [(os.path.join(src, f[0]), os.path.join(dst, f[0]), mode) for f in files]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with contextlib.redirect_stdout(io.StringIO()):         # the per-wave / per-job messages
                    cli.execute(vf, jobs, batch=batch, say=lambda *a: None)
                dt = time.perf_counter() - t0
                return dt, [open(j[1], "rb").read() for j in jobs]

            best = {False: None, True: None}
            for rep in range(args.reps + 1):                           # pass 0 is the warm-up
                for batch in (False, True):
                    dt, _ = run(batch, 0)
                    if rep:
                        best[batch] = dt if best[batch] is None else min(best[batch], dt)
            equal = {f"mode{m}": run(False, m)[1] == run(True, m)[1] for m in (0, 1)}
            line[name] = {"files": len(files), "audio_s": round(audio_s, 1),
                          "per_file_s": round(best[False], 3), "batch_s": round(best[True], 3),
                          "per_file_audio_s_per_s": round(audio_s / best[False], 1),
                          "batch_audio_s_per_s": round(audio_s / best[True], 1), "equal_bytes": equal}
            print(json.dumps({name: line[name]}), file=sys.stderr)
    print(json.dumps(line))
    assert all(all(line[n]["equal_bytes"].values()) for n in ("short16k", "cli10s", "flac48k")), "the two paths differ"


if __name__ == "__main__":
    main()
