"""VoiceFixer.restore_files over several GPUs (gpus=N, one process per device) on tools/bench_files.py's three seeded
folders, each scaled up --scale times (every file repeated with a new seed; default 8) and run with waves of
--wave-seconds of audio (default 600 s) so that each device restores several waves:

  short16k:  64 x scale utterances of 1 .. 10 s at 16 kHz, mono 16-bit WAV;
  cli10s:    16 x scale recordings of 10 s at 44.1 kHz, mono 16-bit WAV;
  flac48k:   24 x scale recordings of 2 .. 45 s at 48 kHz, stereo FLAC (mono mix restored, the default).

Settings: gpus = 1, 2, 4, ... up to the devices present, and "gpu0x2": two processes on device 0 (restore_files'
_devices=[0, 0]), which shows what a second process's host capacity gives without a second GPU.  The settings
alternate within each repetition; each figure is audio-seconds per wall-second, mode 0, the best of --reps after one
warm-up pass, timed with the host clock around a call that returns once every output file is written and every worker
has exited (so start-up is inside it).  Start-up on its own: the wall time of restore_files on one 0.5 s file per
process, less that of gpus=1 on one such file.  Every output is compared byte for byte across the settings.  The
card's name, power limit and maximum SM clock are read in the same run.  Synthetic weights; everything is written under
a temporary directory.  Prints one JSON line.  Usage:
  python tools/bench_gpus.py [--reps 2] [--scale 8] [--wave-seconds 600] [--precision tf32] [--seed 0]"""
import argparse
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
from tools.bench_files import folders  # noqa: E402
import audio_files  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--scale", type=int, default=8)
    ap.add_argument("--wave-seconds", type=float, default=600.0)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine

    vf = VoiceFixer.from_engine(Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1),
                                       precision=args.precision))
    n_dev = torch.cuda.device_count()
    settings = {f"gpus{g}": {"gpus": g} for g in (1, 2, 4, 8, 16) if g <= n_dev}
    settings["gpu0x2"] = {"gpus": 2, "_devices": [0, 0]}
    budget = int(args.wave_seconds * 44100)
    rng = np.random.default_rng(args.seed)
    line = {"gpu": gpu_info(), "devices": n_dev, "precision": args.precision, "reps": args.reps, "scale": args.scale,
            "wave_seconds": args.wave_seconds}
    with tempfile.TemporaryDirectory() as tmp:
        def timed(srcs, dst, kw, **extra):
            os.makedirs(dst, exist_ok=True)
            outs = [os.path.join(dst, os.path.basename(s)) for s in srcs]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            vf.restore_files(srcs, outs, mode=0, **kw, **extra)
            return time.perf_counter() - t0, outs

        tiny = [audio_files.write(os.path.join(tmp, f"tiny{k}.wav"), 22050, 44100, 1, "s16", seed=k) for k in range(8)]
        timed(tiny[:1], os.path.join(tmp, "tiny-warm"), {})
        base = min(timed(tiny[:1], os.path.join(tmp, "tiny1"), {})[0] for _ in range(3))
        line["startup_s"] = {}
        for name, kw in settings.items():
            if kw["gpus"] > 1:
                procs = len(kw.get("_devices", range(kw["gpus"])))
                t = min(timed(tiny[:procs], os.path.join(tmp, f"tiny-{name}"), kw)[0] for _ in range(2))
                line["startup_s"][name] = round(t - base, 2)
        print(json.dumps({"startup_s": line["startup_s"]}), file=sys.stderr)

        for name, files in folders(rng).items():
            src = os.path.join(tmp, name)
            os.makedirs(src)
            srcs = []
            for r in range(args.scale):
                for k, (fname, n, sr, ch, fmt) in enumerate(files):
                    stem, ext = os.path.splitext(fname)
                    srcs.append(audio_files.write(os.path.join(src, f"{stem}-{r}{ext}"), n, sr, ch, fmt,
                                                  seed=1000 * len(files) * (r + 1) + k))
            audio_s = args.scale * sum(n / sr for _, n, sr, _, _ in files)
            best, outs = {}, {}
            for rep in range(args.reps + 1):                              # pass 0 is the warm-up
                for s, kw in settings.items():
                    dt, outs[s] = timed(srcs, os.path.join(tmp, f"{name}-{s}"), kw, _budget=budget)
                    if rep:
                        best[s] = min(best.get(s, dt), dt)
            ref = [open(o, "rb").read() for o in outs["gpus1"]]
            equal = all([open(o, "rb").read() for o in outs[s]] == ref for s in settings)
            line[name] = {"files": len(srcs), "audio_s": round(audio_s, 1), "equal_bytes": equal,
                          "wall_s": {s: round(best[s], 3) for s in settings},
                          "audio_s_per_s": {s: round(audio_s / best[s], 1) for s in settings}}
            print(json.dumps({name: line[name]}), file=sys.stderr)
    print(json.dumps(line))
    assert all(line[n]["equal_bytes"] for n in ("short16k", "cli10s", "flac48k")), "the settings' outputs differ"


if __name__ == "__main__":
    main()
