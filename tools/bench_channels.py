"""Multichannel restores and the 16-bit packer, synthetic weights, mode 0, through VoiceFixer.restore_files (what the
command line's --batch runs), every file written under a temporary directory:

  keep:  bench_files' 24 x 2 .. 45 s 48 kHz stereo FLAC folder with channels="keep" against its mono mix, alternating;
  mono:  bench_files' three folders (short16k, cli10s, flac48k) restored to mono by this tree and, with --parent DIR (a
         built checkout of another commit), by that tree, each in its own process, the processes alternating
         (--rounds); the outputs of the two trees are compared byte for byte.  D2H bytes per wave are computed from the
         wave's output samples and the element the tree copies back (int16 where Engine.pack_pcm16 exists, float32
         before);
  pack:  Engine.pack_pcm16 on a table shaped like the keep folder's wave (24 stereo files), CUDA events around 20 calls
         after a warm-up, against its 6 bytes per sample (4 read, 2 written; the per-file maximum reads the 4 again).

Audio figures are audio-seconds per second of the folder, the best of --reps passes after one warm-up pass, with the
host clock around a call that returns once every output file is written.  The card's name, power limit and maximum SM
clock are read in the same run.  Prints one JSON line.  Usage:
  python tools/bench_channels.py [--parent DIR] [--rounds 2] [--reps 3] [--precision tf32] [--seed 0]"""
import argparse
import contextlib
import hashlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _vf(precision):
    from voicefixer_b200 import synthetic
    from voicefixer_b200.api import VoiceFixer
    from voicefixer_b200.engine import Engine
    return VoiceFixer.from_engine(Engine(synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1),
                                         precision=precision))


def _pass(vf, files, src, dst, channels, waves):
    """One restore_files pass over a folder: seconds, and the md5 of every output file."""
    import torch
    os.makedirs(dst, exist_ok=True)
    jobs = [(os.path.join(src, f[0]), os.path.join(dst, f[0]), 0) for f in files]
    kw = {"channels": channels} if channels != "mix" else {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        if kw:
            vf.restore_files([j[0] for j in jobs], [j[1] for j in jobs], mode=0, _on_wave=waves.append, **kw)
        else:
            vf.restore_files([j[0] for j in jobs], [j[1] for j in jobs], mode=0, _on_wave=waves.append)
    dt = time.perf_counter() - t0
    return dt, hashlib.md5(b"".join(open(j[1], "rb").read() for j in jobs)).hexdigest()


def _out_samples(files, src, channels):
    """Output samples of each file (44.1 kHz frames times the channels written)."""
    from voicefixer_b200 import resample, wavio
    n = []
    for f in files:
        x, sr = getattr(wavio, "load_native", wavio._read_pcm)(os.path.join(src, f[0]))   # a parent may lack it
        n.append(resample.out_len(x.shape[0], sr) * (x.shape[1] if channels == "keep" else 1))
    return n


def worker(args):
    """Runs in the tree under test (sys.path[0] = args.tree); prints one JSON line."""
    sys.path.insert(0, args.tree)
    import torch
    from voicefixer_b200 import engine as engine_mod
    from tools.bench_files import folders
    vf = _vf(args.precision)
    elem = 2 if hasattr(engine_mod.Engine, "pack_pcm16") else 4
    out = {"tree": args.tree, "d2h_bytes_per_sample": elem}
    all_files = folders(np.random.default_rng(args.seed))
    names = ["flac48k"] if args.job == "keep" else list(all_files)
    for name in names:
        files, src = all_files[name], os.path.join(args.data, name)
        audio_s = sum(n / sr for _, n, sr, _, _ in files)
        kinds = ["mix", "keep"] if args.job == "keep" else ["mix"]
        best, digest, waves = {}, {}, {}
        for rep in range(args.reps + 1):                        # pass 0 is the warm-up
            for ch in kinds:
                waves[ch] = []
                dt, digest[ch] = _pass(vf, files, src, os.path.join(args.out, f"{name}-{ch}"), ch, waves[ch])
                if rep:
                    best[ch] = min(best.get(ch, dt), dt)
                torch.cuda.empty_cache()
        for ch in kinds:
            n = _out_samples(files, src, ch)
            d2h = [elem * sum(n[i] for i in w) for w in waves[ch]]
            out[f"{name}-{ch}"] = {"files": len(files), "audio_s": round(audio_s, 1), "best_s": round(best[ch], 3),
                                   "audio_s_per_s": round(audio_s / best[ch], 1), "waves": len(waves[ch]),
                                   "d2h_MB_per_wave": [round(b / 1e6, 1) for b in d2h], "md5": digest[ch]}
    if args.job == "keep":
        out["pack"] = _bench_pack(vf, all_files["flac48k"])
    print(json.dumps(out))


def _bench_pack(vf, files):
    import torch
    eng = vf._engine
    dev = f"cuda:{eng.device}"
    rows = [[torch.rand(int(n * 44100 / sr), device=dev) * 2 - 1 for _ in range(ch)] for _, n, sr, ch, _ in files]
    samples = sum(r.numel() for f in rows for r in f)
    y, _ = eng.pack_pcm16(rows)
    for _ in range(3):
        eng.pack_pcm16(rows, y=y)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        eng.pack_pcm16(rows, y=y)
    b.record()
    b.synchronize()
    t = a.elapsed_time(b) / 20 / 1e3
    return {"files": len(rows), "samples": samples, "us_per_call": round(t * 1e6, 1),
            "GB_per_s_at_6_bytes_per_sample": round(6 * samples / t / 1e9, 1),
            "GB_per_s_at_10_bytes_per_sample": round(10 * samples / t / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="a built checkout of another commit to compare the mono folders with")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="tf32")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tree", help=argparse.SUPPRESS)
    ap.add_argument("--job", help=argparse.SUPPRESS)
    ap.add_argument("--data", help=argparse.SUPPRESS)
    ap.add_argument("--out", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from tools.bench_ragged import gpu_info
    from tools.bench_files import folders
    import audio_files
    line = {"gpu": gpu_info(), "precision": args.precision, "reps": args.reps}
    with tempfile.TemporaryDirectory() as tmp:
        for name, files in folders(np.random.default_rng(args.seed)).items():
            os.makedirs(os.path.join(tmp, "data", name))
            for k, (fname, n, sr, ch, fmt) in enumerate(files):
                audio_files.write(os.path.join(tmp, "data", name, fname), n, sr, ch, fmt, seed=1000 * len(files) + k)

        def run(tree, job, tag):
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--tree", os.path.abspath(tree), "--job", job,
                   "--data", os.path.join(tmp, "data"), "--out", os.path.join(tmp, tag), "--reps", str(args.reps),
                   "--precision", args.precision, "--seed", str(args.seed)]
            r = subprocess.run(cmd, stdout=subprocess.PIPE, text=True, check=True, cwd=tmp)
            res = json.loads(r.stdout.strip().splitlines()[-1])
            print(json.dumps({tag: res}), file=sys.stderr)
            return res

        line["keep"] = run(ROOT, "keep", "keep")
        trees = [("tree", ROOT)] + ([("parent", args.parent)] if args.parent else [])
        line["mono"] = {t: [] for t, _ in trees}
        for rnd in range(args.rounds):
            for t, path in (trees if rnd % 2 == 0 else trees[::-1]):
                line["mono"][t].append(run(path, "mono", f"{t}{rnd}"))
        if args.parent:
            line["mono_equal_bytes"] = all(a[k]["md5"] == b[k]["md5"] for a in line["mono"]["tree"]
                                           for b in line["mono"]["parent"] for k in a if isinstance(a[k], dict))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
