"""Command line mirror of the reference's `voicefixer` entry point (voicefixer/__main__.py:13-219):

    python -m voicefixer_b200 --infile in.wav --outfile out.wav [--mode 0|1|2|all]
    python -m voicefixer_b200 --infolder wavs/ --outfolder restored/ [--mode ...] [--batch] [--keep-channels] [--gpus N]

Same flags, same output naming (`--mode all` writes `<name>-mode<k><ext>` for k = 0,1,2), same
`.wav`-only input rule, same messages.  The work is planned first (`plan_jobs`, a pure function) and
then executed with one VoiceFixer instance (`execute`), one file at a time through the reader -> GPU ->
writer pipeline of `VoiceFixer.restore_files` (`api.run_waves`); with `--batch` the same jobs run
through `VoiceFixer.restore_files` itself, many files per batch.  With `--keep-channels` every channel
of a file is restored and written (restore(..., channels="keep")), on either path, with the same bytes.
With `--gpus N` (N > 1) the jobs run as with `--batch`, spread over N GPUs by
`VoiceFixer.restore_files(..., gpus=N)`, again with the same bytes."""
import argparse
import os
import re
import sys
import time

OUTPUT_FORMATS = {"WAV", "FLAC"}               # stdlib `wave` + in-tree FLAC codec (soundfile is not in this image)


def build_parser():
    p = argparse.ArgumentParser(prog="voicefixer_b200", description="VoiceFixer - restores degraded speech")
    p.add_argument("-i", "--infile", type=str, default="", help="An input file to be processed by VoiceFixer.")
    p.add_argument("-o", "--outfile", type=str, default="outfile.wav", help="An output file to store the result.")
    p.add_argument("-ifdr", "--infolder", type=str, default="",
                   help="Input folder. Place all your wav file that need process in this folder.")
    p.add_argument("-ofdr", "--outfolder", type=str, default="outfolder",
                   help="Output folder. The processed files will be stored in this folder.")
    p.add_argument("--mode", choices=["0", "1", "2", "all"], default="0",
                   help="0: Original Model (default), 1: Add preprocessing module (remove higher frequencies), "
                        "2: Train mode (might work sometimes on seriously degraded real speech), "
                        "all: Run all modes - will output one wav file for each supported mode.")
    p.add_argument("--disable-cuda", default=False, action="store_true",
                   help="Accepted for compatibility; this build has no CPU path and always runs on the GPU.")
    p.add_argument("--silent", default=False, action="store_true", help="Set this flag if you do not want to see any message.")
    p.add_argument("--weight_prepare", default=False, action="store_true",
                   help="Only check that the checkpoints are present (the reference uses it to trigger the download).")
    p.add_argument("--batch", default=False, action="store_true",
                   help="Restore many files at once (VoiceFixer.restore_files): the same outputs, batched across files.")
    p.add_argument("--keep-channels", default=False, action="store_true",
                   help="Restore every channel of a multichannel file and write them all, instead of its mono mix.")
    p.add_argument("--gpus", type=int, default=1,
                   help="Spread the files over this many GPUs, one process each (as --batch, with the same outputs).")
    return p


def _mode_name(path, mode):
    base, ext = os.path.splitext(os.path.basename(path))
    return os.path.join(os.path.dirname(path), "{}-mode{}{}".format(base, mode, ext))


def plan_jobs(args):
    """[(infile, outfile, mode)] for the parsed arguments; raises the reference's AssertionError /
    ValueError texts on bad input (voicefixer/__main__.py:36-68,147-153)."""
    process_file, process_folder = len(args.infile) != 0, len(args.infolder) != 0
    assert process_file or process_folder, (
        "Error: You need to specify a input file path (--infile) or a input folder path (--infolder) to proceed. "
        "For more information please run: voicefixer -h")
    modes = [0, 1, 2] if args.mode == "all" else [int(args.mode)]
    name = (lambda path, m: _mode_name(path, m)) if args.mode == "all" else (lambda path, m: path)
    jobs = []
    if process_file:
        assert os.path.exists(args.infile), "Error: The input file %s is not found." % args.infile
        fmt = re.search(r"\.(\w+)$", args.outfile)
        assert fmt is not None, "Error: A file-extension for the outfile is missing."
        assert fmt.groups()[0].upper() in OUTPUT_FORMATS, "Error: Unsupported output format."
        ext = os.path.splitext(os.path.basename(args.infile))[-1]
        if ext != ".wav":
            raise ValueError("Error: Error processing the input file. We only support the .wav format currently. "
                             "Please convert your %s format to .wav. Thanks." % ext)
        jobs += [(args.infile, name(args.outfile, m), m) for m in modes]
    if process_folder:
        assert os.path.exists(args.infolder), "Error: The input folder %s is not found." % args.infolder
        for f in sorted(os.listdir(args.infolder)):
            if os.path.splitext(f)[-1] == ".wav":
                src, dst = os.path.join(args.infolder, f), os.path.join(args.outfolder, f)
                jobs += [(src, name(dst, m), m) for m in modes]
    return jobs


def execute(vf, jobs, batch=False, cuda=True, say=print, channels="mix", gpus=1):
    """Runs [(src, dst, mode)] with the VoiceFixer vf: one file at a time, or with batch through vf.restore_files, which
    prints the same `Processing` line per job as its wave starts and one `Restoration took` line per wave.
    channels: restore()'s ("mix" or "keep").  gpus > 1 runs the jobs through vf.restore_files(..., gpus=gpus) whatever
    batch is; each device then prints its own lines, the `Processing` ones only when say is print, and lines from
    different devices interleave.

    One file at a time is restore_files' pipeline (api.run_waves) with a budget of 0, so that every job is a wave of
    its own: a reader thread decodes the next inputs, the calling thread restores one job with vf.restore_inmem (or
    vf.restore_columns), a writer thread writes the previous outputs with wavio.save_wave.  An input that the job before
    also read (`--mode all`) is decoded once.  Every job before a failing one is written, nothing after it is started."""
    from . import api, wavio
    if gpus != 1 and jobs:
        vf.restore_files([j[0] for j in jobs], [j[1] for j in jobs], mode=[j[2] for j in jobs], cuda=cuda,
                         channels=channels, gpus=gpus, _messages=("processing", "took") if say is print else ("took",))
    elif not batch:
        if channels == "keep":                                            # = vf.restore(..., channels="keep") per job
            read = lambda src: wavio.read_wave(src, 44100)                # noqa: E731
            run = vf.restore_columns
        else:                                                             # = vf.restore(input, output, ...) per job
            read = lambda src: vf._load_wav(src, sample_rate=44100)       # noqa: E731  base.py:141-146, staged
            run = vf.restore_inmem

        def load(i, prev):                    # length 1: a 0 fits budget 0, and every job would join one wave
            return (read(jobs[i][0]) if prev is None else prev), 1

        def restore(wave):
            [(i, wav)] = wave
            say("Processing {}, mode={}".format(jobs[i][0], jobs[i][2]))
            t0 = time.time()
            out = run(wav, cuda=cuda, mode=jobs[i][2])
            print("Restoration took {} s".format(round(time.time() - t0, 1)))
            return out

        api.run_waves([j[0] for j in jobs], 0, load, restore,
                      lambda ids, out: wavio.save_wave(out, fname=jobs[ids[0]][1], sample_rate=44100))
    elif jobs:
        kw = {"channels": channels} if channels != "mix" else {}        # "mix" is restore_files' default
        vf.restore_files([j[0] for j in jobs], [j[1] for j in jobs], mode=[j[2] for j in jobs], cuda=cuda, **kw,
                         _on_wave=lambda ids: [say("Processing {}, mode={}".format(jobs[i][0], jobs[i][2])) for i in ids],
                         _on_wave_done=lambda ids, s: print("Restoration took {} s".format(round(s, 1))))


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.weight_prepare:
        from . import api
        for rel in (api.ANALYSIS_CKPT, api.VOCODER_CKPT):
            if not os.path.exists(os.path.join(os.path.expanduser("~"), rel)):
                print("missing checkpoint: ~/" + rel)
                return 1
        return 0
    jobs = plan_jobs(args)
    say = (lambda *a: None) if args.silent else print
    for _, dst, _ in jobs:
        d = os.path.dirname(dst)
        if len(d) > 1:
            os.makedirs(d, exist_ok=True)
    say("Initializing VoiceFixer")
    from .api import VoiceFixer
    vf = VoiceFixer()
    say("Start processing %d job(s)." % len(jobs))
    t0 = time.time()
    execute(vf, jobs, batch=args.batch, cuda=not args.disable_cuda, say=say,
            channels="keep" if args.keep_channels else "mix", gpus=args.gpus)
    say("Done: {} job(s) in {} s".format(len(jobs), round(time.time() - t0, 3)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
