"""Command line mirror of the reference's `voicefixer` entry point (voicefixer/__main__.py:13-219):

    python -m voicefixer_b200 --infile in.wav --outfile out.wav [--mode 0|1|2|all]
    python -m voicefixer_b200 --infolder wavs/ --outfolder restored/ [--mode ...] [--batch] [--keep-channels]

Same flags, same output naming (`--mode all` writes `<name>-mode<k><ext>` for k = 0,1,2), same
`.wav`-only input rule, same messages.  The work is planned first (`plan_jobs`, a pure function) and
then executed with one VoiceFixer instance as a reader -> GPU -> writer pipeline (`run_jobs`), one
file at a time; with `--batch` the same jobs run through `VoiceFixer.restore_files`, many files per
batch (`execute`).  With `--keep-channels` every channel of a file is restored and written (restore(...,
channels="keep")), on either path, with the same bytes."""
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


def run_jobs(jobs, load, restore, save, say=print, depth=2):
    """Executes [(src, dst, mode)] as a three-stage pipeline so that disk and codec time hide behind GPU time:
    a reader thread decodes / resamples the next inputs (`load(src)`), the calling thread runs `restore(wav, mode)`
    on the GPU, a writer thread encodes and writes the previous results (`save(out, dst)`).  At most `depth` decoded
    inputs and `depth` finished outputs are in flight.  Jobs complete in order; like the sequential loop of the reference,
    every job before a failing one is still written, nothing after it is started, and the exception is re-raised once
    the threads have drained.  A source that is
    used by consecutive jobs (`--mode all`) is decoded once.  Returns the per-job GPU-stage seconds."""
    import queue
    import threading
    loaded, finished, took = queue.Queue(maxsize=depth), queue.Queue(maxsize=depth), []
    stop, write_errors = threading.Event(), []

    def reader():                                        # failures travel down the queue IN ORDER, so that every
        last_src, last_wav = None, None                  # job before the failing one still completes
        try:
            for job in jobs:
                if stop.is_set():
                    break
                if job[0] != last_src:
                    last_src, last_wav = job[0], load(job[0])
                loaded.put((job, last_wav))
        except BaseException as e:                       # noqa: BLE001 - re-raised by the caller's thread
            loaded.put(e)
        finally:
            loaded.put(None)

    def writer():
        while True:
            item = finished.get()
            if item is None:
                return
            if write_errors:
                continue                                 # drain
            try:
                save(item[1], item[0][1])
            except BaseException as e:                   # noqa: BLE001
                write_errors.append(e)
                stop.set()

    threads = [threading.Thread(target=reader, name="vfx-reader", daemon=True),
               threading.Thread(target=writer, name="vfx-writer", daemon=True)]
    for t in threads:
        t.start()
    failure = None
    try:
        while True:
            item = loaded.get()
            if item is None:
                break
            if failure is not None or stop.is_set():
                continue                                 # keep draining so the reader can finish
            if isinstance(item, BaseException):
                failure = item
                stop.set()
                continue
            (src, dst, mode), wav = item
            say("Processing {}, mode={}".format(src, mode))
            t0 = time.time()
            try:
                out = restore(wav, mode)
            except BaseException as e:                   # noqa: BLE001
                failure = e
                stop.set()
                continue
            took.append(time.time() - t0)
            print("Restoration took {} s".format(round(took[-1], 1)))
            finished.put((item[0], out))
    finally:
        finished.put(None)
        for t in threads:
            t.join()
    if write_errors:
        raise write_errors[0]
    if failure is not None:
        raise failure
    return took


def execute(vf, jobs, batch=False, cuda=True, say=print, channels="mix"):
    """Runs [(src, dst, mode)] with the VoiceFixer vf: one file at a time through run_jobs, or with batch through
    vf.restore_files, which prints the same `Processing` line per job as its wave starts and one `Restoration took`
    line per wave.  channels: restore()'s ("mix" or "keep")."""
    from . import wavio
    if not batch:
        if channels == "keep":                                            # = vf.restore(..., channels="keep") per job
            load = lambda src: wavio.read_wave(src, 44100)                # noqa: E731
            restore = lambda wav, mode: vf.restore_columns(wav, cuda=cuda, mode=mode)   # noqa: E731
        else:                                                             # = vf.restore(input, output, ...) per job
            load = lambda src: vf._load_wav(src, sample_rate=44100)       # noqa: E731  base.py:141-146, staged
            restore = lambda wav, mode: vf.restore_inmem(wav, cuda=cuda, mode=mode)     # noqa: E731
        run_jobs(jobs, load=load, restore=restore,
                 save=lambda out, dst: wavio.save_wave(out, fname=dst, sample_rate=44100), say=say)
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
            channels="keep" if args.keep_channels else "mix")
    say("Done: {} job(s) in {} s".format(len(jobs), round(time.time() - t0, 3)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
