"""Drop-in mirror of the reference's public API (voicefixer/base.py, voicefixer/vocoder/base.py).

Same class names, method signatures, checkpoint paths and error types; the bodies run the
hand-written sm_90a kernels through the C-ABI engine.  The `cuda` argument is accepted for
signature compatibility: the computation always runs on the GPU (there is no CPU path)."""
import numbers
import os
from collections import deque

import numpy as np
import torch

from .engine import Engine, default_precision
from ._lib import PCM16_MAX_CHANNELS
from . import resample, wavio

SEG_LENGTH = 44100 * 30                      # voicefixer/base.py:116
ANALYSIS_CKPT = ".cache/voicefixer/analysis_module/checkpoints/vf.ckpt"
VOCODER_CKPT = ".cache/voicefixer/synthesis_module/44100/model.ckpt-1490000_trimed.pt"

_ERR0 = ("Error 0: The checkpoint for analysis module (vf.ckpt) is not found in "
         "~/.cache/voicefixer/analysis_module/checkpoints.")
_ERR1 = ("Error 1: The checkpoint for synthesis module / vocoder (model.ckpt-1490000_trimed) is not found in "
         "~/.cache/voicefixer/synthesis_module/44100.")


def _check_cuda(cuda):
    # tools/pytorch_util.py:6-8
    if not torch.cuda.is_available():
        if cuda:
            raise RuntimeError("Error: You set cuda=True but no cuda device found.")
        raise RuntimeError("voicefixer_b200 has no CPU path: an H100 (sm_90a) device is required.")


def _load_vocoder_state():
    path = os.path.join(os.path.expanduser("~"), VOCODER_CKPT)
    if not os.path.exists(path):
        raise RuntimeError(_ERR1)
    return torch.load(path, map_location="cpu")["generator"]


def ragged_plan(wavs):
    """Validates the list form of VoiceFixer.restore_batch: a non-empty list of 1-D arrays of 1025 .. 30 s samples each.
    Returns (items as contiguous float32 arrays, their lengths, L_cap): L_cap is the longest length rounded up to a
    whole second, so batches of other lengths under the same cap share one captured graph."""
    if len(wavs) == 0:
        raise ValueError("restore_batch takes a non-empty list of 1-D arrays")
    items, lens = [], []
    for i, w in enumerate(wavs):
        a = np.ascontiguousarray(w, dtype=np.float32)
        if a.ndim != 1:
            raise ValueError(f"restore_batch: item {i} has shape {a.shape}; the list form takes 1-D arrays, one utterance each")
        if a.shape[0] <= 1024:
            raise ValueError(f"restore_batch: item {i} has {a.shape[0]} samples; the front end reflect-pads 1024, "
                             "so every item needs at least 1025")
        if a.shape[0] > SEG_LENGTH:
            raise ValueError(f"restore_batch: item {i} has {a.shape[0]} samples, more than 30 s "
                             "(longer inputs: restore_inmem segments them)")
        items.append(a)
        lens.append(a.shape[0])
    L_cap = -(-max(lens) // 44100) * 44100
    return items, lens, L_cap


_MODE2_MSG = ("Expected more than 1 value per channel when training, got input size "
              "torch.Size([1, 384, 1, 1])")


def segment_bounds(n):
    """[(start, stop)] of the 30 s segments restore_inmem cuts a recording of n samples into (voicefixer/base.py:117-119):
    full segments, then the rest; a recording of a whole number of segments has no empty tail."""
    return [(a, min(a + SEG_LENGTH, n)) for a in range(0, n, SEG_LENGTH)]


def _net_len(L, mode):
    """Samples a segment of L samples has after the mode-1 pre-filter (512 * (L // 512)); L in the other modes."""
    return 512 * (L // 512) if mode == 1 else L


def _gen_len(T):
    """Samples the Generator writes for a mel of T frames."""
    return (T + T % 2 + 4) * 441


def _pack(lengths, max_items):
    """Packs items of the given lengths into ragged batches [(cap, [index, ...]), ...]: longest first (stable on ties), each
    batch the longest item left, cap being its length, plus up to max_items(cap) - 1 of the next ones (so at least one).
    max_items is called once per batch, in batch order."""
    order = sorted(range(len(lengths)), key=lambda i: -lengths[i])
    batches, k = [], 0
    while k < len(order):
        cap = lengths[order[k]]
        n = max(1, int(max_items(cap)))
        batches.append((cap, order[k:k + n]))
        k += n
    return batches


def plan_many(lengths, mode, max_items, what="restore_many"):
    """Segments the recordings of the given lengths exactly as restore_inmem does and packs all their segments into ragged
    batches by length with _pack (VoiceFixer.restore_many), L_cap being a batch's longest segment (its capacity).
    Returns [(L_cap, [(recording, start, stop), ...]), ...].

    Raises ValueError, naming the recording and starting `<what>`, before anything runs: for an empty list, a segment of
    1024 samples or fewer (after the mode-1 pre-filter's 512 * (L // 512) in mode 1: the front end reflect-pads 1024), or
    in mode 2 a segment of 64 frames or fewer (the reference's train-mode BatchNorm refuses its 1 x 1 UNet centre)."""
    if mode not in (0, 1, 2):
        raise ValueError("mode must be 0, 1 or 2")
    if len(lengths) == 0:
        raise ValueError(f"{what} takes a non-empty list of 1-D arrays")
    segs = []
    for i, n in enumerate(lengths):
        bounds = segment_bounds(int(n))
        if not bounds:
            raise ValueError(f"{what}: recording {i} is empty")
        for a, b in bounds:
            L = b - a
            Lnet = _net_len(L, mode)
            if mode == 2 and 1 + Lnet // 441 <= 64:
                raise ValueError(f"{what}: recording {i}, samples {a}..{b}: {_MODE2_MSG}")
            if Lnet <= 1024:
                size = f"{L} samples, {Lnet} after the mode-1 pre-filter" if mode == 1 else f"{L} samples"
                raise ValueError(f"{what}: recording {i} has a segment (samples {a}..{b}) of {size}; the front end "
                                 "reflect-pads 1024, so every segment needs at least 1025")
            segs.append((i, a, b))
    return [(L_cap, [segs[j] for j in idx]) for L_cap, idx in _pack([b - a for _, a, b in segs], max_items)]


def plan_waves(lengths, budget):
    """The waves VoiceFixer.restore_files runs files in: consecutive runs of indices into lengths (the files' lengths at
    44.1 kHz), in input order, every index in exactly one.  A wave takes the next file while the lengths in it still sum
    to at most budget samples; a file longer than budget is a wave of its own (restore_many cuts it into batches).
    A generator that reads lengths lazily: each wave is yielded once the first length past it is known, so a reader can
    decode the files as it goes."""
    wave, total = [], 0
    for i, n in enumerate(lengths):
        if wave and total + int(n) > budget:
            yield wave
            wave, total = [], 0
        wave.append(i)
        total += int(n)
    if wave:
        yield wave


def file_samples(shape, sr, mode, src):
    """The samples a file counts against VoiceFixer.restore_files' wave budget (plan_waves): its length at 44.1 kHz
    times the channels restored, shape being the decoded file's, (L,) for a mono mix or (L, C) with every channel kept.
    Raises ValueError naming src for what restore_many would refuse (plan_many) and for more than PCM16_MAX_CHANNELS
    channels, the most one file of the device packer (Engine.pack_pcm16) and one FLAC stream hold."""
    C = shape[1] if len(shape) == 2 else 1
    if C > PCM16_MAX_CHANNELS:
        raise ValueError(f"restore_files: {src} has {C} channels; channels=\"keep\" restores at most "
                         f"{PCM16_MAX_CHANNELS} per file (the device packer's bound, and the most a FLAC stream holds)")
    n44 = resample.out_len(shape[0], sr)
    plan_many([n44], mode, lambda L: 1, what=f"restore_files: {src}")             # restore_many's refusals
    return n44 * C


def run_waves(srcs, budget, load, restore, write, depth=2):
    """The pipeline of VoiceFixer.restore_files over jobs 0 .. len(srcs) - 1, srcs[i] being job i's input file:

    a reader thread calls load(i, prev) -> (item, length at 44.1 kHz) for each job in order and groups the jobs into
    waves by plan_waves(lengths, budget).  prev is the item load returned for an earlier job of the same wave with the
    same source, or None: load then checks that item for job i rather than reading the file again.
    The calling thread calls restore(wave) -> result for each wave [(i, item), ...]; it may return before the GPU is done.
    A writer thread calls write([i, ...], result) for each wave, which writes the wave's outputs in order.

    At most `depth` loaded and `depth` restored waves are in flight.  Errors follow run_jobs's order rule: a failing load
    cuts its wave short (the jobs before it in the wave are restored and written), a failing restore fails its wave,
    every job before the failure is written and nothing after it is started, and the exception is re-raised once the
    threads have drained.  The exception's `vfx_job` attribute is then the job it stopped at: the one whose load failed,
    the first of a failed wave, or for a failed write the job write set it to (else the wave's first).  Returns the
    number of waves restored."""
    import queue
    import threading
    loaded, finished = queue.Queue(maxsize=depth), queue.Queue(maxsize=depth)
    stop, write_errors = threading.Event(), []

    def reader():
        pending = {}                                     # job -> item: loaded and not yet handed on
        at = [0]                                         # the job being loaded

        def lengths():
            for i, src in enumerate(srcs):
                if stop.is_set():
                    return
                at[0] = i
                prev = next((pending[j] for j in pending if srcs[j] == src), None)
                pending[i], n = load(i, prev)
                yield n

        try:
            for wave in plan_waves(lengths(), budget):
                loaded.put([(i, pending.pop(i)) for i in wave])
        except BaseException as e:                       # noqa: BLE001 - re-raised by the caller's thread
            if pending:                                  # the jobs before the failing one
                loaded.put(sorted(pending.items()))
            loaded.put(_stopped_at(e, at[0]))
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
                write(*item)
            except BaseException as e:                   # noqa: BLE001
                write_errors.append(_stopped_at(e, item[0][0]))
                stop.set()

    threads = [threading.Thread(target=reader, name="vfx-wave-reader", daemon=True),
               threading.Thread(target=writer, name="vfx-wave-writer", daemon=True)]
    for t in threads:
        t.start()
    failure, waves = None, 0
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
            try:
                result = restore(item)
            except BaseException as e:                   # noqa: BLE001
                failure = _stopped_at(e, item[0][0])
                stop.set()
                continue
            waves += 1
            finished.put(([i for i, _ in item], result))
    finally:
        finished.put(None)
        for t in threads:
            t.join()
    if write_errors:
        raise write_errors[0]
    if failure is not None:
        raise failure
    return waves


def _stopped_at(e, job):
    """e, with `vfx_job` (the job run_waves stopped at) set to job unless a stage closer to the failure set it."""
    if getattr(e, "vfx_job", None) is None:
        e.vfx_job = job
    return e


def plan_devices(weights, sources, n):
    """The files of VoiceFixer.restore_files(..., gpus=n) per device: n lists of indices into weights (each file's
    samples against a wave, file_samples' count; 0 for a file that cannot be probed) that together hold every index
    once, each in input order.  Every occurrence of one source (an input listed several times, as --mode all does) goes
    to one device, so that it is decoded once; these groups are placed longest first, each on the least-loaded device
    (ties: the lower index), so the largest load is at most the largest group's weight plus the mean load.  A device
    gets no files when there are fewer groups than devices."""
    groups = {}
    for i, src in enumerate(sources):
        groups.setdefault(src, []).append(i)
    groups = sorted(groups.values(), key=lambda g: (-sum(int(weights[i]) for i in g), g[0]))
    loads, shards = [0] * n, [[] for _ in range(n)]
    for g in groups:
        d = min(range(n), key=lambda k: (loads[k], k))
        shards[d] += g
        loads[d] += sum(int(weights[i]) for i in g)
    return [sorted(s) for s in shards]


def _probe_samples(inputs, modes, keep):
    """plan_devices' weights: file_samples' count for each input from its headers (wavio.probe), 0 where that fails."""
    probed, weights = {}, []
    for src, m in zip(inputs, modes):
        try:
            if src not in probed:
                probed[src] = wavio.probe(src)
            frames, ch, sr = probed[src]
            weights.append(file_samples((frames, ch) if keep else (frames,), sr, m, src))
        except Exception:                                 # noqa: BLE001 - its error surfaces on its device, as today
            weights.append(0)
    return weights


class _ShardArgs:
    """What every device's shard of restore_files(..., gpus=N) shares: the caller's VoiceFixer (vf, which stays in the
    calling process: a worker receives None and builds its own), the engine's precision, weight layout and arena in
    host shared memory, and the call's arguments over all files."""

    def __init__(self, vf, **kw):
        self.vf = vf
        self.__dict__.update(kw)

    def __getstate__(self):
        return dict(self.__dict__, vf=None)


def _restore_shard(device, shard, args):
    """parallel.run_on_devices' target for restore_files(..., gpus=N): restores the files `shard` (indices into the
    call's lists) on device with the single-device restore_files, on the caller's VoiceFixer in the calling process and
    on one around the shared weights in a worker.  Returns None, or (the index of the file it stopped at, the error)."""
    vf = args.vf
    if vf is None:
        torch.cuda.set_device(device)
        eng = Engine(device=device, precision=args.precision)
        eng.attach(args.arena.to(f"cuda:{device}"), args.table)
        vf = VoiceFixer.from_engine(eng)
    modes = [args.modes[i] for i in shard]
    seeds = [args.seeds[i] for i in shard] if args.seeds is not None and 2 in modes else None
    kw = {}
    if "processing" in args.messages:
        kw["_on_wave"] = lambda ids: [print(f"Processing {args.inputs[shard[i]]}, mode={modes[i]}", flush=True)
                                      for i in ids]
    if "took" in args.messages:
        kw["_on_wave_done"] = lambda ids, s: print("Restoration took {} s".format(round(s, 1)), flush=True)
    try:
        vf.restore_files([args.inputs[i] for i in shard], [args.outputs[i] for i in shard], mode=modes,
                         dropout_seed=seeds, channels=args.channels, _budget=args.budget, **kw)
    except Exception as e:                               # noqa: BLE001 - reported by run_on_devices
        return shard[getattr(e, "vfx_job", None) or 0], e
    return None


def plan_vocoder_many(items, kind, max_items, pack_lengths=None):
    """Packs the items of Vocoder.forward_many (kind "mel": [1, 1, T, 128] mels) or Vocoder.oracle_many (kind "wav": 1-D
    float32 recordings) into ragged batches by length with _pack, cap being a batch's longest item in frames (mels) or
    samples (recordings): its capacity.  Returns [(cap, [item, ...]), ...].  pack_lengths (optional): the lengths to pack
    by in place of the items' own, e.g. recordings' lengths at 44.1 kHz when they are resampled on the device; the items
    are validated all the same.

    Raises before anything is sized or launched, naming the item: ValueError for an empty list, a mel that is not
    [1, 1, T >= 1, 128], or a recording that is empty, not 1-D or all zeros (the reference divides by its zero peak);
    AssertionError for a mel whose last dimension is not 128, as Vocoder.forward asserts.  A recording that is a CUDA
    tensor is not checked for all zeros: that would read it on the host."""
    what = {"mel": "forward_many", "wav": "oracle_many"}[kind]
    if len(items) == 0:
        raise ValueError(f"{what} takes a non-empty list")
    lengths = []
    for i, x in enumerate(items):
        shape = tuple(x.shape)
        if kind == "mel":
            if len(shape) >= 1 and shape[-1] != 128:
                raise AssertionError(f"{what}: item {i} has shape {shape}; the mel must have 128 bins")
            if len(shape) != 4 or shape[:2] != (1, 1) or shape[2] < 1:
                raise ValueError(f"{what}: item {i} has shape {shape}; each mel must be [1, 1, T >= 1, 128]")
            lengths.append(shape[2])
        else:
            if len(shape) != 1:
                raise ValueError(f"{what}: item {i} has shape {shape}; each recording must be 1-D")
            if shape[0] == 0:
                raise ValueError(f"{what}: item {i} is empty")
            if not is_cuda(x) and not np.any(x):          # a device item is not read on the host
                raise ValueError(f"{what}: item {i} is all zeros; its peak normalisation would divide by zero")
            lengths.append(shape[0])
    if pack_lengths is not None:
        lengths = [int(n) for n in pack_lengths]
    return _pack(lengths, max_items)


def is_cuda(w):
    """Whether w is a CUDA tensor (anything else, e.g. an array or a list, is not)."""
    return getattr(w, "is_cuda", False) is True


def check_device_items(wavs, device, what):
    """True when every item of wavs (restore_many / oracle_many) is a CUDA tensor, False when none is (the host path).
    Raises ValueError naming the recording, before anything is launched, for a list that mixes CUDA and host items, and
    for a CUDA item that is on another device than `device` (a torch.device), not float32, not 1-D, or of element stride
    0 (an expanded tensor).  Any positive element stride is accepted."""
    cuda = [is_cuda(w) for w in wavs]
    if not any(cuda):
        return False
    if not all(cuda):
        raise ValueError(f"{what}: recording {cuda.index(False)} is not a CUDA tensor but recording {cuda.index(True)} is; "
                         "give every recording as a CUDA tensor, or none")
    for i, w in enumerate(wavs):
        if torch.device(w.device) != torch.device(device):
            raise ValueError(f"{what}: recording {i} is on {w.device}; this engine runs on {device}")
        if w.dtype != torch.float32:
            raise ValueError(f"{what}: recording {i} has dtype {w.dtype}; CUDA recordings must be torch.float32")
        if len(w.shape) != 1:
            raise ValueError(f"{what}: recording {i} has shape {tuple(w.shape)}; each recording must be 1-D")
        if w.stride(0) < 1:
            raise ValueError(f"{what}: recording {i} has element stride {w.stride(0)} (an expanded tensor); its samples "
                             "must be distinct elements (.contiguous() makes them so)")
    return True


def resample_rows(ranges, rates):
    """The input rows of a batch of CUDA recordings: ranges = [(recording, a, b), ...] of their 44.1 kHz streams, rates
    one per recording -> one (recording, rate, y_first, y_len) per row (Engine.resample_src; 44100 is a copy)."""
    return [(i, int(rates[i]), int(a), int(b - a)) for i, a, b in ranges]


def restore_out_len(n, mode):
    """Samples restore_many returns for a recording of n samples at 44.1 kHz: its segments' _net_len, summed."""
    return sum(_net_len(b - a, mode) for a, b in segment_bounds(int(n)))


def restore_rows(segs, mode):
    """Where each row of a restore_many batch of CUDA recordings goes: segs = [(recording, a, b), ...] (plan_many) -> one
    (recording, dst_off, len) per row (Engine.scatter_rows): the segment's _net_len(b - a, mode) restored samples at its
    offset in its recording's output, after the full 30 s segments before it."""
    return [(i, (a // SEG_LENGTH) * _net_len(SEG_LENGTH, mode), _net_len(b - a, mode)) for i, a, b in segs]


def oracle_rows(idx, lengths):
    """Where each row of an oracle_many batch of CUDA recordings goes: items idx (plan_vocoder_many) of lengths[i]
    samples at 44.1 kHz -> one (item, 0, _gen_len(1 + lengths[i] // 441)) per row: the whole output of the item."""
    return [(i, 0, _gen_len(1 + lengths[i] // 441)) for i in idx]


def stream_rows(rows):
    """The tables of one device StreamPool step: rows = [(rate, base, n, (lo, hi, keep_lo, keep_hi)), ...], one per
    window, its stream holding input samples [base, n) at `rate`, base a multiple of down ((up, down) =
    resample.ratio(rate)), and every input the window reads at or after base.  Returns (gather, emit):

    gather: one (n_in, y_first, y_len) per row (Engine.resample_src): the window is output samples [y_first, y_first +
    y_len) of the held input read as a recording of its own, n_in = n - base samples.  With base = k * down, output J
    of the stream is output J - k * up of that recording: both sum the same inputs with the same taps in the same
    order, so the row is bit-identical to the window resampled from the whole stream.
    emit: one (src_off, len) per row (Engine.scatter_rows): the kept samples [keep_lo, keep_hi) start src_off = keep_lo
    - lo samples into the window's row."""
    gather, emit = [], []
    for rate, base, n, (lo, hi, keep_lo, keep_hi) in rows:
        up, down = resample.ratio(rate)
        if base % down:
            raise ValueError(f"stream_rows: base {base} is not a multiple of down = {down} (rate {rate})")
        gather.append((int(n - base), int(lo - base // down * up), int(hi - lo)))
        emit.append((int(keep_lo - lo), int(keep_hi - keep_lo)))
    return gather, emit


class StreamSchedule:
    """The window rule of VoiceFixer.restore_stream and StreamPool in `mode`, in samples at 44.1 kHz.  Each chunk of
    `chunk` samples is restored inside the window [pos - ctx, pos + chunk + ctx), clipped to the stream, as soon as that
    window has arrived; at the end of the stream the last windows are flushed without (full) look-ahead.  Only the chunk
    itself is kept from each window.  No window is shorter than min_len, the shortest window the mode can restore, or
    longer than capacity.

    Mode 1's pre-filter keeps the first 512 * (n // 512) samples of a window of n (as restore_inmem keeps them of each
    30 s segment, voicefixer/base.py:121-122), so a window [lo, hi) emits only the kept samples below
    lo + 512 * ((hi - lo) // 512); pos still moves past the lost ones.  With ctx >= 511 no sample is lost but the
    stream's last (hi - lo) % 512 <= 511 (a flush window that reaches the stream's end keeps everything up to it); with
    ctx = 0 every window loses its last (hi - lo) % 512 samples, as the 30 s segments do."""

    # the shortest window of each mode: the front end reflect-pads 1024 (base.py:78); mode 1's pre-filter keeps
    # 512 * (L // 512) samples, which must exceed 1024 (plan_many); mode 2 needs 1 + L // 441 > 64 frames (_MODE2_MSG)
    MIN_LEN = {0: 1025, 1: 1536, 2: 64 * 441}
    _WHY = {0: "the front end reflect-pads 1024",
            1: "mode 1's pre-filter keeps 512 * (L // 512) samples of L and the front end reflect-pads 1024",
            2: "mode 2's train-mode statistics need more than 64 frames (1 + L // 441 > 64)"}

    def __init__(self, chunk, ctx, mode=0):
        if mode not in (0, 1, 2):
            raise ValueError("mode must be 0, 1 or 2")
        self.chunk, self.ctx, self.mode = int(chunk), int(ctx), mode
        self.min_len = m = self.MIN_LEN[mode]
        # the longest window due() returns: chunk + 2 ctx for a full window; a flush window shorter than min_len samples
        # is widened to min_len + ctx; with ctx = 0 a flush window may take in a tail of up to min_len - 1 samples after
        # its chunk
        if self.ctx == 0:
            self.capacity = max(self.chunk + m - 1, m)
        else:
            self.capacity = max(self.chunk + 2 * self.ctx, m + self.ctx)

    def check_first_window(self, who):
        """Raises ValueError `<who>: ...` when a stream's first window, chunk + ctx samples, is shorter than min_len."""
        if self.chunk + self.ctx < self.min_len:
            raise ValueError(f"{who}: chunk_seconds + context_seconds is {self.chunk + self.ctx} samples, the length of "
                             f"a stream's first window; {self._WHY[self.mode]}, so it needs at least {self.min_len}")

    def due(self, pos, avail, ended):
        """([(lo, hi, keep_lo, keep_hi), ...], new pos): the windows that are due once samples [0, avail) of the stream
        have arrived (and nothing more will, if `ended`) and every sample before `pos` has been scheduled.  Window
        [lo, hi) is restored whole and its samples [keep_lo, keep_hi) are emitted; the new pos follows the last of them
        (in mode 1 also the samples the pre-filter dropped).  Raises RuntimeError, restore_stream's message, when an
        ended stream leaves a flush window that cannot reach min_len samples."""
        chunk, ctx, m = self.chunk, self.ctx, self.min_len
        windows = []
        while avail >= pos + chunk + ctx:                                # a full chunk plus its look-ahead has arrived
            lo, hi = max(0, pos - ctx), pos + chunk + ctx
            windows.append((lo, hi, pos, self._kept(lo, hi, pos, pos + chunk)))
            pos += chunk
        while ended and pos < avail:                                     # flush: the last windows have no (full) look-ahead
            hi = min(avail, pos + chunk + ctx)
            keep_hi = min(avail, pos + chunk)
            if 0 < avail - keep_hi < m and ctx == 0:                     # never leave a tail too short to restore
                keep_hi = hi = avail
            if self.mode == 1 and hi == avail:       # the next window would re-read this one's end: lose nothing mid-stream
                keep_hi = avail
            lo = max(0, pos - ctx)
            if hi - lo < m:                                              # e.g. reflect padding needs > 1024 (base.py:78)
                lo = max(0, hi - m - ctx)
                if hi - lo < m:
                    raise RuntimeError(f"restore_stream: fewer than {m} samples in total; {self._WHY[self.mode]}")
            windows.append((lo, hi, pos, self._kept(lo, hi, pos, keep_hi)))
            pos = keep_hi
        return windows, pos

    def _kept(self, lo, hi, keep_lo, keep_hi):
        """keep_hi, clipped in mode 1 to the samples the pre-filter keeps of the window [lo, hi)."""
        if self.mode != 1:
            return keep_hi
        return max(keep_lo, min(keep_hi, lo + 512 * ((hi - lo) // 512)))


class _Stream:
    """One stream of a StreamPool: its recent input at its own rate, where its schedule stands, and in mode 2 its dropout
    seed; window k of the stream (counting from 0) draws its masks from key (seed, k)."""

    def __init__(self, rate, seed=None):
        self.rate = rate
        self.seed = seed
        self.restored = 0                          # windows restored so far: the index of the oldest pending one
        self._data = np.zeros(0, dtype=np.float32)  # buf = _data[_lo:_hi], grown by doubling: a push copies its block once
        self._lo = self._hi = 0
        self.base = 0                              # buf holds input samples [base, n) at `rate`
        self.n = 0                                 # input samples received
        self.pos = 0                               # next 44.1 kHz sample to schedule
        self.pending = deque()                     # windows scheduled and not yet restored, oldest first
        self.closed = False

    @property
    def buf(self):
        return self._data[self._lo:self._hi]

    def append(self, a):
        if self._hi + a.shape[0] > self._data.shape[0]:
            held = self.buf
            self._data = np.empty(max(4096, 2 * (held.shape[0] + a.shape[0])), dtype=np.float32)
            self._data[:held.shape[0]] = held
            self._lo, self._hi = 0, held.shape[0]
        self._data[self._hi:self._hi + a.shape[0]] = a
        self._hi += a.shape[0]
        self.n += a.shape[0]

    def drop_before(self, first):
        """Forgets the input before sample `first`."""
        if first > self.base:
            self._lo += first - self.base
            self.base = first


class _DevStream(_Stream):
    """One stream of a device StreamPool: _Stream's bookkeeping, its recent input at its own rate in one device buffer
    (grown by doubling: a push copies its block in once, from any element stride).  Old input is dropped by moving the
    start, as _Stream does, but only to a multiple of down ((up, down) = resample.ratio(rate)): base stays a multiple
    of down, so the held input is a recording of its own to the resampler (stream_rows), and at most down - 1 samples
    more than _Stream's are held."""

    def __init__(self, rate, device, seed=None):
        super().__init__(rate, seed)
        self.down = resample.ratio(rate)[1]
        self._data = torch.empty(0, device=device)

    def append(self, a, st=None):
        """a: a 1-D float32 tensor on the buffer's device.  st: the stream the copy runs on; a buffer this replaces is
        not reused before st's queued work (which follows every earlier read of it) is done."""
        m = a.shape[0]
        if self._hi + m > self._data.shape[0]:
            held = self.buf
            data = torch.empty(max(4096, 2 * (held.shape[0] + m)), device=self._data.device)
            data[:held.shape[0]].copy_(held)
            self.release(st)
            self._data = data
            self._lo, self._hi = 0, held.shape[0]
        self._data[self._hi:self._hi + m].copy_(a)
        self._hi += m
        self.n += m

    def drop_before(self, first):
        super().drop_before(first - first % self.down)

    def release(self, st):
        """Hands the buffer back to the allocator for reuse only after st's queued work is done."""
        if st is not None and self._data.numel():
            self._data.record_stream(st)


class StreamPool:
    """Many live streams restored together (VoiceFixer.stream_pool), driven by one caller thread.

    Every stream follows restore_stream's window rule (StreamSchedule) on its own 44.1 kHz samples.  A window is due as
    soon as the input it needs has arrived; step() restores the due windows of all streams, oldest first, as one ragged
    batch: the rows of a (B, window_len) input, B the smallest bucket (a power of two, or max_windows) that holds them,
    and one replay of a restore graph captured for that bucket.  The concatenation of everything step() returns for a
    stream is bit-identical to restore_stream on that stream's audio alone, however pushes, closes and steps interleave.

    A stream at another rate than 44.1 kHz is kept at its own rate on the host; its 44.1 kHz samples [0, m) are available
    once the input they read has arrived (resample.available), all of them after close().  Its windows are resampled on
    the device (Engine.resample) into the step's input rows, bit-identical to wavio._resample on the whole stream.

    Host and device pools.  The first block pushed fixes the pool's kind for its lifetime: host blocks (anything numpy
    takes), or 1-D float32 CUDA tensors on the engine's device, of any element stride >= 1 (e.g. x[:, c] of an
    interleaved (L, C) tensor).  A host pool stages each step's windows on the host and returns numpy blocks, waiting
    for the device at the end of every step.  A device pool keeps each stream's recent input in a device buffer at its
    own rate (_DevStream); a step builds all its window rows with one Engine.resample_src launch (a copy at 44.1 kHz),
    replays the bucket's graph, and copies each window's kept samples into a new 1-D float32 CUDA tensor with one
    Engine.scatter_rows launch.  Everything is queued on torch.cuda.current_stream(); push, close and step return
    without waiting for the GPU, except that the step which first uses a bucket captures its graph, and capturing
    synchronises the device once.  Each stream's device blocks are bit-identical, block by block, to the host pool's
    for the same audio and the same calls, at every rate and precision.  Calls on several CUDA streams run in the order
    they were made (Engine._shared_stream), and a stream buffer a pool replaces or forgets is not reused before the
    work that reads it is done.

    mode (0, 1 or 2, for the pool's lifetime): restore_stream's mode.  In mode 1 each bucket's graph runs the ragged
    pre-filter and then the restore (restore_many's pair); in mode 2 a restore with train-mode statistics and seeded
    dropout, window k of a stream keyed (the stream's dropout_seed, k) whatever step or bucket it runs in and whatever
    the other streams do.  The keys go to the device from pinned memory without a host wait, so a device step is still
    two library launches and one replay."""

    def __init__(self, engine, chunk_seconds=2.0, context_seconds=1.0, max_windows=None, device=None, mode=0):
        chunk = int(round(chunk_seconds * 44100))
        ctx = int(round(context_seconds * 44100))
        if chunk <= 0 or ctx < 0:
            raise ValueError("chunk_seconds must be positive and context_seconds non-negative")
        self._sched = StreamSchedule(chunk, ctx, mode)
        self._sched.check_first_window("stream_pool")
        if max_windows is not None and (isinstance(max_windows, (bool, np.bool_))
                                        or not isinstance(max_windows, numbers.Integral) or max_windows < 1):
            raise ValueError(f"stream_pool: max_windows is {max_windows!r}; give a positive integer or None")
        self.mode = mode
        self._eng = engine
        self._dev = device or f"cuda:{engine.device}"
        self._cuda = torch.device(self._dev).type == "cuda"
        self.window_len = L = self._sched.capacity
        # a row of input and of output per window, and the resampler's output row (its staged input is smaller); in
        # mode 1 also the pre-filter's, twice its output row: each bucket's graph holds rows of its own, and the buckets
        # (powers of two up to max_windows, and max_windows) hold fewer than two rows per window in all
        extra = 4 * 3 * L + (prefilter_bytes(engine, L) + 4 * L if mode == 1 else 0)
        fit = engine.max_batch(L, extra_per_item=extra)
        self.max_windows = fit if max_windows is None else min(int(max_windows), fit)
        self.buckets = sorted({1 << k for k in range(self.max_windows.bit_length())} | {self.max_windows})
        self._streams = {}
        self._queue = deque()                      # (sid, window) of every stream, in the order they fell due
        self._next_sid = 0
        self._graphs = {}                          # bucket -> captured restore graph
        self._bufs = None
        self._kind = None                          # "host" or "device": fixed by the first block pushed

    # ------------------------------------------------------------------ the caller's side
    def open(self, sample_rate=44100, dropout_seed=None):
        """Starts a stream whose blocks come at sample_rate Hz; returns its id.  dropout_seed (mode 2): an int in
        [0, 2^64) whose masks the stream's windows draw, as restore_stream(mode=2, dropout_seed=...) draws them; without
        it one is drawn from torch's CPU generator (torch.manual_seed controls it).  A bad rate or seed, or a seed in
        another mode, raises ValueError naming the stream, and uses up no id."""
        sid = self._next_sid
        who = f"stream_pool.open: stream {sid}"
        rate = resample.check_rate(sample_rate, who)
        seed = stream_dropout_seed(self.mode, dropout_seed, who)
        self._next_sid += 1
        self._streams[sid] = _DevStream(rate, self._dev, seed) if self._kind == "device" else _Stream(rate, seed)
        return sid

    def push(self, sid, block):
        """Appends a 1-D block of any size, at the stream's own rate, to stream sid: a host block, or in a device pool a
        1-D float32 CUDA tensor on the engine's device (any element stride >= 1), which is read, never written.  A
        block of the other kind than the pool's first, or a CUDA block that cannot be taken, raises ValueError naming
        the stream, before anything changes."""
        s = self._open_stream(sid, "push")
        cuda = is_cuda(block)
        if self._kind is not None and cuda != (self._kind == "device"):
            raise ValueError(f"stream_pool.push: stream {sid}: a {'CUDA' if cuda else 'host'} block in a pool of "
                             f"{'CUDA' if self._kind == 'device' else 'host'} blocks; the first block pushed fixes a "
                             "pool's kind for its lifetime")
        if cuda:
            self._check_device_block(sid, block)
            if self._kind is None:
                self._to_device()
                s = self._streams[sid]
            s.append(block, self._eng._shared_stream())
        else:
            a = np.asarray(block, dtype=np.float32)
            if a.ndim != 1:
                raise ValueError(f"stream_pool.push: stream {sid}: a block has shape {a.shape}; blocks are 1-D")
            self._kind = "host"
            s.append(a)
        self._schedule(sid, s, resample.available(s.n, s.rate), ended=False)

    def close(self, sid):
        """Marks the end of stream sid's input: its last windows fall due.  A stream of fewer than 1025 samples at
        44.1 kHz raises restore_stream's RuntimeError, naming the stream, and is dropped; the other streams go on."""
        s = self._open_stream(sid, "close")
        try:
            self._schedule(sid, s, resample.out_len(s.n, s.rate), ended=True)
        except RuntimeError as e:
            self._forget(sid)
            self._queue = deque(q for q in self._queue if q[0] != sid)
            raise RuntimeError(f"stream_pool.close: stream {sid}: {e}") from None
        s.closed = True

    def step(self):
        """Restores the due windows, oldest first, at most max_windows of them, in one graph replay; the rest wait for
        the next step.  Returns {sid: [restored blocks, in order]} for the streams that had windows in this step.  A
        stream that is closed and fully restored is forgotten afterwards."""
        n = min(len(self._queue), self.max_windows)
        batch = [self._queue.popleft() for _ in range(n)]
        out = {}
        if batch:
            if self._kind == "device":
                blocks = self._run_device(batch)
            else:
                rows = self._run(batch)
                blocks = [rows[k, keep_lo - lo:keep_hi - lo].copy()
                          for k, (_, (lo, hi, keep_lo, keep_hi)) in enumerate(batch)]
            for (sid, _), y in zip(batch, blocks):
                out.setdefault(sid, []).append(y)
                self._streams[sid].pending.popleft()
                self._streams[sid].restored += 1
        for sid in [sid for sid, s in self._streams.items() if s.closed and not s.pending]:
            self._forget(sid)
        for sid in out:
            if sid in self._streams:
                self._trim(self._streams[sid])
        return out

    @property
    def streams(self):
        """Ids of the streams the pool still holds: open ones, and closed ones with windows left to restore."""
        return list(self._streams)

    @property
    def pending(self):
        """Windows due and not yet restored, of all streams."""
        return len(self._queue)

    @property
    def graph_count(self):
        """Restore graphs captured so far (one per bucket used)."""
        return len(self._graphs)

    # ------------------------------------------------------------------ bookkeeping
    def _open_stream(self, sid, what):
        s = self._streams.get(sid)
        if s is None:
            raise ValueError(f"stream_pool.{what}: stream {sid!r} is not open in this pool (never opened, or closed and "
                             "fully restored)")
        if s.closed:
            raise ValueError(f"stream_pool.{what}: stream {sid} is closed; its input has ended")
        return s

    def _check_device_block(self, sid, block):
        """Raises ValueError naming the stream for a CUDA block a device pool cannot take."""
        who = f"stream_pool.push: stream {sid}: a CUDA block"
        if torch.device(block.device) != torch.device(self._dev):
            raise ValueError(f"{who} is on {block.device}; this pool runs on {self._dev}")
        if block.dtype != torch.float32:
            raise ValueError(f"{who} has dtype {block.dtype}; CUDA blocks must be torch.float32")
        if len(block.shape) != 1:
            raise ValueError(f"{who} has shape {tuple(block.shape)}; blocks are 1-D")
        if block.stride(0) < 1:
            raise ValueError(f"{who} has element stride {block.stride(0)} (an expanded tensor); its samples must be "
                             "distinct elements (.contiguous() makes them so)")

    def _to_device(self):
        """Makes this a device pool; its streams, opened before any block was pushed, hold no input yet."""
        for sid, s in self._streams.items():
            assert s.n == 0 and not s.pending
            d = _DevStream(s.rate, self._dev, s.seed)
            d.closed = s.closed
            self._streams[sid] = d
        self._kind = "device"

    def _forget(self, sid):
        """Drops stream sid; a device buffer goes back to the allocator once the work queued on the engine's last
        stream, which follows every read of it, is done."""
        s = self._streams.pop(sid)
        if isinstance(s, _DevStream):
            s.release(self._eng._last_stream)

    def _schedule(self, sid, s, avail, ended):
        windows, s.pos = self._sched.due(s.pos, avail, ended)
        for w in windows:
            s.pending.append(w)
            self._queue.append((sid, w))
        self._trim(s)

    def _trim(self, s):
        """Drops input that no window of s will read again: before its oldest pending window, and before the lowest
        start a later window can have (a short flush window is widened by up to min_len samples before pos - ctx)."""
        keep = max(0, s.pos - self._sched.ctx - self._sched.min_len)
        if s.pending:
            keep = min(keep, s.pending[0][0])
        first, stop = resample.window(s.n, s.rate, keep, keep + 1)
        if stop > first:
            s.drop_before(first)

    def bucket(self, n):
        """The number of rows a step of n windows runs: the smallest bucket that holds them."""
        return next(b for b in self.buckets if b >= n)

    # ------------------------------------------------------------------ the launch
    def _buffers(self):
        """Input / output rows of the largest bucket, and one workspace that every bucket's graph shares (they replay
        one at a time on one stream); each bucket's graph reads and writes row prefixes of them."""
        if self._bufs is None:
            B, L, dev = self.max_windows, self.window_len, self._dev
            pin = (lambda t: t.pin_memory()) if self._cuda else (lambda t: t)
            ws = self._eng.graph_workspace_bytes(B, L, 1) if self.mode == 1 else self._eng.workspace_bytes(B, L)
            self._bufs = {"dev_in": torch.zeros((B, L), device=dev), "dev_out": torch.empty((B, L), device=dev),
                          "dev_lens": torch.empty(B, dtype=torch.int32, device=dev),
                          "ws": torch.empty(ws, dtype=torch.uint8, device=dev)}
            if self.mode == 2:                     # the windows' dropout keys, read by every bucket's graph
                self._bufs["dev_keys"] = torch.zeros((B, 2), dtype=torch.int64, device=dev)
            if self._kind != "device":             # a device pool stages nothing on the host
                self._bufs.update({"host_in": pin(torch.zeros((B, L))), "host_out": pin(torch.empty((B, L))),
                                   "host_lens": pin(torch.empty(B, dtype=torch.int32))})
        return self._bufs

    def _graph(self, B):
        """The restore graph of bucket B, captured on first use (once its lengths and keys are in place: the capture's
        warm-up runs read them)."""
        if B not in self._graphs:
            p = self._bufs
            keys = {"drop_keys": p["dev_keys"][:B]} if self.mode == 2 else {}
            self._graphs[B] = self._eng.make_graph(p["dev_in"][:B], p["dev_out"][:B], mode=self.mode,
                                                   lens=p["dev_lens"][:B], ws=p["ws"], **keys)
        return self._graphs[B]

    def _put_keys(self, batch, B):
        """Mode 2: fills rows [0, B) of the key buffer, row k with window k's (stream seed, window index), unused rows
        with (0, 0), from pinned memory with a stream-ordered copy (a fresh pinned buffer per step: the host does not
        wait for the previous step's copy)."""
        if self.mode != 2:
            return
        rows = np.zeros((B, 2), dtype=np.uint64)
        seen = {}
        for k, (sid, _) in enumerate(batch):
            s = self._streams[sid]
            seen[sid] = j = seen.get(sid, s.restored - 1) + 1
            rows[k] = (s.seed, j)
        keys = torch.from_numpy(rows.view(np.int64))
        self._bufs["dev_keys"][:B].copy_(keys.pin_memory() if self._cuda else keys, non_blocking=True)

    def _run(self, batch):
        """Restores the windows of batch [(sid, (lo, hi, keep_lo, keep_hi)), ...] and returns the output rows (host)."""
        p = self._buffers()
        n, B = len(batch), self.bucket(len(batch))
        streams = [self._streams[sid] for sid, _ in batch]
        lens = p["host_lens"]
        lens[:B] = self._sched.min_len             # unused rows: any valid length; their output is never read
        lens[:n] = torch.tensor([hi - lo for _, (lo, hi, _, _) in batch], dtype=torch.int32)
        if any(s.rate != resample.RATE for s in streams):
            x, lens_dev = self._eng.resample(*_stage([s.buf for s in streams], [s.rate for s in streams],
                                                     [(k, w[0], w[1]) for k, (_, w) in enumerate(batch)], self._dev,
                                                     extents=[(s.base, s.n) for s in streams]), self.window_len)
            p["dev_in"][:n].copy_(x)
            p["dev_lens"][n:B].copy_(lens[n:B], non_blocking=True)
            p["dev_lens"][:n].copy_(lens_dev)
        else:
            hin = p["host_in"].numpy()
            for k, (s, (_, (lo, hi, _, _))) in enumerate(zip(streams, batch)):
                hin[k, :hi - lo] = s.buf[lo - s.base:hi - s.base]
            p["dev_in"][:n].copy_(p["host_in"][:n], non_blocking=True)
            p["dev_lens"][:B].copy_(lens[:B], non_blocking=True)
        self._put_keys(batch, B)
        self._graph(B).replay()
        p["host_out"][:n].copy_(p["dev_out"][:n], non_blocking=True)
        if self._cuda:
            torch.cuda.current_stream().synchronize()
        return p["host_out"].numpy()

    def _run_device(self, batch):
        """Restores the windows of batch [(sid, (lo, hi, keep_lo, keep_hi)), ...] of a device pool and returns each
        window's kept samples as a new CUDA tensor: one vfx_resample_src launch gathers the rows from the streams'
        buffers, one graph replay restores them, one vfx_scatter_rows launch emits the kept spans.  Nothing waits."""
        p = self._buffers()
        n, B = len(batch), self.bucket(len(batch))
        streams = [self._streams[sid] for sid, _ in batch]
        gather, emit = stream_rows([(s.rate, s.base, s.n, w) for s, (_, w) in zip(streams, batch)])
        self._eng.resample_src([(s.buf, s.rate, y_first, y_len) for s, (_, y_first, y_len) in zip(streams, gather)],
                               self.window_len, y=p["dev_in"][:n], lens=p["dev_lens"][:n])
        p["dev_lens"][n:B].fill_(self._sched.min_len)  # unused rows: any valid length; their output is never read
        self._put_keys(batch, B)
        self._graph(B).replay()
        blocks = [torch.empty(m, device=self._dev) for _, m in emit]
        self._eng.scatter_rows(p["dev_out"][:n], [(y, 0, m, off) for y, (off, m) in zip(blocks, emit)])
        return blocks


class _ModelShim:
    """Stands in for `VoiceFixer._model` (the reference nn.Module): callers poke
    `.parameters()`, `.to()`, `.eval()`, `.train()` and `.vocoder` (test/streamlit.py:40-42)."""

    def __init__(self, owner):
        self._owner = owner
        self.vocoder = owner._vocoder

    def parameters(self):
        return iter([self._owner._engine.arena])

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def train(self, mode=True):
        return self


class Vocoder:
    """voicefixer/vocoder/base.py:10-77."""

    def __init__(self, sample_rate, _engine=None, precision=None):
        if sample_rate != 44100:           # vocoder/config.py:28-31
            raise RuntimeError("Error: Vocoder currently only support 44100 samplerate.")
        self.rate = sample_rate
        if _engine is None:
            voc = _load_vocoder_state()
            _check_cuda(False)
            from .weights import pack_vocoder
            _engine = Engine(packed=pack_vocoder(voc, precision or default_precision()), precision=precision)
            self._standalone = True
        self._engine = _engine

    def forward(self, mel, cuda=False):
        """non-normalised mel [B, 1, T, 128] -> [B, 1, (T + T%2 + 4)*441] (vocoder/base.py:42-56)."""
        assert mel.size()[-1] == 128
        _check_cuda(cuda)
        out = self._engine.vocoder(mel[:, 0], input_is_log=False)
        out = out[:, None, :]
        return out if cuda else out.cpu()

    __call__ = forward

    @torch.no_grad()
    def forward_many(self, mels, cuda=False):
        """Extension of the reference API: forward() on a list of [1, 1, T_i, 128] mels (tensors or arrays) of any lengths.
        Element i is bit-identical to forward(mels[i], cuda), on the device or the CPU as forward places it.  The mels run
        as ragged batches ordered by length (plan_vocoder_many, vfx_vocoder_ragged), each sized to the device memory that
        is free (Engine.max_batch_frames).  Bad input raises before anything is launched."""
        _check_cuda(cuda)
        eng = self._engine
        dev = f"cuda:{eng.device}"

        def max_items(T):
            return eng.max_batch_frames(T, extra_per_item=4 * (T * 128 + _gen_len(T)))   # + the batch's input and output

        outs = [None] * len(mels)
        for T_cap, idx in plan_vocoder_many(mels, "mel", max_items):
            x, lens = _pad_rows([torch.as_tensor(mels[i])[0, 0] for i in idx], T_cap, dev)
            y = eng.vocoder(x, lens=lens)
            for k, i in enumerate(idx):
                o = y[k:k + 1, None, :_gen_len(mels[i].shape[2])]
                outs[i] = o.clone() if cuda else o.cpu()
        return outs

    def oracle(self, fpath, out_path, cuda=False):
        """vocoder/base.py:58-77: wav file -> |STFT| -> Slaney mel -> normalise -> Generator -> file."""
        _check_cuda(cuda)
        wav = wavio.read_wave(fpath, self.rate)[..., 0]
        cond = oracle_conditions(wav)
        out = self._engine.vocoder_cond(torch.from_numpy(cond), scale=2.0 ** 15)
        wavio.save_wave(out[:, None, :].cpu().numpy(), out_path, sample_rate=self.rate)

    @torch.no_grad()
    def oracle_many(self, wavs, cuda=True, sample_rate=44100):
        """Extension of the reference API: oracle()'s computation on a list of 1-D float32 recordings of any lengths, each
        one whole sequence (no 30 s segments), front end included on the device (vfx_oracle).  Element i is a
        (1, (T_i + T_i % 2 + 4) * 441) float32 array, T_i = 1 + L_i // 441: the Generator output before oracle()'s x 2^15
        and int16 file write.  The recordings run as ragged batches ordered by length (plan_vocoder_many), each sized to
        the device memory that is free.  Bad input raises before anything is launched.

        sample_rate: the recordings' rate in Hz, one positive int or one per recording.  A recording at another rate than
        44100 is resampled on the device (vfx_resample) straight into the batch, bit-identical to oracle_many on
        wavio._resample(wavs[i], rate_i, 44100), the host resampler oracle() reads files with; L_i is then its length at
        44.1 kHz.  A call in which every rate is 44100 launches nothing for it.

        Device-resident recordings: when every item is a 1-D float32 CUDA tensor on the engine's device (any positive element
        stride), they are read in place and element i is a new (1, (T_i + T_i % 2 + 4) * 441) float32 CUDA tensor,
        bit-identical to torch.from_numpy of this call's element i on the items' host copies, at every sample_rate.  Each
        batch's rows come from one vfx_resample_src launch and go to the outputs with one vfx_scatter_rows launch, all on
        torch.cuda.current_stream(); the call returns without waiting for the GPU, and no sample crosses PCIe.  A list that
        mixes CUDA and host items, or a CUDA item on another device, of another dtype or not 1-D, raises ValueError
        before anything is launched.  A CUDA recording is not checked for all zeros (that would read it on the host): an
        all-zero one gives whatever the device front end makes of its zero peak."""
        _check_cuda(cuda)
        eng = self._engine
        dev = f"cuda:{eng.device}"
        wavs = list(wavs)
        on_dev = check_device_items(wavs, torch.device(dev), "oracle_many")
        items = list(wavs) if on_dev else [np.ascontiguousarray(w, dtype=np.float32) for w in wavs]
        rates = resample.rates(sample_rate, len(items), "oracle_many")

        def max_items(L):
            per_item = eng.oracle_workspace_bytes(2, L) - eng.oracle_workspace_bytes(1, L) + 4 * (L + _gen_len(1 + L // 441))
            return eng._fit(per_item + (0 if on_dev else _staging_extra(L, rates)), 64, 2 << 30)

        # the recordings' lengths at 44.1 kHz (a recording that is not 1-D is refused by plan_vocoder_many)
        lengths = [resample.out_len(a.shape[0], r) if len(a.shape) == 1 else 0 for a, r in zip(items, rates)]
        if on_dev:                     # allocated before planning, so that max_items sees the memory they take
            outs = [torch.empty((1, _gen_len(1 + n // 441)), device=dev) for n in lengths]
        else:
            outs = [None] * len(items)
        for L_cap, idx in plan_vocoder_many(items, "wav", max_items, pack_lengths=lengths):
            x, lens = _batch_input(eng, items, rates, [(i, 0, lengths[i]) for i in idx], L_cap, dev)
            y = eng.oracle(x, lens=lens)
            if on_dev:
                eng.scatter_rows(y, [(outs[i], off, n) for i, off, n in oracle_rows(idx, lengths)])
                continue
            y = y.cpu().numpy()
            for k, i in enumerate(idx):
                outs[i] = y[k:k + 1, :_gen_len(1 + lengths[i] // 441)].copy()
        return outs


def _staging_extra(L, rates):
    """Device bytes per item of L output samples that _batch_input adds for a call at these rates: none when they are all
    44100, else the staged input window (the largest resample.staging_bound) and the item's row of the resampler's table."""
    if all(r == resample.RATE for r in rates):
        return 0
    return 4 * max(resample.staging_bound(L, r) for r in set(rates)) + 64


def _pad_rows(rows, cap, dev):
    """Tensors [n_k, ...] as one float32 batch (B, cap, ...) on dev, row k holding rows[k] then zeros, and the n_k as an
    int32 (B,) tensor on dev.  Host rows are assembled on the host and uploaded in one copy; if any row is already on
    the GPU, the batch is assembled there, so no row goes through the host."""
    on_gpu = any(r.is_cuda for r in rows)
    x = torch.zeros((len(rows), cap) + tuple(rows[0].shape[1:]), device=dev if on_gpu else "cpu")
    for k, r in enumerate(rows):
        x[k, :r.shape[0]] = r
    return x.to(dev), torch.tensor([r.shape[0] for r in rows], dtype=torch.int32).to(dev)


def _batch_input(eng, items, rates, ranges, cap, dev):
    """(x (B, cap), lens (B,) int32), both on dev: row k of x holds range k of ranges [(item, a, b), ...] of the items'
    44.1 kHz streams, then zeros.  Items that are CUDA tensors (check_device_items) are read in place by one
    vfx_resample_src launch at every rate (Engine.resample_src).  Host items: if any of `rates` (one per item) is not
    44100, every row is resampled on the device from its own input window (_stage, Engine.resample); otherwise the
    samples are copied (_pad_rows), no resampler runs."""
    if isinstance(items[0], torch.Tensor):
        return eng.resample_src([(items[i], r, a, n) for i, r, a, n in resample_rows(ranges, rates)], cap)
    if any(r != resample.RATE for r in rates):
        return eng.resample(*_stage(items, rates, ranges, dev), cap)
    return _pad_rows([torch.from_numpy(items[i][a:b]) for i, a, b in ranges], cap, dev)


def _drop_masks(drop_masks_fn, B, T):
    """Mode 2's dropout keep-masks for B segments of up to T frames: uint8 (2, B, T, 512) from drop_masks_fn(B, T), or
    None for drop_masks_fn=False.  The reference's mode 2 is module.train(): both Dropout(0.5) of the denoiser draw from
    torch's global RNG (base.py:114-115, restorer/model.py:76,90).  Without drop_masks_fn, same distribution here (from
    torch's CPU generator, so torch.manual_seed controls it); the RNG *stream* differs, which no reference test pins."""
    if drop_masks_fn is False:
        return None
    masks = drop_masks_fn(B, T) if drop_masks_fn else (torch.rand(2, B, T, 512) >= 0.5)
    masks = torch.as_tensor(masks).to(torch.uint8)
    if tuple(masks.shape) != (2, B, T, 512):
        raise ValueError(f"dropout masks must have shape (2, {B}, {T}, 512), got {tuple(masks.shape)}")
    return masks


def _upload_masks(masks, dev):
    """Mode 2's keep-masks on dev, for a device-resident call: a host tensor goes through pinned memory with a
    stream-ordered copy, so the host does not wait for the device."""
    if masks is None or masks.is_cuda:
        return masks
    return masks.pin_memory().to(dev, non_blocking=True)


def check_dropout_seed(s, who):
    """s as an int if it is a valid seed of mode 2's seeded dropout (an integer in [0, 2^64), not a bool); else raises
    ValueError `<who> has dropout_seed ...`."""
    if isinstance(s, (bool, np.bool_)) or not isinstance(s, numbers.Integral) or not 0 <= int(s) < 1 << 64:
        raise ValueError(f"{who} has dropout_seed {s!r}; a dropout seed is an integer in [0, 2^64)")
    return int(s)


def dropout_seeds(dropout_seed, mode, drop_masks_fn, n, what):
    """restore_many's dropout_seed as one seed per recording: one int for all n recordings, or a list / tuple / array of
    n of them (sample_rate's convention); None for dropout_seed=None.  Raises ValueError, naming the recording, for a bad
    seed or a wrong count, and for a seed given in another mode than 2 or together with a drop_masks_fn."""
    if dropout_seed is None:
        return None
    check_seeded(mode, drop_masks_fn, what)
    if isinstance(dropout_seed, (list, tuple, np.ndarray)):
        ss = list(np.asarray(dropout_seed, dtype=object).reshape(-1)) if isinstance(dropout_seed, np.ndarray) \
            else list(dropout_seed)
        if len(ss) != n:
            raise ValueError(f"{what}: dropout_seed has {len(ss)} entries for {n} recordings; give one seed, or one per "
                             "recording")
    else:
        ss = [dropout_seed] * n
    return [check_dropout_seed(s, f"{what}: recording {i}") for i, s in enumerate(ss)]


def check_seeded(mode, drop_masks_fn, what):
    """Refuses a dropout seed outside mode 2, or next to a drop_masks_fn other than None (two sources of the masks)."""
    if mode != 2:
        raise ValueError(f"{what}: dropout_seed is mode 2's dropout; mode is {mode!r}")
    if drop_masks_fn is not None:
        raise ValueError(f"{what}: give dropout_seed or drop_masks_fn, not both")


def stream_dropout_seed(mode, dropout_seed, who):
    """The dropout seed of one stream (restore_stream, StreamPool.open): dropout_seed checked (check_seeded,
    check_dropout_seed), or in mode 2 without one a 64-bit seed drawn from torch's CPU generator, so that
    torch.manual_seed controls it as it controls restore_inmem's default masks; None outside mode 2."""
    if dropout_seed is not None:
        check_seeded(mode, None, who)
        return check_dropout_seed(dropout_seed, who)
    if mode != 2:
        return None
    lo, hi = (int(v) for v in torch.randint(0, 1 << 32, (2,), dtype=torch.int64))
    return hi << 32 | lo


def prefilter_bytes(eng, L):
    """Device bytes per item that mode 1's pre-filter adds alongside a restore of items of (at most) L samples: its
    workspace's growth per item and its (L,) float32 output row."""
    return eng.hf_cut_workspace_bytes(2, L) - eng.hf_cut_workspace_bytes(1, L) + 4 * L


def check_channels(channels, who):
    """Refuses a channels argument other than "mix" (the mono mix, as the reference reads files) or "keep" (every
    channel restored on its own)."""
    if not isinstance(channels, str) or channels not in ("mix", "keep"):
        raise ValueError(f'{who}: channels is {channels!r}; it must be "mix" or "keep"')


def drop_key_rows(segs, seeds, bases=None):
    """The seeded dropout keys of a batch (vfx_drop_key): segs = [(recording, a, b), ...] (plan_many's segments, a the
    first sample of a 30 s segment), seeds one per recording -> uint64 (B, 2) rows (seed of the recording,
    base of the recording + a // SEG_LENGTH): segment k of a recording draws its masks from stream base + k of its seed,
    whatever batch it runs in.  bases: one stream base per recording, 0 for each without it (restore_files gives
    channel c of a file the base c << 32, so that the channels of one file never share masks)."""
    return np.array([(seeds[i], (int(bases[i]) if bases is not None else 0) + a // SEG_LENGTH) for i, a, _ in segs],
                    dtype=np.uint64).reshape(-1, 2)


def _upload_keys(rows, dev):
    """drop_key_rows on dev as the int64 (B, 2) tensor Engine.restore(drop_keys=) takes: 16 bytes per segment, from pinned
    memory with a stream-ordered copy, so the host does not wait for the device."""
    return torch.from_numpy(rows.view(np.int64)).pin_memory().to(dev, non_blocking=True)


def _stage(items, rates, segs, dev, extents=None):
    """The device resampler's input for output ranges segs = [(recording, a, b), ...] of the 44.1 kHz streams: each
    range's input window (resample.window), concatenated on the host and uploaded as one staging buffer, and the items
    of Engine.resample.  extents (live streams, whose older input is dropped): one (base, n) per item, items[i] then
    holding input samples [base, base + len(items[i])) of a recording of which n samples have arrived so far; without
    it each item is a whole recording."""
    windows, table, off = [], [], 0
    for i, a, b in segs:
        base, n = extents[i] if extents is not None else (0, items[i].shape[0])
        first, stop = resample.window(n, rates[i], a, b)
        windows.append(items[i][first - base:stop - base])
        table.append((rates[i], n, off, first, stop - first, a, b - a))
        off += stop - first
    return torch.from_numpy(np.concatenate(windows)).to(dev), table


def _many_inputs(eng, wavs, sample_rate, mode, drop_masks_fn, dropout_seed, what):
    """The recordings of restore_many / analysis_many, checked before anything is launched: (on_dev, items, rates, seeds,
    lengths), items being the CUDA tensors themselves (check_device_items) or contiguous float32 arrays, and lengths the
    recordings' lengths at 44.1 kHz."""
    wavs = list(wavs)
    on_dev = check_device_items(wavs, torch.device(f"cuda:{eng.device}"), what)
    items = list(wavs) if on_dev else []
    for i, w in ([] if on_dev else enumerate(wavs)):
        a = np.ascontiguousarray(w, dtype=np.float32)
        if a.ndim != 1:
            raise ValueError(f"{what}: recording {i} has shape {a.shape}; the list takes 1-D arrays")
        items.append(a)
    rates = resample.rates(sample_rate, len(items), what)
    seeds = dropout_seeds(dropout_seed, mode, drop_masks_fn, len(items), what)
    lengths = [resample.out_len(a.shape[0], r) for a, r in zip(items, rates)]
    return on_dev, items, rates, seeds, lengths


def _segment_batches(eng, items, rates, lengths, mode, drop_masks_fn, seeds, on_dev, what, sizing="restore",
                     bases=None):
    """The batch loop of restore_many and analysis_many: plan_many's batches as (segs, x, lens, masks, keys): the rows
    (mode 1: after the ragged pre-filter) and lengths of the batch's segments on the device, and mode 2's dropout masks
    or seeded keys (None otherwise).  Each batch is sized to the device memory that is free (Engine.max_batch) for
    `sizing`: "restore", a restore; "analysis", analysis_ragged and the batch's two mel tensors; "hook", the same calls
    sized as a restore, so that the memory the engine's own vocoder would take is left to the caller's vocoder.
    bases: the recordings' seeded dropout stream bases (drop_key_rows), or None."""
    dev = f"cuda:{eng.device}"

    def max_items(L_cap):
        extra = 0 if on_dev else _staging_extra(L_cap, rates)
        if mode == 1:     # the pre-filter's workspace and its (B, L_cap) output live alongside the restore
            extra += prefilter_bytes(eng, L_cap)
        if sizing != "restore":      # the log mel and the denoised mel of the batch
            extra += 2 * 4 * 128 * (1 + L_cap // 441)
        return eng.max_batch(L_cap, extra_per_item=extra, analysis=sizing == "analysis")

    for L_cap, segs in plan_many(lengths, mode, max_items, what):
        x, lens = _batch_input(eng, items, rates, segs, L_cap, dev)
        if mode == 1:
            x, _, lens = eng.hf_cut(x, lens=lens)
        masks = keys = None
        if seeds is not None:
            keys = _upload_keys(drop_key_rows(segs, seeds, bases), dev)
        elif mode == 2:
            masks = _drop_masks(drop_masks_fn, len(segs), 1 + L_cap // 441)
            if on_dev:
                masks = _upload_masks(masks, dev)
        yield segs, x, lens, masks, keys


def _denoised(eng, x, lens, mode, masks, keys):
    """The denoised mels (B, T_cap, 128) of a batch of _segment_batches: restore_inmem's 10 ** clip(mel_log, max=5) on
    analysis_ragged's log mels, row b's first 1 + lens[b] // 441 frames being segment b's."""
    mel_log = eng.analysis_ragged(x, lens, mode=2 if mode == 2 else 0, drop_masks=masks, drop_keys=keys)
    return 10 ** torch.clip(mel_log, max=5)


def _seg_frames(a, b, mode):
    """Mel frames of the segment [a, b) of a recording in `mode`."""
    return 1 + _net_len(b - a, mode) // 441


def oracle_conditions(wav):
    """Host front end of Vocoder.oracle (vocoder/base.py:61-73; numpy in the reference too):
    peak-normalise, |STFT| (2048/441/Hann/center, librosa-0.10 zero padding), Slaney-normalised
    HTK mel (librosa.filters.mel defaults), dB - 20, normalise, pad -> (1, Tc, 128) channels-last.  The window is
    float64, as librosa's get_window returns it, so the windowed frames are float64 like librosa.stft's."""
    wav = np.asarray(wav, dtype=np.float32)
    wav = wav / np.max(np.abs(wav))
    n_fft, hop = 2048, 441
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)
    x = np.pad(wav, (n_fft // 2, n_fft // 2), mode="constant")
    nfr = 1 + (len(x) - n_fft) // hop
    idx = np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]
    stft = np.abs(np.fft.rfft(x[idx] * win[None, :], axis=1).astype(np.complex64))      # (T, 1025)
    mel = stft @ wavio.slaney_htk_mel_basis().T                                         # (T, 128)
    min_level = np.exp(-100 / 20 * np.log(10))
    S = 20 * np.log10(np.maximum(min_level, np.abs(mel))) - 20
    S = np.clip(8.0 * ((S + 115.0) / 115.0) - 4.0, -4.0, 4.0).astype(np.float32)
    pad_tail = S.shape[0] % 2 + 4
    return np.concatenate([S, np.full((pad_tail, 128), -4.0, np.float32)], 0)[None]


class VoiceFixer:
    """voicefixer/base.py:10-146."""

    def __init__(self, precision=None):
        self.analysis_module_ckpt = os.path.join(os.path.expanduser("~"), ANALYSIS_CKPT)
        voc = _load_vocoder_state()        # the reference builds Vocoder first (restorer/model.py:180)
        if not os.path.exists(self.analysis_module_ckpt):
            raise RuntimeError(_ERR0)
        ana = torch.load(self.analysis_module_ckpt, map_location="cpu")
        _check_cuda(False)
        self._engine = Engine(ana, voc, precision=precision)
        self._vocoder = Vocoder(44100, _engine=self._engine)
        self._model = _ModelShim(self)

    @classmethod
    def from_engine(cls, engine):
        """The same API object around an engine whose weights are already on the device (e.g. an arena received through
        parallel.broadcast_arena on a non-zero rank: no checkpoint files are read)."""
        self = cls.__new__(cls)
        self.analysis_module_ckpt = os.path.join(os.path.expanduser("~"), ANALYSIS_CKPT)
        self._engine = engine
        self._vocoder = Vocoder(44100, _engine=engine)
        self._model = _ModelShim(self)
        return self

    # -- helpers kept from the reference API
    def _load_wav(self, path, sample_rate, threshold=0.95):
        return wavio.load_mono(path, sample_rate)                       # base.py:47-49

    def _trim_center(self, est, ref):                                   # base.py:63-76
        diff = abs(est.shape[-1] - ref.shape[-1])
        if est.shape[-1] == ref.shape[-1]:
            return est, ref
        if est.shape[-1] > ref.shape[-1]:
            min_len = min(est.shape[-1], ref.shape[-1])
            est = est[..., int(diff // 2): -int(diff // 2)]
            return est[..., :min_len], ref[..., :min_len]
        min_len = min(est.shape[-1], ref.shape[-1])
        ref = ref[..., int(diff // 2): -int(diff // 2)]
        return est[..., :min_len], ref[..., :min_len]

    def _vocode_segment(self, f, m, n, cuda):
        """One segment through the vocoder hook as restore_inmem runs it (base.py:126-133): f gets the segment's denoised
        mel m [1, 1, T, 128] (on the CPU unless cuda), its output comes to the engine's device as float32, is divided by
        its peak with the reference's warning when that exceeds 1, and is cut by _trim_center to the segment's n
        samples.  Returns a (1, n) tensor (shorter if f's output is)."""
        y = torch.as_tensor(f(m if cuda else m.cpu())).to(f"cuda:{self._engine.device}").float()
        if torch.max(torch.abs(y)) > 1.0:
            y = y / torch.max(torch.abs(y))
            print("Warning: Exceed energy limit,", "input")
        return self._trim_center(y[:, 0], torch.empty(1, n, device="meta"))[0]   # ref: only its length is read

    def remove_higher_frequency(self, wav, ratio=0.95):                 # base.py:87-104
        out, _ = self._engine.hf_cut(torch.from_numpy(np.ascontiguousarray(wav, dtype=np.float32))[None], ratio)
        return out[0].cpu().numpy()

    @torch.no_grad()
    def restore_inmem(self, wav_10k, cuda=False, mode=0, your_vocoder_func=None, drop_masks_fn=None, dropout_seed=None):
        """np (L,) float32 -> np (1, L) float32 (base.py:106-139).  The 30 s segments are
        independent (SURVEY D4), so all full segments run as one batch and the ragged tail as a
        second one; results are concatenated in order.

        drop_masks_fn (extension, mode 2 only): None = random Bernoulli(0.5) keep-masks like the reference's
        train-mode dropout; a callable (B, T) -> uint8 [2, B, T, 512] supplies them explicitly; False = no
        dropout (deterministic train-mode BN only).

        dropout_seed (extension, mode 2 only, with drop_masks_fn=None): an int in [0, 2^64).  The masks are then
        computed on the GPU from the seed (Philox4x32-10, DESIGN.md §3): segment k (the one starting at sample
        k * SEG_LENGTH) uses philox.seeded_masks(dropout_seed, k, T_k), and no mask is drawn on the host or uploaded.
        The result depends on the recording and the seed only; restore_many gives the same bits."""
        _check_cuda(cuda)
        if mode not in (0, 1, 2):
            raise ValueError("mode must be 0, 1 or 2")
        if dropout_seed is not None:
            check_seeded(mode, drop_masks_fn, "restore_inmem")
            dropout_seed = check_dropout_seed(dropout_seed, "restore_inmem")
        wav = np.ascontiguousarray(wav_10k, dtype=np.float32)
        bounds = segment_bounds(wav.shape[0])
        segs = [wav[a:b] for a, b in bounds]
        eng = self._engine
        dev = f"cuda:{eng.device}"
        groups = {}
        for i, s in enumerate(segs):
            groups.setdefault(len(s), []).append(i)
        outs = [None] * len(segs)
        for L, all_idxs in groups.items():
            if mode == 2 and 1 + _net_len(L, mode) // 441 <= 64:
                # torch.nn.functional.batch_norm in the reference (train mode, 1x1 UNet centre)
                raise ValueError(_MODE2_MSG)
            # the reference walks the segments one at a time in constant memory; here they are batched, in chunks
            # sized to the device memory that is free right now (a 100-minute recording does not fit one launch sequence)
            chunk = eng.max_batch(L)
            for c0 in range(0, len(all_idxs), chunk):
                idxs = all_idxs[c0:c0 + chunk]
                x = torch.from_numpy(np.stack([segs[i] for i in idxs])).to(dev)
                if mode == 1:
                    x, _ = eng.hf_cut(x)                                 # shorter: _net_len(L, 1)
                masks = keys = None
                if dropout_seed is not None:
                    keys = _upload_keys(drop_key_rows([(0,) + bounds[i] for i in idxs], [dropout_seed]), dev)
                elif mode == 2:
                    masks = _drop_masks(drop_masks_fn, x.shape[0], 1 + x.shape[1] // 441)
                if your_vocoder_func is None:
                    y = eng.restore(x, mode=2 if mode == 2 else 0, drop_masks=masks, drop_keys=keys)
                else:                                                    # base.py:126-129
                    mel = eng.frontend(x)
                    mel_log = eng.analysis(mel, mode=2 if mode == 2 else 0, drop_masks=masks, drop_keys=keys)
                    denoised = (10 ** torch.clip(mel_log, max=5))[:, None]
                    y = torch.cat([self._vocode_segment(your_vocoder_func, denoised[k:k + 1], x.shape[1], cuda)
                                   for k in range(denoised.shape[0])], 0)
                for k, i in enumerate(idxs):
                    outs[i] = y[k]
        out = torch.cat(outs, -1)[None]
        return out.cpu().numpy()

    @torch.no_grad()
    def restore_many(self, wavs, cuda=True, mode=0, drop_masks_fn=None, sample_rate=44100, dropout_seed=None,
                     your_vocoder_func=None, _stream_base=None):
        """Extension of the reference API: restores a list of 1-D recordings of any lengths, in any mode, and returns a
        list of (1, L_i') arrays, element i what restore_inmem(wavs[i], cuda=True, mode=mode) returns -- bit-identical in
        modes 0 and 1 and in mode 2 with drop_masks_fn=False; in mode 2 with dropout, the same distribution.

        The recordings are cut into 30 s segments as restore_inmem cuts them, and all segments of all recordings run as
        ragged batches ordered by length (plan_many), each batch sized to the device memory that is free.  Mode 1 runs the
        ragged pre-filter and then a ragged restore per batch; mode 2 a ragged restore with train-mode statistics per item.
        drop_masks_fn (mode 2): None = Bernoulli(0.5) keep-masks from torch's CPU generator, as restore_inmem draws them;
        a callable (B, T_cap) -> uint8 (2, B, T_cap, 512) supplies them for each launch (item b of a batch reads
        [:, b, :T_b]); False = no dropout.  Bad input raises ValueError before anything is launched.

        your_vocoder_func: restore_inmem's vocoder hook.  Each batch then runs the analysis alone (vfx_analysis_ragged) and
        the hook is called once per segment, as restore_inmem calls it: with the segment's denoised mel [1, 1, T, 128]
        (analysis_many's; on the CPU unless cuda), its output divided by its peak with the reference's warning when that
        exceeds 1, and cut by _trim_center to the segment's output length; the pieces are joined in segment order.  The
        segments are taken in the plan's order (longest first, across recordings), not recording by recording.  Element i
        equals restore_inmem(wavs[i], cuda, mode, your_vocoder_func=f) bit for bit when f's output depends on its input
        only (modes 0 and 1, and mode 2 with dropout_seed or drop_masks_fn=False).  The batches are sized as a restore's,
        so the hook runs in about the memory the engine's own vocoder would have taken (besides the workspace the engine
        keeps between calls).  The hook's output is checked on the host (its peak) and the pieces are joined with
        torch.cat, so this form waits for the GPU once per segment, whatever the input.

        sample_rate: the recordings' rate in Hz, one positive int or one per recording (a bad one raises ValueError naming
        the recording).  Recordings at another rate than 44100 are resampled on the device (vfx_resample): each segment
        of the 44.1 kHz stream is computed from its own window of input samples, uploaded alone, straight into the
        batch.  Element i is then bit-identical to restore_many on wavio._resample(wavs[i], rate_i, 44100), the host
        resampler VoiceFixer.restore() reads files with; the plan is the same, so mode 2's default masks are drawn at the
        same points.  A call in which every rate is 44100 launches nothing for it.

        Device-resident recordings: when every item is a 1-D float32 CUDA tensor on the engine's device (any positive element
        stride, e.g. x[:, c] of an interleaved (L, C) tensor), they are read in place, never written, and element i is a
        new (1, L_i') float32 CUDA tensor, bit-identical to torch.from_numpy of this call's element i on the items' host
        copies (modes 0 and 1, and mode 2 with drop_masks_fn=False, at every sample_rate; mode 2's random masks have the
        same distribution).  Each batch's rows come from one vfx_resample_src launch.  Without a hook, its restored
        segments go to their offsets in the outputs with one vfx_scatter_rows launch, all on torch.cuda.current_stream();
        the call returns without waiting for the GPU, and no sample crosses PCIe.  With a hook, the outputs are the
        hook's pieces joined on the device, and the call waits as the hook paragraph above says.  A list that mixes CUDA
        and host items, or a CUDA item on another device, of another dtype or not 1-D, raises ValueError before anything
        is launched.

        dropout_seed (mode 2, with drop_masks_fn=None): one int in [0, 2^64) for every recording, or a list / tuple /
        array with one per recording; a bad seed or count raises ValueError naming the recording before anything is
        launched.  Segment k of recording i then draws its masks on the GPU from (seed_i, k) (Philox4x32-10, DESIGN.md
        §3): no mask is drawn on the host or exists anywhere, and each batch uploads only its 16-byte keys (from pinned
        memory, without a host wait).  Element i depends on recording i and its seed only: it is bit-identical to
        restore_inmem(wavs[i], cuda=True, mode=2, dropout_seed=seed_i) and to restore_many([wavs[i]], mode=2,
        dropout_seed=seed_i)[0], whatever the other recordings, their order, the batch plan, host or CUDA input, or
        sample_rate.  Recordings given the same seed share their masks segment by segment; distinct seeds avoid that.

        Channels: the list takes 1-D recordings.  The channels of a multichannel recording x (L, C) are restored as the
        columns [x[:, c] for c in range(C)]; for a CUDA tensor those are strided views, read in place without a copy.
        _stream_base (restore_files' channels): one seeded dropout stream base per recording (drop_key_rows)."""
        _check_cuda(cuda)
        eng = self._engine
        dev = f"cuda:{eng.device}"
        on_dev, items, rates, seeds, lengths = _many_inputs(eng, wavs, sample_rate, mode, drop_masks_fn, dropout_seed,
                                                            "restore_many")
        batches = _segment_batches(eng, items, rates, lengths, mode, drop_masks_fn, seeds, on_dev, "restore_many",
                                   sizing="restore" if your_vocoder_func is None else "hook", bases=_stream_base)
        if your_vocoder_func is not None:
            pieces = {}                                                  # (recording, start) -> vocoded segment
            for segs, x, lens, masks, keys in batches:
                den = _denoised(eng, x, lens, mode, masks, keys)
                for k, (i, a, b) in enumerate(segs):
                    pieces[(i, a)] = self._vocode_segment(your_vocoder_func, den[k:k + 1, None, :_seg_frames(a, b, mode)],
                                                          _net_len(b - a, mode), cuda)
            outs = [torch.cat([pieces[(i, a)] for a, _ in segment_bounds(n)], -1) for i, n in enumerate(lengths)]
            return outs if on_dev else [o.cpu().numpy() for o in outs]
        if on_dev:                     # allocated before planning, so that max_items sees the memory they take
            outs = [torch.empty((1, restore_out_len(n, mode)), device=dev) for n in lengths]
        pieces = {}                                                      # (recording, start) -> restored segment
        for segs, x, lens, masks, keys in batches:
            y = eng.restore(x, mode=2 if mode == 2 else 0, drop_masks=masks, lens=lens, drop_keys=keys)
            if on_dev:
                eng.scatter_rows(y, [(outs[i], off, n) for i, off, n in restore_rows(segs, mode)])
                continue
            y = y.cpu().numpy()
            for k, (i, a, b) in enumerate(segs):
                pieces[(i, a)] = y[k, :_net_len(b - a, mode)]
        if on_dev:
            return outs
        return [np.concatenate([pieces[(i, a)] for a, _ in segment_bounds(n)])[None] for i, n in enumerate(lengths)]

    @torch.no_grad()
    def analysis_many(self, wavs, cuda=True, mode=0, drop_masks_fn=None, sample_rate=44100, dropout_seed=None):
        """Extension of the reference API: the restorer alone on a list of 1-D recordings of any lengths.  Element i is a
        list with one entry per 30 s segment of recording i, in order: the (1, 1, T_k, 128) float32 denoised mel that
        restore_inmem(wavs[i], mode=mode, your_vocoder_func=f) hands f for that segment, 10 ** clip(mel_log, max=5),
        linear and not normalised, T_k = 1 + L_k' // 441 for the segment's L_k' samples (after the pre-filter in mode 1).
        Adjacent segments are analysed apart and each has its own edge frame, so they are not joined.

        Inputs, modes, drop_masks_fn, sample_rate, dropout_seed and refusals are restore_many's, and so is the plan: the
        segments of all recordings run as ragged batches ordered by length, each one vfx_analysis_ragged call (after the
        ragged pre-filter in mode 1) sized to the device memory that is free.  Bit-identical to what restore_inmem hands
        the hook in modes 0 and 1, and in mode 2 with dropout_seed or drop_masks_fn=False, whatever the batch plan.

        Host recordings give numpy arrays.  CUDA recordings (restore_many's device-resident form) are read in place and
        give new CUDA tensors, bit-identical to the host call's, filled by one vfx_scatter_rows launch per batch: the call
        queues everything on torch.cuda.current_stream() and returns without waiting for the GPU."""
        _check_cuda(cuda)
        eng = self._engine
        dev = f"cuda:{eng.device}"
        on_dev, items, rates, seeds, lengths = _many_inputs(eng, wavs, sample_rate, mode, drop_masks_fn, dropout_seed,
                                                            "analysis_many")
        frames = [[_seg_frames(a, b, mode) for a, b in segment_bounds(n)] for n in lengths]
        if on_dev:                     # allocated before planning, so that max_items sees the memory they take
            outs = [[torch.empty((1, 1, T, 128), device=dev) for T in fr] for fr in frames]
        else:
            outs = [[None] * len(fr) for fr in frames]
        for segs, x, lens, masks, keys in _segment_batches(eng, items, rates, lengths, mode, drop_masks_fn, seeds, on_dev,
                                                           "analysis_many", sizing="analysis"):
            den = _denoised(eng, x, lens, mode, masks, keys)
            if on_dev:
                eng.scatter_rows(den.view(den.shape[0], -1),
                                 [(outs[i][a // SEG_LENGTH], 0, 128 * _seg_frames(a, b, mode)) for i, a, b in segs])
                continue
            den = den.cpu().numpy()
            for k, (i, a, b) in enumerate(segs):
                outs[i][a // SEG_LENGTH] = den[k:k + 1, None, :_seg_frames(a, b, mode)].copy()
        return outs

    # ------------------------------------------------------------------ batch entry point (extension)
    def pinned_empty(self, shape):
        """numpy float32 array backed by pinned (page-locked) host memory: restore_batch copies such arrays to and from
        the GPU without an extra staging copy."""
        t = torch.empty(tuple(shape), dtype=torch.float32).pin_memory()
        a = t.numpy()
        self._pinned_keep = getattr(self, "_pinned_keep", [])
        self._pinned_keep.append(t)
        return a

    @torch.no_grad()
    def restore_batch(self, wavs, cuda=True, mode=0, out=None):
        """Extension of the reference API for many utterances (the reference restores one array per call,
        voicefixer/base.py:106): wavs np (B, L) float32, L <= 30 s -> np (B, L) float32, every row exactly what
        restore_inmem(row, mode) returns (mode 0 here; modes 1 / 2 go through restore_inmem).  The launch sequence of a
        shape is captured into a CUDA graph on first use and replayed afterwards; host buffers move through pinned
        staging (directly, when `wavs` / `out` are pinned: see pinned_empty).  Without `out`, the result is a view of an
        internal pinned buffer that the next call with the same shape overwrites.

        wavs may also be a list of 1-D arrays of different lengths (1025 samples .. 30 s each): they run as ONE ragged
        batch (vfx_restore_ragged) and the result is a list of new arrays, item i exactly what
        restore_batch(wavs[i][None])[0] returns.  The graph is keyed by (B, L_cap), L_cap = the longest item rounded up
        to a whole second, so later lists of as many items under the same cap replay it.  `out` is not used then."""
        _check_cuda(cuda)
        if mode != 0:
            raise ValueError("restore_batch runs mode 0; use restore_inmem for modes 1 and 2")
        if isinstance(wavs, (list, tuple)):
            return self._restore_ragged(wavs)
        x = np.ascontiguousarray(wavs, dtype=np.float32)
        if x.ndim != 2 or x.shape[1] > SEG_LENGTH:
            raise ValueError("restore_batch takes (B, L) with L <= 30 s (longer inputs: restore_inmem segments them)")
        eng = self._engine
        dev = f"cuda:{eng.device}"
        key = tuple(x.shape)

        def make():
            p = {"dev_in": torch.empty(key, device=dev), "dev_out": torch.empty(key, device=dev),
                 "host_in": torch.empty(key).pin_memory(), "host_out": torch.empty(key).pin_memory()}
            p["dev_in"].copy_(torch.from_numpy(x))
            p["graph"] = eng.make_graph(p["dev_in"], p["dev_out"], mode=0)
            return p

        p = self._graph_plan(key, make)
        src = torch.from_numpy(x)
        if not src.is_pinned():
            p["host_in"].copy_(src)
            src = p["host_in"]
        p["dev_in"].copy_(src, non_blocking=True)
        p["graph"].replay()
        dst = p["host_out"]
        if out is not None:
            o = torch.from_numpy(out)
            if o.is_pinned() and o.is_contiguous() and tuple(o.shape) == key and o.dtype == torch.float32:
                dst = o
        dst.copy_(p["dev_out"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        if out is not None and dst is p["host_out"]:
            out[...] = dst.numpy()
            return out
        return out if out is not None else dst.numpy()

    def _graph_plan(self, key, make):
        """The restore_batch plan for key (buffers and the CUDA graph that reads them), made by make() on first use.  Each
        graph owns its workspace, so at most four shapes are kept, the oldest dropped first."""
        plans = self.__dict__.setdefault("_batch_plans", {})
        if key not in plans:
            if len(plans) >= 4:
                plans.pop(next(iter(plans)))
            plans[key] = make()
        return plans[key]

    def _restore_ragged(self, wavs):
        items, lens, L_cap = ragged_plan(wavs)
        B = len(items)
        eng = self._engine
        dev = f"cuda:{eng.device}"
        p = self._graph_plan(("ragged", B, L_cap), lambda: {
            "dev_in": torch.zeros((B, L_cap), device=dev), "dev_out": torch.empty((B, L_cap), device=dev),
            "dev_lens": torch.empty(B, dtype=torch.int32, device=dev),
            "host_in": torch.zeros((B, L_cap)).pin_memory(), "host_out": torch.empty((B, L_cap)).pin_memory(),
            "host_lens": torch.empty(B, dtype=torch.int32).pin_memory()})
        hin = p["host_in"].numpy()
        for i, a in enumerate(items):            # samples past an item's length are never read: no need to clear them
            hin[i, :lens[i]] = a
        p["host_lens"].copy_(torch.tensor(lens, dtype=torch.int32))
        p["dev_in"].copy_(p["host_in"], non_blocking=True)
        p["dev_lens"].copy_(p["host_lens"], non_blocking=True)
        if "graph" not in p:                     # captured once the lengths are staged: its warm-up runs read them
            p["graph"] = eng.make_graph(p["dev_in"], p["dev_out"], mode=0, lens=p["dev_lens"])
        p["graph"].replay()
        p["host_out"].copy_(p["dev_out"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        hout = p["host_out"].numpy()
        return [hout[i, :lens[i]].copy() for i in range(B)]

    # ------------------------------------------------------------------ streaming entry point (extension, SURVEY 8f-3)
    @torch.no_grad()
    def restore_stream(self, blocks, chunk_seconds=2.0, context_seconds=1.0, cuda=True, mode=0, dropout_seed=None):
        """Low-latency form of restore_inmem for audio that arrives in blocks: a generator that takes an iterable of 1-D
        float32 blocks of any sizes (44.1 kHz mono) and yields restored blocks as soon as they can be computed.

        The reference has no streaming path: it cuts a recording into hard 30 s segments whose BiGRU and UNet see the whole
        segment (voicefixer/base.py:116-138).  Here every emitted chunk of `chunk_seconds` is restored inside a window that
        also holds `context_seconds` of already-received audio on the left and of look-ahead on the right
        (window = [pos - ctx, pos + chunk + ctx), clipped to the stream), and only the chunk itself is kept.  The
        algorithmic latency is chunk + context seconds of audio plus one B = 1 launch sequence (see bench.py
        `workloads.stream`).  With chunk_seconds = 30 and context_seconds = 0 the windows ARE the reference's segments
        and the concatenated output equals restore_inmem's exactly; smaller windows trade fidelity to whole-segment
        processing for latency (how much depends on the trained weights' context dependence; it cannot be pinned with
        the synthetic checkpoints available offline, DESIGN.md 7).  The total output length equals the input length in
        modes 0 and 2.

        mode: restore_inmem's mode, run per window as its eager B = 1 calls.  Mode 1 runs the pre-filter and then the
        restore on each window and emits only the samples the pre-filter keeps (StreamSchedule): with context_seconds
        of at least 511 samples only the stream's last <= 511 samples are lost, as restore_inmem loses them of a
        recording shorter than 30 s; with no context each chunk loses chunk % 512, as restore_inmem's segments do.
        Mode 2 restores each window with train-mode statistics and seeded dropout: window k (counting from 0) draws its
        masks from (dropout_seed, k) on the GPU, so with 30 s chunks and no context the output is bit-identical to
        restore_inmem(mode=2, dropout_seed=dropout_seed).  dropout_seed: an int in [0, 2^64), mode 2 only; without one,
        one is drawn from torch's CPU generator when the generator starts (torch.manual_seed controls it).  The shortest
        window a mode restores (StreamSchedule.min_len) is 1025 samples in mode 0, 1536 in mode 1 and 28 224 (more than
        64 frames) in mode 2: chunk_seconds + context_seconds must reach it, and so must the whole stream."""
        _check_cuda(cuda)
        chunk = int(round(chunk_seconds * 44100))
        ctx = int(round(context_seconds * 44100))
        if chunk <= 0 or ctx < 0:
            raise ValueError("chunk_seconds must be positive and context_seconds non-negative")
        sched = StreamSchedule(chunk, ctx, mode)
        sched.check_first_window("restore_stream")
        seed = stream_dropout_seed(mode, dropout_seed, "restore_stream")
        eng = self._engine
        dev = f"cuda:{eng.device}"
        buf = np.zeros(0, dtype=np.float32)       # samples [base, base + len(buf)) of the stream
        base = 0                                  # stream index of buf[0]
        pos = 0                                   # next sample to emit
        k = 0                                     # windows restored so far

        def run(lo, hi, keep_lo, keep_hi):
            x = torch.from_numpy(np.ascontiguousarray(buf[lo - base: hi - base]))[None].to(dev)
            if mode == 1:                                                # restore_inmem's calls
                x, _ = eng.hf_cut(x)
                y = eng.restore(x, mode=0)
            elif mode == 2:
                y = eng.restore(x, mode=2, drop_keys=_upload_keys(np.array([(seed, k)], dtype=np.uint64), dev))
            else:
                y = eng.restore(x, mode=0)
            return y[0, keep_lo - lo: keep_hi - lo].cpu().numpy()

        for block in blocks:
            block = np.asarray(block, dtype=np.float32).reshape(-1)
            buf = np.concatenate([buf, block])
            windows, pos = sched.due(pos, base + len(buf), ended=False)
            for w in windows:
                yield run(*w)
                k += 1
            # audio no later window reads: before the next window's left context, less the widening of a short flush
            # window (StreamPool._trim's bound)
            drop = max(0, pos - ctx - sched.min_len) - base
            if drop > 0:
                buf, base = buf[drop:], base + drop
        windows, pos = sched.due(pos, base + len(buf), ended=True)
        for w in windows:
            yield run(*w)
            k += 1

    def stream_pool(self, chunk_seconds=2.0, context_seconds=1.0, max_windows=None, mode=0):
        """Extension: restore_stream for many live streams at once (StreamPool).  open() a stream per caller, push() its
        blocks as they arrive, close() it at its end, and call step() to restore every window that is due, of every
        stream, in one ragged CUDA-graph replay.  Each stream's output is bit-identical to restore_stream on that
        stream's audio alone with the same chunk_seconds / context_seconds / mode (and in mode 2 the dropout_seed given
        to open()).  max_windows: the most windows one step restores (default: as many as fit the device memory that is
        free, at most 64).  Blocks may be host arrays, or 1-D float32 CUDA tensors (any element stride), which the pool
        restores where they are and returns as new CUDA tensors without waiting for the GPU (StreamPool: the first block
        pushed fixes which)."""
        _check_cuda(False)
        return StreamPool(self._engine, chunk_seconds, context_seconds, max_windows, mode=mode)

    def restore(self, input, output, cuda=False, mode=0, your_vocoder_func=None, channels="mix"):
        """base.py:141-146.  channels (extension): "mix" (the default) restores the file's mono mix, as the reference
        does; "keep" restores each channel on its own and writes them all (restore_columns on wavio.read_wave), so a
        stereo file stays stereo.  A mono file gives the same output either way."""
        check_channels(channels, "restore")
        if channels == "keep":
            out_np_wav = self.restore_columns(wavio.read_wave(input, 44100), cuda=cuda, mode=mode,
                                              your_vocoder_func=your_vocoder_func)
        else:
            wav_10k = self._load_wav(input, sample_rate=44100)           # base.py:141-146
            out_np_wav = self.restore_inmem(wav_10k, cuda=cuda, mode=mode, your_vocoder_func=your_vocoder_func)
        wavio.save_wave(out_np_wav, fname=output, sample_rate=44100)

    def restore_columns(self, x, cuda=False, mode=0, your_vocoder_func=None):
        """Extension: the channels of x (L, C) float32 at 44.1 kHz, each restored on its own by restore_inmem, as a
        (C, L') array (row c: restore_inmem(x[:, c])[0]), which save_wave writes as C channels."""
        x = np.asarray(x, dtype=np.float32)
        if x.ndim != 2 or x.shape[1] < 1:
            raise ValueError(f"restore_columns takes an (L, C) array, one column per channel; got shape {x.shape}")
        return np.concatenate([self.restore_inmem(x[:, c], cuda=cuda, mode=mode, your_vocoder_func=your_vocoder_func)
                               for c in range(x.shape[1])])

    @torch.no_grad()
    def restore_files(self, inputs, outputs, mode=0, cuda=True, dropout_seed=None, channels="mix", gpus=None,
                      _budget=None, _on_wave=None, _on_wave_done=None, _messages=(), _devices=None):
        """Extension of the reference API: restore(inputs[i], outputs[i]) for many files, the files batched across each
        other.  Output file i is byte for byte what restore(inputs[i], outputs[i], mode=mode_i, channels=channels) writes
        in modes 0 and 1, for .wav and .flac at every rate and channel count the readers take.  In mode 2 with
        dropout_seed it is what save_wave(restore_inmem(load_mono(inputs[i]), mode=2, dropout_seed=seed_i), outputs[i])
        writes (with channels="keep": channel c restored with masks from the Philox keys (seed_i, (c << 32) | k), k the
        segment, so channel 0 has the mono call's masks and no two channels share theirs); without a seed the masks are
        random, with restore()'s distribution.

        mode: one of 0, 1, 2 for every file, or one per file (so an input may be listed several times with different
        outputs and modes).  dropout_seed: one int in [0, 2^64) or one per file, as in restore_many; it is the dropout of
        the files restored in mode 2, and refused when there is none.  channels: "mix" (the default) restores each file's
        mono mix, "keep" each of its channels (at most PCM16_MAX_CHANNELS = 8 per file, the device packer's bound and
        FLAC's).  A length mismatch, an empty list, a bad mode, seed or channels raises ValueError before anything is
        read.  Output directories are not created, as with restore().

        The files run in waves of consecutive files (plan_waves, every channel of a file counted), about twice the audio
        of the largest 30 s batch the free device memory holds, through three stages (run_waves): a reader thread
        decodes each file at its own rate (wavio.load_mono_native, or wavio.load_native's (L, C) with "keep"; the next
        files ahead in a four-thread pool) into pinned memory and checks it as restore_many would; the calling thread
        uploads the wave, runs one device-resident restore_many(..., sample_rate=) per mode present on the files (with
        "keep", on the columns x[:, c] of each uploaded file, read in place; an input listed several times in a wave is
        decoded and uploaded once), packs all the wave's outputs into 16-bit PCM on the device (Engine.pack_pcm16, the
        quantiser of save_wave bit for bit), queues one copy of them into pinned memory and an event, and goes on to the
        next wave without waiting; a writer thread waits for that event and writes each output with wavio.write_pcm16.
        The GPU never waits for the host between waves.

        Errors: every file before a failing one, in input order, is written and none after it is started; the exception
        is re-raised once the threads have drained.  A file that cannot be read or written raises RuntimeError, and one
        too short for its mode, at a bad rate or (with "keep") with more than 8 channels ValueError, each naming the
        file; such a file cuts its wave short, the files before it in that wave still being restored and written.

        gpus: None or 1 runs everything on this instance's device, as above.  gpus=N (an int, at most
        torch.cuda.device_count()) spreads the files over N devices: this instance's and the next N - 1 visible ones in
        index order (wrapping past the last).  Each file is sized from its headers (wavio.probe) and the files are
        assigned by plan_devices, every occurrence of one input on one device.  One worker process per extra device,
        started with the spawn method, receives the engine's weights through host shared memory (one copy of its arena
        from the device, no checkpoint read, so an instance made by from_engine works too), builds an Engine of the same
        precision on its device and restores its files with the single-device restore_files, its own wave budget and
        its files' modes and seeds; this instance restores its own device's files meanwhile.  Every output is the same
        file, byte for byte, as with one device.  Errors: within a device the rule above holds; the other devices go on
        to finish their own files, and once every device has finished the call raises the error of the lowest-indexed
        file that failed, with its type and message (a later file on another device may then have been written, the
        one difference from gpus=1).  A worker that dies raises RuntimeError naming its device.  Every worker process
        has exited when the call returns or raises.  As with DataLoader workers, a script that calls this with gpus > 1
        must guard its entry point with `if __name__ == "__main__":`, since the spawned workers import it.

        _budget (samples at 44.1 kHz per wave), _on_wave(jobs) (called as a wave starts) and _on_wave_done(jobs,
        seconds) (called as its outputs reach the host, with the GPU time from its upload to its copy back) are for the
        command line and the tests; with gpus > 1 the callbacks cannot reach the workers, so _messages names the
        command line's lines each device prints itself ("processing", "took").  _devices (the tests') overrides the
        devices gpus > 1 runs on, e.g. [0, 0] for two processes on one device."""
        inputs, outputs, modes, seeds, keep = self._check_files(inputs, outputs, mode, cuda, dropout_seed, channels)
        if gpus is not None:
            if isinstance(gpus, (bool, np.bool_)) or not isinstance(gpus, numbers.Integral) or gpus < 1:
                raise ValueError(f"restore_files: gpus is {gpus!r}; it must be a positive int")
            if _devices is None and gpus > torch.cuda.device_count():
                raise ValueError(f"restore_files: gpus={gpus}, but {torch.cuda.device_count()} CUDA device(s) are "
                                 "visible")
        if (gpus is None or gpus == 1) and _devices is None:
            return self._restore_files(inputs, outputs, modes, seeds, keep, _budget, _on_wave, _on_wave_done)
        if _on_wave is not None or _on_wave_done is not None:
            raise ValueError("restore_files: _on_wave / _on_wave_done run in one process; with gpus > 1 use _messages")
        eng = self._engine
        devices = list(_devices) if _devices is not None else \
            [(eng.device + k) % torch.cuda.device_count() for k in range(int(gpus))]
        shards = plan_devices(_probe_samples(inputs, modes, keep), inputs, len(devices))
        arena = torch.empty(eng.arena.numel(), dtype=torch.uint8).share_memory_()
        arena.copy_(eng.arena)
        args = _ShardArgs(self, inputs=inputs, outputs=outputs, modes=modes, seeds=seeds,
                          channels="keep" if keep else "mix", budget=_budget, messages=tuple(_messages),
                          precision=eng.precision, table=eng.table, arena=arena)
        from .parallel import run_on_devices
        run_on_devices([(d, s) for d, s in zip(devices, shards) if s], _restore_shard, args)

    def _check_files(self, inputs, outputs, mode, cuda, dropout_seed, channels):
        """restore_files' argument checks: (inputs, outputs, modes, seeds, keep) as lists of one entry per file (seeds
        None without dropout_seed), or ValueError before anything is read."""
        _check_cuda(cuda)
        inputs, outputs = [str(p) for p in inputs], [str(p) for p in outputs]
        n = len(inputs)
        if n == 0 or len(outputs) != n:
            raise ValueError(f"restore_files takes a non-empty list of inputs and as many outputs; got {n} inputs and "
                             f"{len(outputs)} outputs")
        modes = list(mode) if isinstance(mode, (list, tuple, np.ndarray)) else [mode] * n
        if len(modes) != n:
            raise ValueError(f"restore_files: mode has {len(modes)} entries for {n} files; give one mode, or one per file")
        for i, m in enumerate(modes):
            if isinstance(m, (bool, np.bool_)) or m not in (0, 1, 2):
                raise ValueError(f"restore_files: file {i} has mode {m!r}; mode must be 0, 1 or 2")
        modes = [int(m) for m in modes]
        check_channels(channels, "restore_files")
        keep = channels == "keep"
        seeds = None
        if dropout_seed is not None:
            if 2 not in modes:
                raise ValueError("restore_files: dropout_seed is mode 2's dropout; no file is restored in mode 2")
            seeds = dropout_seeds(dropout_seed, 2, None, n, "restore_files")
        return inputs, outputs, modes, seeds, keep

    def _restore_files(self, inputs, outputs, modes, seeds, keep, _budget, _on_wave, _on_wave_done):
        """restore_files on this instance's device, on checked arguments (_check_files)."""
        n = len(inputs)
        eng = self._engine
        dev = f"cuda:{eng.device}"
        budget = _budget if _budget is not None else 2 * eng.max_batch(SEG_LENGTH) * SEG_LENGTH
        from concurrent.futures import ThreadPoolExecutor
        pool = ThreadPoolExecutor(max_workers=4, thread_name_prefix="vfx-decode")
        ahead = {}                                                       # input -> its decode, started ahead of use

        def decode(path):
            x, sr = wavio.load_native(path) if keep else wavio.load_mono_native(path)
            return torch.from_numpy(x).pin_memory(), sr

        def load(i, prev):
            if prev is None:
                for j in range(i, min(n, i + 8)):        # the next inputs decode in the background, each path once
                    if j not in ahead and inputs[j] not in inputs[i:j]:
                        ahead[j] = pool.submit(decode, inputs[j])
                try:
                    x, sr = (ahead.pop(i, None) or pool.submit(decode, inputs[i])).result()
                except Exception as e:
                    raise RuntimeError(f"restore_files: {inputs[i]}: {e}") from e
                prev = (x, resample.check_rate(sr, f"restore_files: {inputs[i]}"))
            return prev, file_samples(tuple(prev[0].shape), prev[1], modes[i], inputs[i])

        def restore(wave):
            ids = [i for i, _ in wave]
            if _on_wave is not None:
                _on_wave(ids)
            start, done = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            up = {}                                                      # id(item) -> the input on the device
            for _, item in wave:
                if id(item) not in up:
                    up[id(item)] = item[0].to(dev, non_blocking=True)
            outs = {}                                                    # file -> its restored channels
            for m in sorted(set(modes[i] for i in ids)):
                run = [(i, item, c) for i, item in wave if modes[i] == m
                       for c in range(up[id(item)].shape[1] if keep else 1)]
                ys = self.restore_many([up[id(item)][:, c] if keep else up[id(item)] for _, item, c in run], cuda=True,
                                       mode=m, sample_rate=[item[1] for _, item, _ in run],
                                       dropout_seed=[seeds[i] for i, _, _ in run] if seeds is not None and m == 2 else None,
                                       _stream_base=[c << 32 for _, _, c in run])
                for (i, _, _), y in zip(run, ys):
                    outs.setdefault(i, []).append(y.view(-1))
            pcm, offs = eng.pack_pcm16([outs[i] for i in ids])
            host = torch.empty(pcm.shape, dtype=torch.int16, pin_memory=True)
            host.copy_(pcm, non_blocking=True)
            done.record()
            return host, {i: (offs[k], offs[k + 1], len(outs[i])) for k, i in enumerate(ids)}, start, done

        def write(ids, result):
            host, spans, start, done = result
            done.synchronize()
            if _on_wave_done is not None:
                _on_wave_done(ids, start.elapsed_time(done) / 1e3)
            y = host.numpy()
            for i in ids:
                a, b, C = spans[i]
                try:
                    wavio.write_pcm16(y[a:b].reshape(-1, C), fname=outputs[i], sample_rate=44100)
                except Exception as e:
                    raise _stopped_at(RuntimeError(f"restore_files: {outputs[i]}: {e}"), i) from e

        try:
            run_waves(inputs, budget, load, restore, write)
        finally:
            pool.shutdown(wait=True, cancel_futures=True)
