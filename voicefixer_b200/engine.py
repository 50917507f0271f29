"""Python wrapper of the C-ABI engine: device memory, streams and weight upload (plumbing only).

All compute goes through libvfx_b200.so; torch is used for device buffers, the current CUDA
stream and (in parallel.py) torch.distributed."""
import ctypes
import os
import numpy as np
import torch

from . import _lib, resample
from .weights import pack_analysis, pack_vocoder

ALIGN = 256


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def default_precision():
    """"tf32": wgmma tf32 on tf32-rounded fp32 operands -- the arithmetic class of the reference's own CUDA path
    (cuDNN TF32 convolutions; waveform within 2e-3 relative RMS of the fp32 CPU path).  VFX_PRECISION selects another mode:
    "bf16" (wgmma on bf16 operands, half the operand traffic; within 3e-2 relative RMS / 5e-3 mean-abs, inside the reference's
    own 1e-2 mean-abs acceptance bar), "fp16" (wgmma on fp16 operands: tf32's 10-bit mantissa, hence tf32's tolerance, with the
    bf16 mode's traffic -- within fp16's exponent range) or "fp32" (SIMT fp32 validation path, within 2e-4 of the reference)."""
    return os.environ.get("VFX_PRECISION", "tf32")


class _WorkspaceQueries:
    """The library's workspace planners on the engine handle `self.h`."""

    def workspace_bytes(self, B, L):
        """restore() on B items of L samples; 0 for a vocoder-only weight set."""
        return int(self.lib.vfx_workspace_bytes(self.h, int(B), int(L)))

    def workspace_bytes_frames(self, B, T):
        """analysis / vocoder entry points on B items of T mel frames."""
        return int(self.lib.vfx_workspace_bytes_frames(self.h, int(B), int(T)))

    def analysis_workspace_bytes(self, B, L):
        """analysis_ragged() on B items of (at most) L samples, in either mode; 0 for a vocoder-only weight set."""
        return int(self.lib.vfx_analysis_workspace_bytes(self.h, int(B), int(L)))

    def oracle_workspace_bytes(self, B, L):
        """Vocoder.oracle's device path on B recordings of (at most) L samples (0 for an out-of-range shape)."""
        return int(self.lib.vfx_oracle_workspace_bytes(self.h, int(B), int(L)))


class Planner(_WorkspaceQueries):
    """Planning-only engine (vfx_engine_create with device -1): validates a packed weight set against what the
    kernels expect (names, byte sizes) and sizes the activation workspace for a batch -- no GPU, no CUDA call.
    `packed`: {name: CPU tensor} from weights.pack_analysis / pack_vocoder (either both, or the vocoder alone)."""

    def __init__(self, packed, precision):
        self.lib = _lib.load()
        self.precision = precision
        h = ctypes.c_void_p()
        _lib.check(self.lib.vfx_engine_create(ctypes.byref(h), -1, _lib.PREC[precision]), "vfx_engine_create")
        self.h = h
        table, self.weight_bytes = Engine.layout(packed)
        for name, off, nbytes in table:          # addresses are never dereferenced by a planning-only engine
            _lib.check(self.lib.vfx_engine_set_tensor(self.h, name.encode(), ctypes.c_void_p(ALIGN + off), nbytes),
                       f"set_tensor({name})")
        _lib.check(self.lib.vfx_engine_finalize(self.h), "vfx_engine_finalize")

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.vfx_engine_destroy(self.h)
            self.h = None


class Engine(_WorkspaceQueries):
    """One engine per process / GPU.  `ana`, `voc`: reference-layout state dicts (CPU tensors).

    Every call launches on torch.cuda.current_stream().  The engine's workspace and its resampling taps are shared by
    all its calls, so a call made on another stream than the one before it first makes its stream wait for the work
    already queued on that one (_shared_stream): calls on several streams run in the order they were made, never at
    the same time, and a buffer the engine replaces is not reused before every stream that read it has finished with
    it.  Calls are made from one host thread at a time."""

    def __init__(self, ana=None, voc=None, device=None, precision=None, packed=None):
        if not torch.cuda.is_available():
            raise RuntimeError("voicefixer_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")
        self.lib = _lib.load()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.precision = precision or default_precision()
        if self.precision not in _lib.PREC:
            raise ValueError(f"precision must be one of {list(_lib.PREC)}")
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.vfx_engine_create(ctypes.byref(h), self.device, _lib.PREC[self.precision]),
                       "vfx_engine_create")
        self.h = h
        self._ws = None
        self._last_stream = None  # the stream of the last call that used the shared workspace or taps
        self.arena = None
        self.table = None
        if packed is None and ana is not None:
            packed = {}
            packed.update(pack_analysis(ana, self.precision))
            packed.update(pack_vocoder(voc, self.precision))
        if packed is not None:
            self.upload(packed)

    # ------------------------------------------------------------------ weights
    @staticmethod
    def layout(packed):
        """[(name, offset, nbytes)] and total bytes of the single weight arena."""
        table, off = [], 0
        for name in sorted(packed):
            t = packed[name]
            nbytes = t.numel() * t.element_size()
            table.append((name, off, nbytes))
            off += (nbytes + ALIGN - 1) // ALIGN * ALIGN
        return table, off

    def upload(self, packed):
        table, total = self.layout(packed)
        host = torch.empty(total, dtype=torch.uint8).pin_memory()
        for name, off, nbytes in table:
            host[off:off + nbytes] = packed[name].contiguous().view(torch.uint8).reshape(-1)
        arena = torch.empty(total, dtype=torch.uint8, device=f"cuda:{self.device}")
        arena.copy_(host, non_blocking=False)
        self.attach(arena, table)

    def attach(self, arena, table):
        """Registers views of an arena that is already on this device (e.g. after an NCCL broadcast)."""
        self.arena, self.table = arena, table
        base = arena.data_ptr()
        for name, off, nbytes in table:
            _lib.check(self.lib.vfx_engine_set_tensor(self.h, name.encode(), ctypes.c_void_p(base + off), nbytes),
                       f"set_tensor({name})")
        _lib.check(self.lib.vfx_engine_finalize(self.h), "vfx_engine_finalize")

    def set_option(self, key, value):
        _lib.check(self.lib.vfx_engine_set_option(self.h, key.encode(), int(value)), "set_option")

    def profile(self, on=True):
        self.set_option("profile", 1 if on else 0)

    def profile_report(self):
        """{tag: dict(count, ms, flops, bytes)} of everything launched since the last report."""
        buf = ctypes.create_string_buffer(1 << 16)
        _lib.check(self.lib.vfx_profile_report(self.h, buf, len(buf)), "vfx_profile_report")
        rep = {}
        for line in buf.value.decode().splitlines():
            tag, n, ms, fl, by = line.split()
            rep[tag] = dict(count=int(n), ms=float(ms), flops=float(fl), bytes=float(by))
        return rep

    def launch_count(self):
        return int(self.lib.vfx_launch_count())

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.vfx_engine_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ------------------------------------------------------------------ workspace
    def _shared_stream(self):
        """The current stream, made to wait for the work queued on the stream of the previous call that used the shared
        workspace or taps, if that was another stream (a device-side wait: the host does not wait)."""
        st = torch.cuda.current_stream(self.device)
        if self._last_stream is not None and self._last_stream != st:
            st.wait_stream(self._last_stream)
        self._last_stream = st
        return st

    def _workspace(self, nbytes):
        if nbytes == 0:
            raise _lib.VfxError("workspace query returned 0: the shape is out of range (restore() needs L > 1024 samples) or this "
                                "engine holds the vocoder weights only (stand-alone Vocoder: restore/analysis are unavailable)")
        st = self._shared_stream()
        if self._ws is None or self._ws.numel() < nbytes:
            if self._ws is not None:   # not reused before st's queued work, which follows every earlier use, is done
                self._ws.record_stream(st)
            self._ws = None     # (captured graphs own their workspace tensors; see make_graph)
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=f"cuda:{self.device}")
        return self._ws

    def max_batch(self, L, cap=64, reserve=2 << 30, extra_per_item=0, analysis=False):
        """Largest number of equal-length items (<= cap) whose restore() workspace fits the memory that is free right now,
        or the workspace this engine already holds if that is larger (_fit), keeping `reserve` bytes back.  At least 1.
        extra_per_item: other
        device bytes each item needs alongside (e.g. the mode-1 pre-filter's workspace and output).  analysis: size by
        analysis_ragged()'s workspace instead, which leaves out the vocoder's."""
        q = self.analysis_workspace_bytes if analysis else self.workspace_bytes
        return self._fit(q(2, L) - q(1, L) + int(extra_per_item), cap, reserve)

    def max_batch_frames(self, T, cap=64, reserve=2 << 30, extra_per_item=0):
        """max_batch for the vocoder: the largest number of mels of T frames (<= cap) whose vocoder() workspace fits the
        memory that is free right now, keeping `reserve` bytes back.  At least 1."""
        return self._fit(self.workspace_bytes_frames(2, T) - self.workspace_bytes_frames(1, T) + int(extra_per_item),
                         cap, reserve)

    def _fit(self, per_item, cap, reserve):
        """How many items of per_item bytes fit: at most cap, at least 1, keeping `reserve` bytes back.  A batch either
        reuses the workspace this engine holds or gets a new one out of the memory that is free now; the two are never
        added up.  A new workspace cannot count on the held one's memory: the caching allocator keeps a freed block
        cached, and cannot hand it back to the device while a smaller tensor has been carved out of it."""
        free, _ = torch.cuda.mem_get_info(self.device)
        avail = max(free, self._ws.numel() if self._ws is not None else 0) - reserve
        return int(max(1, min(cap, avail // max(1, per_item))))

    def _dev(self, x):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        return x.to(device=f"cuda:{self.device}", dtype=torch.float32).contiguous()

    # ------------------------------------------------------------------ the five seams
    def frontend(self, wav, return_sp=False):
        """wav (B, L) -> mel (B, T, 128) [, sp (B, T, 1025)]."""
        wav = self._dev(wav)
        B, L = wav.shape
        T = 1 + L // 441
        mel = torch.empty(B, T, 128, device=wav.device)
        sp = torch.empty(B, T, 1025, device=wav.device) if return_sp else None
        _lib.check(self.lib.vfx_frontend_mel(self.h, _ptr(wav), B, L, _ptr(mel), _ptr(sp), _stream()), "vfx_frontend_mel")
        return (mel, sp) if return_sp else mel

    def analysis(self, mel, mode=0, drop_masks=None, drop_keys=None):
        """mel (B, T, 128) linear -> log10 mel (B, T, 128).  drop_keys (mode 2, in place of drop_masks): seeded dropout
        keys, as in restore() (vfx_analysis_seeded)."""
        mel = self._dev(mel)
        B, T, F = mel.shape
        if F != 128:
            raise AssertionError("mel must have 128 bins")
        if drop_keys is not None:
            self._check_keys(drop_keys, B, mode, drop_masks)
        out = torch.empty_like(mel)
        ws = self._workspace(self.workspace_bytes_frames(B, T))
        if drop_keys is not None:
            _lib.check(self.lib.vfx_analysis_seeded(self.h, _ptr(mel), B, T, _ptr(drop_keys), _ptr(out), _ptr(ws),
                                                    ws.numel(), _stream()), "vfx_analysis_seeded")
            return out
        dm = None
        if drop_masks is not None:
            dm = drop_masks.to(device=mel.device, dtype=torch.uint8).contiguous()
            assert tuple(dm.shape) == (2, B, T, 512)
        _lib.check(self.lib.vfx_analysis(self.h, _ptr(mel), B, T, int(mode), _ptr(dm), _ptr(out), _ptr(ws), ws.numel(),
                                         _stream()), "vfx_analysis")
        return out

    def vocoder(self, mel, input_is_log=False, trim_len=-1, scale=1.0, lens=None, ws=None):
        """mel (B, T, 128) -> wav (B, out_len).

        lens (ragged batch): int32 device tensor (B,) of per-item frame counts <= T.  Row b of `mel` then holds item b in
        its first lens[b] frames, and row b of the result (B, (T + T % 2 + 4) * 441) is bit-identical to the vocoder on
        that item alone, its (T_b + T_b % 2 + 4) * 441 samples untrimmed, followed by zeros (vfx_vocoder_ragged).  Lengths
        are read on the device, so a captured graph serves any lengths.  trim_len must stay -1."""
        mel = self._dev(mel)
        B, T, F = mel.shape
        if F != 128:
            raise AssertionError("mel must have 128 bins")
        S = (T + T % 2 + 4) * 441
        if ws is None:
            ws = self._workspace(self.workspace_bytes_frames(B, T))
        if lens is not None:
            _check_lens(lens, B)
            if trim_len != -1:
                raise ValueError("a ragged vocoder batch is untrimmed: trim_len must be -1")
            out = torch.empty(B, S, device=mel.device)
            _lib.check(self.lib.vfx_vocoder_ragged(self.h, _ptr(mel), B, T, _ptr(lens), int(bool(input_is_log)), _ptr(out),
                                                   float(scale), _ptr(ws), ws.numel(), _stream()), "vfx_vocoder_ragged")
            return out
        out = torch.empty(B, S if trim_len < 0 else trim_len, device=mel.device)
        _lib.check(self.lib.vfx_vocoder(self.h, _ptr(mel), B, T, int(bool(input_is_log)), _ptr(out), int(trim_len),
                                        float(scale), _ptr(ws), ws.numel(), _stream()), "vfx_vocoder")
        return out

    def vocoder_cond(self, cond, trim_len=-1, scale=1.0):
        """normalised conditions (B, Tc, 128) [channels-last] -> wav (B, Tc*441)."""
        cond = self._dev(cond)
        B, Tc, F = cond.shape
        out = torch.empty(B, Tc * 441 if trim_len < 0 else trim_len, device=cond.device)
        ws = self._workspace(self.workspace_bytes_frames(B, Tc))
        _lib.check(self.lib.vfx_vocoder_cond(self.h, _ptr(cond), B, Tc, _ptr(out), int(trim_len), float(scale), _ptr(ws),
                                             ws.numel(), _stream()), "vfx_vocoder_cond")
        return out

    def oracle(self, wav, lens=None, scale=1.0, return_cond=False):
        """Vocoder.oracle on the device (vfx_oracle): wav (B, L) -> wav (B, Tc * 441), Tc = T + T % 2 + 4, T = 1 + L // 441,
        times `scale` (oracle() writes 2^15 x the Generator output).  Each row is peak-normalised on its own.

        lens (ragged batch): int32 device tensor (B,) of per-item lengths <= L; row b of the result then holds item b's
        (T_b + T_b % 2 + 4) * 441 samples and zeros after.  return_cond: run the front end only (vfx_oracle_cond) and
        return its fp32 conditions (B, Tc, 128), channels-last, with zeros after each item's Tc_b rows."""
        wav = self._dev(wav)
        B, L = wav.shape
        if lens is not None:
            _check_lens(lens, B)
        T = 1 + L // 441
        Tc = T + T % 2 + 4
        if return_cond:                                    # the front end's workspace: its per-item peaks
            ws = self._workspace((4 * B + 255) // 256 * 256)
            cond = torch.empty(B, Tc, 128, device=wav.device)
            _lib.check(self.lib.vfx_oracle_cond(self.h, _ptr(wav), B, L, _ptr(lens), _ptr(cond), _ptr(ws), ws.numel(),
                                                _stream()), "vfx_oracle_cond")
            return cond
        ws = self._workspace(self.oracle_workspace_bytes(B, L))
        out = torch.empty(B, Tc * 441, device=wav.device)
        _lib.check(self.lib.vfx_oracle(self.h, _ptr(wav), B, L, _ptr(lens), float(scale), _ptr(out), _ptr(ws), ws.numel(),
                                       _stream()), "vfx_oracle")
        return out

    def restore(self, wav, mode=0, drop_masks=None, out=None, ws=None, lens=None, drop_keys=None):
        """wav (B, L) on device -> restored wav (B, L) on device (one launch sequence).

        lens (ragged batch): int32 device tensor (B,) of per-item lengths <= L.  Row b of `wav` then holds item b in its
        first lens[b] samples; row b of the result is bit-identical to restoring that item alone, followed by zeros.
        Lengths are read on the device (vfx_restore_ragged_mode), so a captured graph serves any lengths.  In mode 2,
        drop_masks is (2, B, T_cap, 512) with T_cap = 1 + L // 441 (item b reads [:, b, :T_b]) and every item needs more
        than 64 frames (1 + lens[b] // 441 > 64; an item below that gets finite, unspecified samples).

        drop_keys (mode 2, in place of drop_masks): seeded dropout (vfx_restore_seeded), a contiguous int64 CUDA tensor
        (B, 2) whose row b holds the bit patterns of item b's (seed, stream) (vfx_drop_key; a value >= 2^63 appears as
        its negative two's complement).  Item b's masks are then philox.seeded_masks(seed_b, stream_b, T_b), computed in
        the kernels, so its row depends on its own samples and key only."""
        wav = self._dev(wav)
        B, L = wav.shape
        if drop_keys is not None:
            self._check_keys(drop_keys, B, mode, drop_masks)
        if out is None:
            out = torch.empty_like(wav)
        if ws is None:
            ws = self._workspace(self.workspace_bytes(B, L))
        if drop_keys is not None:
            if lens is not None:
                _check_lens(lens, B)
            _lib.check(self.lib.vfx_restore_seeded(self.h, _ptr(wav), B, L, _ptr(lens), _ptr(drop_keys), _ptr(out),
                                                   _ptr(ws), ws.numel(), _stream()), "vfx_restore_seeded")
            return out
        dm = None
        if drop_masks is not None:
            dm = drop_masks.to(device=wav.device, dtype=torch.uint8).contiguous()
        if lens is not None:
            _check_lens(lens, B)
            if dm is not None and tuple(dm.shape) != (2, B, 1 + L // 441, 512):
                raise ValueError(f"drop_masks must have shape (2, {B}, {1 + L // 441}, 512), got {tuple(dm.shape)}")
            _lib.check(self.lib.vfx_restore_ragged_mode(self.h, _ptr(wav), B, L, _ptr(lens), int(mode), _ptr(dm), _ptr(out),
                                                        _ptr(ws), ws.numel(), _stream()), "vfx_restore_ragged_mode")
            return out
        _lib.check(self.lib.vfx_restore(self.h, _ptr(wav), B, L, int(mode), _ptr(dm), _ptr(out), _ptr(ws), ws.numel(),
                                        _stream()), "vfx_restore")
        return out

    def analysis_ragged(self, wav, lens, mode=0, drop_masks=None, drop_keys=None):
        """The analysis half of restore(..., lens=lens) (vfx_analysis_ragged): wav (B, L) on device, row b holding item b in
        its first lens[b] samples -> log10 mel (B, T_cap, 128), T_cap = 1 + L // 441.  The first 1 + lens[b] // 441 rows
        of item b are bit-identical to analysis(frontend(item b alone)); the rows after them are unspecified.

        mode 0 or 2 (mode 1: hf_cut(wav, lens=lens) first, then mode 0).  In mode 2, drop_masks (2, B, T_cap, 512) or
        drop_keys (restore()'s seeded keys) supply the dropout, and every item needs more than 64 frames."""
        wav = self._dev(wav)
        B, L = wav.shape
        _check_lens(lens, B)
        T = 1 + L // 441
        if drop_keys is not None:
            self._check_keys(drop_keys, B, mode, drop_masks)
        dm = None
        if drop_masks is not None:
            dm = drop_masks.to(device=wav.device, dtype=torch.uint8).contiguous()
            if tuple(dm.shape) != (2, B, T, 512):
                raise ValueError(f"drop_masks must have shape (2, {B}, {T}, 512), got {tuple(dm.shape)}")
        out = torch.empty(B, T, 128, device=wav.device)
        ws = self._workspace(self.analysis_workspace_bytes(B, L))
        _lib.check(self.lib.vfx_analysis_ragged(self.h, _ptr(wav), B, L, _ptr(lens), int(mode), _ptr(dm), _ptr(drop_keys),
                                                _ptr(out), _ptr(ws), ws.numel(), _stream()), "vfx_analysis_ragged")
        return out

    def _check_keys(self, keys, B, mode, drop_masks):
        if drop_masks is not None:
            raise ValueError("drop_keys and drop_masks are two sources of the same masks: give one of them")
        if int(mode) != 2:
            raise ValueError(f"drop_keys is mode 2's dropout; mode is {mode}")
        if not (keys.is_cuda and keys.device == torch.device(f"cuda:{self.device}") and keys.dtype == torch.int64
                and tuple(keys.shape) == (B, 2) and keys.is_contiguous()):
            raise ValueError(f"drop_keys must be a contiguous int64 tensor of shape ({B}, 2) on cuda:{self.device}")

    def make_graph(self, wav, out, mode=0, lens=None, ws=None, drop_keys=None):
        """Captures the whole restore() launch sequence (~360 kernels) for the given device buffers into a
        CUDA graph; returns an object whose .replay() re-runs it (inputs are read from `wav`, results land in
        `out`).  Shapes, buffers and the workspace are frozen into the graph.  With `lens` (ragged batch) the graph
        reads the lengths from that buffer at every replay: refill it, like `wav`, before replay().

        ws (optional): a uint8 device workspace of at least graph_workspace_bytes(*wav.shape, mode) bytes for the graph to
        use, e.g. one that several graphs share because they never replay at the same time; without it the graph gets
        its own.

        mode 1 (needs lens): the graph runs restore_many's pair, the ragged pre-filter (hf_cut) into a (B, L) row buffer
        and lengths of the graph's own, then restore(mode=0) on them: row b of `out` holds item b's 512 * (lens[b] // 512)
        restored samples, then zeros.  Both use `ws`, one after the other.  drop_keys (mode 2, optional): seeded dropout
        (restore()), a contiguous int64 (B, 2) CUDA buffer read at every replay, like lens."""
        assert wav.is_cuda and out.is_cuda and wav.shape == out.shape
        B, L = wav.shape
        mid = mid_lens = None
        if mode == 1:
            if lens is None:
                raise ValueError("make_graph: mode 1 runs the ragged pre-filter, which needs lens")
            mid = torch.empty_like(wav)
            mid_lens = torch.empty(B, dtype=torch.int32, device=wav.device)
        # the graph bakes raw device pointers in: it gets its OWN workspace unless given one, and the returned object keeps
        # every buffer it touches alive (a later, larger call may replace the engine's shared workspace)
        need = self.graph_workspace_bytes(B, L, mode)
        if ws is None:
            ws = torch.empty(need, dtype=torch.uint8, device=wav.device)
        elif not (ws.is_cuda and ws.dtype == torch.uint8 and ws.numel() >= need):
            raise ValueError(f"make_graph: ws must be a uint8 CUDA tensor of at least {need} bytes")

        def run():
            if mode == 1:
                self.hf_cut(wav, lens=lens, out=mid, lens_out=mid_lens, ws=ws)
                self.restore(mid, mode=0, out=out, ws=ws, lens=mid_lens)
            else:
                self.restore(wav, mode=mode, out=out, ws=ws, lens=lens, drop_keys=drop_keys)

        side = torch.cuda.Stream(device=wav.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                                # warm-up: one-time attribute / table setup
            for _ in range(2):
                run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run()
        g._keep = (ws, wav, out, lens, mid, mid_lens, drop_keys, self.arena)
        return g

    def graph_workspace_bytes(self, B, L, mode=0):
        """The workspace make_graph's graph uses on B items of (at most) L samples in `mode`: restore()'s, and in mode 1
        the pre-filter's if that is larger (the two run one after the other)."""
        need = self.workspace_bytes(B, L)
        return max(need, self.hf_cut_workspace_bytes(B, L)) if mode == 1 else need

    @staticmethod
    def hf_cut_workspace_bytes(B, L):
        """Workspace of hf_cut() on B items of (at most) L samples (vfx_hf_cut_workspace_bytes; no engine needed)."""
        return int(_lib.load().vfx_hf_cut_workspace_bytes(int(B), int(L)))

    @staticmethod
    def resample_workspace_bytes(B):
        """Workspace of resample() on B items (vfx_resample_workspace_bytes; no engine needed)."""
        return int(_lib.load().vfx_resample_workspace_bytes(int(B)))

    def _taps_for(self, rates):
        """{(up, down): (offset, length)} of the rates' taps in the engine's device tap buffer, which holds every ratio
        this engine has resampled so far; a new ratio re-uploads the buffer once."""
        if not hasattr(self, "_taps_off"):
            self._taps_off, self._taps_host, self._taps_dev = {}, [], None
        fresh = False
        for r in rates:
            key = resample.ratio(r)
            if key != (1, 1) and key not in self._taps_off:
                h, _ = resample.taps(r)
                self._taps_off[key] = (sum(len(t) for t in self._taps_host), len(h))
                self._taps_host.append(h)
                fresh = True
        if fresh:                              # pinned and stream-ordered: the upload makes the host wait for nothing
            st = self._shared_stream()
            if self._taps_dev is not None:     # not reused before st's queued work, which follows every earlier read, is done
                self._taps_dev.record_stream(st)
            host = torch.from_numpy(np.concatenate(self._taps_host)).pin_memory()
            self._taps_dev = host.to(f"cuda:{self.device}", non_blocking=True)
        return self._taps_off

    def resample(self, x, items, L_cap):
        """Rate conversion to 44.1 kHz on the device (vfx_resample), bit-identical to wavio._resample on the host.

        x: 1-D float32 device tensor, the staged input windows.  items: one (rate, n_in, x_off, x_first, x_len, y_first,
        y_len) per row: output samples [y_first, y_first + y_len) of a recording of n_in samples at `rate`, whose samples
        [x_first, x_first + x_len) are x[x_off : x_off + x_len] (resample.window gives the window an output range needs).
        Returns (y (B, L_cap) with row b's y_len samples then zeros, lens (B,) int32 device tensor of the y_len)."""
        x = x.reshape(-1)
        if not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()):
            raise ValueError("x must be a contiguous float32 CUDA tensor")
        B = len(items)
        offs = self._taps_for([it[0] for it in items])
        table = (_lib.ResampleItem * B)()
        for b, (rate, n_in, x_off, x_first, x_len, y_first, y_len) in enumerate(items):
            up, down = resample.ratio(rate)
            h_off, h_len = offs.get((up, down), (0, 0))
            t = table[b]
            t.x_off, t.x_first, t.n_in, t.x_len = int(x_off), int(x_first), int(n_in), int(x_len)
            t.y_first, t.y_len = int(y_first), int(y_len)
            t.up, t.down, t.rem, t.h_off, t.h_len = up, down, resample.taps(rate)[1], h_off, h_len
        h = self._taps_dev
        y = torch.empty(B, int(L_cap), device=x.device)
        lens = torch.empty(B, dtype=torch.int32, device=x.device)
        ws = self._workspace(self.resample_workspace_bytes(B))
        _lib.check(self.lib.vfx_resample(self.h, _ptr(x), x.numel(), _ptr(h), 0 if h is None else h.numel(), table, B,
                                         _ptr(y), int(L_cap), _ptr(lens), _ptr(ws), ws.numel(), _stream()), "vfx_resample")
        return y, lens

    @staticmethod
    def resample_src_workspace_bytes(B):
        """Workspace of resample_src() on B items (vfx_resample_src_workspace_bytes; no engine needed)."""
        return int(_lib.load().vfx_resample_src_workspace_bytes(int(B)))

    def resample_src(self, items, L_cap, y=None, lens=None):
        """resample() on recordings that are already on the device, read in place (vfx_resample_src): the same
        arithmetic, bit for bit, without staged windows; a rate of 44100 is a copy, so one launch builds a batch's rows.

        items: one (src, rate, y_first, y_len) per row: output samples [y_first, y_first + y_len) of the 44.1 kHz stream
        of src, a 1-D float32 CUDA tensor on this engine's device with any element stride, at `rate`.  src is never
        written.  Returns (y (B, L_cap) with row b's y_len samples then zeros, lens (B,) int32 device tensor of the
        y_len).  y, lens (optional): existing contiguous (B, L_cap) float32 / (B,) int32 tensors on this device to
        write them into (e.g. the first rows of a captured graph's input), instead of new ones."""
        dev = torch.device(f"cuda:{self.device}")
        for b, (src, *_) in enumerate(items):
            if not (src.is_cuda and src.device == dev and src.dtype == torch.float32 and src.dim() == 1):
                raise ValueError(f"resample_src: item {b}: src must be a 1-D float32 tensor on {dev}")
        B = len(items)
        if y is not None and not (y.is_cuda and y.device == dev and y.dtype == torch.float32 and y.is_contiguous()
                                  and tuple(y.shape) == (B, int(L_cap))):
            raise ValueError(f"resample_src: y must be a contiguous ({B}, {int(L_cap)}) float32 tensor on {dev}")
        if lens is not None and not (lens.device == dev and lens.dtype == torch.int32 and lens.is_contiguous()
                                     and tuple(lens.shape) == (B,)):
            raise ValueError(f"resample_src: lens must be a contiguous ({B},) int32 tensor on {dev}")
        offs = self._taps_for([it[1] for it in items])
        table = (_lib.ResampleSrcItem * B)()
        for b, (src, rate, y_first, y_len) in enumerate(items):
            up, down = resample.ratio(rate)
            t = table[b]
            t.src, t.stride, t.n_in = src.data_ptr(), src.stride(0), src.shape[0]
            t.y_first, t.y_len = int(y_first), int(y_len)
            t.up, t.down, t.rem = up, down, resample.taps(rate)[1]
            t.h_off, t.h_len = offs.get((up, down), (0, 0))
        h = self._taps_dev
        if y is None:
            y = torch.empty(B, int(L_cap), device=dev)
        if lens is None:
            lens = torch.empty(B, dtype=torch.int32, device=dev)
        ws = self._workspace(self.resample_src_workspace_bytes(B))
        _lib.check(self.lib.vfx_resample_src(self.h, _ptr(h), 0 if h is None else h.numel(), table, B, _ptr(y),
                                             int(L_cap), _ptr(lens), _ptr(ws), ws.numel(), _stream()),
                   "vfx_resample_src")
        return y, lens

    @staticmethod
    def scatter_rows_workspace_bytes(B):
        """Workspace of scatter_rows() on B rows (vfx_scatter_rows_workspace_bytes; no engine needed)."""
        return int(_lib.load().vfx_scatter_rows_workspace_bytes(int(B)))

    def scatter_rows(self, x, items):
        """Copies the rows of a batch into their own tensors in one launch (vfx_scatter_rows): row b of x (B, ldx), a
        float32 CUDA tensor with unit column stride, gives its samples [src_b, src_b + len_b) to dst_b.view(-1)[off_b :
        off_b + len_b].  items: one (dst_b, off_b, len_b) or (dst_b, off_b, len_b, src_b) per row, dst_b a contiguous
        float32 CUDA tensor on this device; src_b defaults to 0 (the row's first len_b samples).  The destination
        ranges must not overlap."""
        dev = torch.device(f"cuda:{self.device}")
        if not (x.is_cuda and x.device == dev and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1):
            raise ValueError(f"scatter_rows: x must be a (B, ldx) float32 tensor on {dev} with unit column stride")
        B = x.shape[0]
        if len(items) != B:
            raise ValueError(f"scatter_rows: {len(items)} items for {B} rows")
        table = (_lib.ScatterItem * B)()
        for b, (dst, off, n, *src_off) in enumerate(items):
            if not (dst.is_cuda and dst.device == dev and dst.dtype == torch.float32 and dst.is_contiguous()):
                raise ValueError(f"scatter_rows: item {b}: dst must be a contiguous float32 tensor on {dev}")
            t = table[b]
            t.dst, t.dst_elems, t.dst_off, t.len = dst.data_ptr(), dst.numel(), int(off), int(n)
            t.src_off = int(src_off[0]) if src_off else 0
        ws = self._workspace(self.scatter_rows_workspace_bytes(B))
        _lib.check(self.lib.vfx_scatter_rows(_ptr(x), B, x.stride(0), table, _ptr(ws), ws.numel(), _stream()),
                   "vfx_scatter_rows")

    @staticmethod
    def pack_pcm16_workspace_bytes(B):
        """Workspace of pack_pcm16() on B files (vfx_pack_pcm16_workspace_bytes; no engine needed)."""
        return int(_lib.load().vfx_pack_pcm16_workspace_bytes(int(B)))

    def pack_pcm16(self, files, y=None):
        """16-bit PCM of many files in one call (vfx_pack_pcm16): files is a list of lists of channels, each channel a
        float32 CUDA tensor on this device with n_i elements (contiguous), the same n_i for every channel of file i, 1 to
        PCM16_MAX_CHANNELS channels.  Returns (y, offsets): y an int16 CUDA tensor holding file i's interleaved (n_i, C_i)
        samples at y[offsets[i]:offsets[i + 1]], each file quantised as wavio.pcm16 quantises its (C_i, n_i) array, bit
        for bit.  y (optional): a contiguous int16 CUDA tensor of exactly sum n_i * C_i elements to write into."""
        dev = torch.device(f"cuda:{self.device}")
        B = len(files)
        if B == 0:
            raise ValueError("pack_pcm16 takes a non-empty list of files")
        table, offs = (_lib.Pcm16Item * B)(), [0]
        for b, rows in enumerate(files):
            rows = list(rows)
            if not 1 <= len(rows) <= _lib.PCM16_MAX_CHANNELS:
                raise ValueError(f"pack_pcm16: file {b} has {len(rows)} channels; 1 .. {_lib.PCM16_MAX_CHANNELS} are packed")
            n = rows[0].numel()
            for r in rows:
                if not (r.is_cuda and r.device == dev and r.dtype == torch.float32 and r.is_contiguous()
                        and r.numel() == n):
                    raise ValueError(f"pack_pcm16: file {b}: every channel must be a contiguous float32 tensor on {dev} "
                                     f"of the same length")
            t = table[b]
            for c, r in enumerate(rows):
                t.rows[c] = r.data_ptr()
            t.n, t.dst_off, t.C = n, offs[-1], len(rows)
            offs.append(offs[-1] + n * len(rows))
        if y is None:
            y = torch.empty(offs[-1], dtype=torch.int16, device=dev)
        elif not (y.is_cuda and y.device == dev and y.dtype == torch.int16 and y.is_contiguous() and y.numel() == offs[-1]):
            raise ValueError(f"pack_pcm16: y must be a contiguous int16 tensor of {offs[-1]} elements on {dev}")
        ws = self._workspace(self.pack_pcm16_workspace_bytes(B))
        _lib.check(self.lib.vfx_pack_pcm16(table, B, _ptr(y), y.numel(), _ptr(ws), ws.numel(), _stream()),
                   "vfx_pack_pcm16")
        return y, offs

    def hf_cut(self, wav, ratio=0.95, lens=None, out=None, lens_out=None, ws=None):
        """Mode-1 pre-filter: wav (B, L) -> (out (B, 512 * (L // 512)), cut bins (B,)).

        lens (ragged batch): int32 device tensor (B,); item b is the first lens[b] samples of row b and is filtered as if
        alone.  Returns (out (B, L), cut bins, lens_out): row b holds 512 * (lens[b] // 512) samples, then zeros, and
        lens_out (int32 device tensor) holds those lengths, ready for restore(..., lens=lens_out).

        out, lens_out (ragged batch only), ws (optional): caller-owned buffers to write the result, the lengths and the
        intermediate spectra into, instead of new ones and the engine's shared workspace (e.g. inside a captured graph,
        which must not bake in a workspace a later call may replace): a contiguous float32 CUDA tensor of the result's
        shape, a contiguous (B,) int32 CUDA tensor, and a uint8 CUDA tensor of at least hf_cut_workspace_bytes(B, L)."""
        wav = self._dev(wav)
        B, L = wav.shape
        cut = torch.empty(B, dtype=torch.int32, device=wav.device)
        if ws is None:
            ws = self._workspace(self.hf_cut_workspace_bytes(B, L))
        elif not (ws.is_cuda and ws.dtype == torch.uint8 and ws.numel() >= self.hf_cut_workspace_bytes(B, L)):
            raise ValueError(f"hf_cut: ws must be a uint8 CUDA tensor of at least {self.hf_cut_workspace_bytes(B, L)} bytes")
        shape = (B, L) if lens is not None else (B, 512 * (L // 512))
        if out is None:
            out = torch.empty(shape, device=wav.device)
        elif not (out.is_cuda and out.device == wav.device and out.dtype == torch.float32 and out.is_contiguous()
                  and tuple(out.shape) == shape):
            raise ValueError(f"hf_cut: out must be a contiguous float32 tensor of shape {shape} on {wav.device}")
        if lens is not None:
            _check_lens(lens, B)
            if lens_out is None:
                lens_out = torch.empty(B, dtype=torch.int32, device=wav.device)
            else:
                _check_lens(lens_out, B)
            _lib.check(self.lib.vfx_hf_cut_ragged(self.h, _ptr(wav), B, L, _ptr(lens), float(ratio), _ptr(out),
                                                  _ptr(lens_out), _ptr(cut), _ptr(ws), ws.numel(), _stream()),
                       "vfx_hf_cut_ragged")
            return out, cut, lens_out
        if lens_out is not None:
            raise ValueError("hf_cut: lens_out is the ragged batch's output lengths; it needs lens")
        _lib.check(self.lib.vfx_hf_cut(self.h, _ptr(wav), B, L, float(ratio), _ptr(out), _ptr(cut), _ptr(ws), ws.numel(),
                                       _stream()), "vfx_hf_cut")
        return out, cut


def _check_lens(lens, B):
    if not (lens.is_cuda and lens.dtype == torch.int32 and tuple(lens.shape) == (B,) and lens.is_contiguous()):
        raise ValueError(f"lens must be a contiguous int32 CUDA tensor of shape ({B},)")
