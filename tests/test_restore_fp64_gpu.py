"""The whole restore path (every seam of the engine, ~360 launches) against the float64 oracle.

The kernel tests compare each kernel with a float64 reference of its own; what they cannot see is how the launches
are put together: which tensor stays fp32 and which is stored in the operand format, where the eval BatchNorms are
folded, which skip / residual / concat buffer a layer reads and which extents each level uses for each ragged item.
Here the engine's outputs are compared with the oracle run in float64 on the GPU (oracle.vf_oracle on float64 copies
of the checkpoints, on the float32 samples the engine reads; float64 has no TF32 path):

  A. precision "fp32": the engine against the float64 oracle, at fp32-level bounds, on every seam (analysis in modes
     0 / 2, vocoder, oracle, restore in modes 0 / 1 / 2), at the lengths where the UNet padding, the frame count and
     the last window change, in ragged batches (each row against its own item's reference) and through restore_many
     on a recording that spans two 30 s segments.
  B. "tf32" / "fp16" / "bf16": a tight comparison cannot work (a flipped rounding costs a whole operand step, and
     two runs that round differently become independent draws of rounding noise), but the size of the error is
     stable.  So the engine's error against float64 must equal, within DELTA, the error of the oracle's operand
     rounding model (vf_oracle.operand_rounding, float64 sums) against float64: from above and from below (a layer
     that silently ran in fp32 breaks the contract too).

Metrics, each over one item's own length: whole-item relative RMS; for waveforms the worst 441-sample (10 ms) window
of the error, divided by the item's RMS; for log-mel the worst frame, divided by the RMS of that frame.  An error
confined to an item's end, a padding boundary or one frame is averaged away in the first and not in the others.

Thresholds are at least 3x the worst value measured on an H100 80GB HBM3 (700 W power limit); every input is seeded,
so those values repeat.  Each test records its statistics as pytest properties (written by --junitxml with
-o junit_family=legacy).  tests/test_restore_fp64_cpu.py checks on the CPU that these bounds separate a correct
path from a path with a wiring fault.
"""
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, HOP, WIN = 44100, 441, 441

# A. fp32 engine against the float64 oracle: one bound per seam for both metrics (relative RMS, and worst window or
# frame).  The fp32 oracle itself is 1.3e-6 .. 3.0e-6 from float64 on most inputs (tests/test_restore_fp64_cpu.py).
FP32_TOL = {
    # log-mel, modes 0 and 2: measured worst 2.5e-6 relative RMS, 3.2e-6 worst frame (mode 2, T = 128)
    "analysis": 1e-5,
    # vocoder and oracle waveforms, single and ragged: measured worst 2.7e-6 / 3.1e-6
    "vocoder": 1e-5,
    # restore mode 0, single, ragged and restore_many: measured worst 3.4e-6 / 3.8e-6 (T = 1001)
    "restore": 1.2e-5,
    # restore modes 1 and 2: measured worst 6.7e-6 / 8.9e-6.  Some inputs are ill-conditioned in these modes, and the
    # same arithmetic in torch fp32 does no better: on the mode-2 item at T = 128 (train-mode statistics over a 2 x 1
    # UNet centre) the fp32 oracle is 1.7e-5 / 2.4e-5 from float64 where the engine is 6.6e-6 / 8.9e-6, and on the
    # mode-1 item at T = 64 it is 5.3e-6 / 8.4e-6 where the engine is 5.6e-6 / 6.9e-6.
    "restore_m12": 3e-5,
}
# B. tensor-core modes: E_engine / E_model in [1 - DELTA, 1 + DELTA].  The spread of that ratio, measured on the CPU as
# the rounding model with fp32 sums against the same model with float64 sums (0.7 s and 1.6 s, 3 seeds each, tf32 /
# fp16 / bf16): 0.990 .. 1.011; on the H100 the engine gives 0.995 .. 0.999.  A ResStack residual stream stored in the
# operand format gives 1.23 .. 1.25 (tests/test_restore_fp64_cpu.py).
DELTA = 0.05
# every ragged item: the engine's worst window <= WIN_FACTOR x the model's worst window; measured worst 1.08 (fp16)
WIN_FACTOR = 3.0
TC_PRECS = ["tf32", "fp16", "bf16"]

# restore / oracle lengths: T = 3 (L = 1025), T = 63 / 64 / 65 (the UNet pads to 64 / 64 / 128 frames), T = 128 / 129
# (the padding 128 -> 192), T = 1001 (10 s); L % 441 is 0 or 440 in all but the first
LENS = [1025, 441 * 62, 441 * 64 - 1, 441 * 64, 441 * 128 - 1, 441 * 128, 441 * 1000]
LENS_M2 = [L for L in LENS if 1 + L // HOP > 64]         # train-mode BN needs more than 64 frames
VOC_T = [1, 2, 3, 20, 65]


# ---------------------------------------------------------------------------- metrics (shared with the CPU file)
def _f64(a):
    return np.asarray(a.detach().cpu().numpy() if torch.is_tensor(a) else a, np.float64).reshape(-1)


def rel_rms(y, ref):
    y, ref = _f64(y), _f64(ref)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    return float(np.sqrt(np.mean((y - ref) ** 2)) / np.sqrt(np.mean(ref ** 2)))


def worst_window(y, ref, win=WIN):
    """max over consecutive win-sample windows (the last one partial) of rms(y - ref), / rms(ref) of the item"""
    y, ref = _f64(y), _f64(ref)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    n = ref.shape[0]
    k = -(-n // win)
    e2 = np.zeros(k * win)
    e2[:n] = (y - ref) ** 2
    cnt = np.full(k, float(win))
    cnt[-1] = n - (k - 1) * win
    return float(np.sqrt(np.max(e2.reshape(k, win).sum(1) / cnt)) / np.sqrt(np.mean(ref ** 2)))


def worst_frame(y, ref):
    """log-mel (T, 128): max over frames of rms(y - ref) / rms(ref) of that frame"""
    y, ref = _f64(y).reshape(-1, 128), _f64(ref).reshape(-1, 128)
    assert y.shape == ref.shape
    return float(np.max(np.sqrt(np.mean((y - ref) ** 2, 1)) / np.sqrt(np.mean(ref ** 2, 1))))


def pooled_rel_rms(ys, refs):
    num = sum(float(np.sum((_f64(y) - _f64(r)) ** 2)) for y, r in zip(ys, refs))
    return float(np.sqrt(num / sum(float(np.sum(_f64(r) ** 2)) for r in refs)))


def check_fp32(record_property, seam, tag, y, ref):
    log_mel = seam == "analysis"
    rel = rel_rms(y, ref)
    loc = worst_frame(y, ref) if log_mel else worst_window(y, ref)
    record_property(f"{tag}rel_rms", rel)
    record_property(f"{tag}{'worst_frame' if log_mel else 'worst_window'}", loc)
    record_property(f"{tag}tolerance", FP32_TOL[seam])
    assert rel < FP32_TOL[seam], f"{tag}relative RMS {rel:.3e} against float64"
    assert loc < FP32_TOL[seam], f"{tag}worst {'frame' if log_mel else 'window'} {loc:.3e} against float64"


def check_ratio(record_property, tag, e_engine, e_model, delta=DELTA):
    ratio = e_engine / e_model
    record_property(f"{tag}E_engine", e_engine)
    record_property(f"{tag}E_model", e_model)
    record_property(f"{tag}ratio", ratio)
    record_property(f"{tag}delta", delta)
    assert 1 - delta <= ratio <= 1 + delta, \
        f"{tag}E_engine / E_model = {e_engine:.4e} / {e_model:.4e} = {ratio:.4f}, outside 1 +- {delta}"


# ---------------------------------------------------------------------------- inputs and float64 references
@functools.lru_cache(maxsize=None)
def _item(L):
    """a seeded float32 utterance of L samples (read only)"""
    from voicefixer_b200 import synthetic
    return synthetic.make_utterances(1, seconds=L / SR + 0.01, seed=L % 9973 + 1)[0, :L].copy()


def _mask(T, seed):
    """(2, 1, T, 512) dropout keep-masks"""
    return torch.rand(2, 1, T, 512, generator=torch.Generator().manual_seed(seed)) >= 0.5


def _item_mask(L):
    return _mask(1 + L // HOP, L)


@functools.lru_cache(maxsize=None)
def _mel(L):
    """the fp32 linear mel (T, 128) of _item(L), T = 1 + L // 441 (read only)"""
    from oracle import vf_oracle as O
    return O.frontend(torch.from_numpy(_item(L))[None], _fe_state())[1][0, 0]


@functools.lru_cache(maxsize=None)
def _voc_mel(T):
    """the vocoder's input of T frames: the first T frames of a 1 s utterance's mel (read only)"""
    return _mel(SR)[:T]


@functools.lru_cache(maxsize=None)
def _fe_state():
    from voicefixer_b200 import synthetic
    sd = synthetic.make_analysis_state(0)
    return {k: sd[k] for k in ("f_helper.stft.conv_real.weight", "f_helper.stft.conv_imag.weight", "mel.fb")}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a))[None].to(DEV)


_ENGINES = {}


def _engine(states, prec):
    if prec not in _ENGINES:
        from voicefixer_b200.engine import Engine
        _ENGINES[prec] = Engine(states[0], states[1], precision=prec)
    return _ENGINES[prec]


@pytest.fixture(scope="module")
def states64(states):
    return tuple({k: (v.to(DEV, torch.float64) if v.is_floating_point() else v) for k, v in sd.items()} for sd in states)


class Refs:
    """float64 oracle results, computed once per module"""

    def __init__(self, ana, voc):
        self.ana, self.voc, self.cache = ana, voc, {}

    def _get(self, key, fn, rounding=None):
        """fn() in float64, or under the operand-rounding model `rounding` (a format name or an OperandRounding)"""
        from oracle import vf_oracle as O
        key = key + (rounding,)
        if key not in self.cache:
            with torch.no_grad():
                if rounding is None:
                    self.cache[key] = _f64(fn())
                else:
                    with O.operand_rounding(rounding):
                        self.cache[key] = _f64(fn())
        return self.cache[key]

    def restore(self, L, mode=0, rounding=None):
        from oracle import vf_oracle as O
        masks = (lambda T: _item_mask(L)) if mode == 2 else None
        return self._get(("restore", L, mode), lambda: O.restore_inmem(_item(L), self.ana, self.voc, mode=mode,
                                                                       drop_masks_fn=masks), rounding)

    def analysis(self, L, mode, rounding=None):
        from oracle import vf_oracle as O
        masks = _item_mask(L) if mode == 2 else None
        return self._get(("analysis", L, mode), lambda: O.analysis(
            _mel(L).to(DEV, torch.float64)[None, None], self.ana, mode == 2, masks)[0, 0], rounding).reshape(-1, 128)

    def vocoder(self, T, rounding=None):
        from oracle import vf_oracle as O
        return self._get(("vocoder", T), lambda: O.vocoder_forward(_voc_mel(T).to(DEV, torch.float64)[None, None],
                                                                   self.voc), rounding)

    def oracle(self, L, rounding=None):
        from oracle import vf_oracle as O
        return self._get(("oracle", L), lambda: O.oracle_wave(_item(L), self.voc) / 2 ** 15, rounding)


@pytest.fixture(scope="module")
def refs(states64):
    return Refs(*states64)


def _batch(items, L_cap):
    x = torch.zeros(len(items), L_cap, device=DEV)
    for i, a in enumerate(items):
        x[i, :a.shape[0]] = torch.from_numpy(a).to(DEV)
    return x, torch.tensor([a.shape[0] for a in items], dtype=torch.int32, device=DEV)


def _ragged_masks(lens):
    T_cap = 1 + max(lens) // HOP
    m = torch.zeros(2, len(lens), T_cap, 512, dtype=torch.bool)
    for b, L in enumerate(lens):
        m[:, b, :1 + L // HOP] = _item_mask(L)[:, 0]
    return m


def _check_tail_zero(y, n, what):
    assert bool((y[n:] == 0).all()), f"{what}: samples past the item's length are not zero"


# ============================================================================ A. fp32 engine against float64
@pytest.mark.parametrize("mode,L", [(0, L) for L in LENS] + [(2, L) for L in LENS_M2])
def test_analysis_fp32(states, refs, mode, L, record_property):
    eng = _engine(states, "fp32")
    masks = _item_mask(L) if mode == 2 else None
    y = eng.analysis(_mel(L)[None], mode=mode, drop_masks=masks)[0]
    check_fp32(record_property, "analysis", "", y, refs.analysis(L, mode))


@pytest.mark.parametrize("T", VOC_T)
def test_vocoder_fp32(states, refs, T, record_property):
    y = _engine(states, "fp32").vocoder(_voc_mel(T)[None])[0]
    assert y.shape[0] == (T + T % 2 + 4) * HOP
    check_fp32(record_property, "vocoder", "", y, refs.vocoder(T))


def test_vocoder_ragged_fp32(states, refs, record_property):
    T_cap = max(VOC_T)
    mel = torch.zeros(len(VOC_T), T_cap, 128)
    for b, T in enumerate(VOC_T):
        mel[b, :T] = _voc_mel(T)
    frames = torch.tensor(VOC_T, dtype=torch.int32, device=DEV)
    y = _engine(states, "fp32").vocoder(mel, lens=frames)
    for b, T in enumerate(VOC_T):
        n = (T + T % 2 + 4) * HOP
        check_fp32(record_property, "vocoder", f"T{T}_", y[b, :n], refs.vocoder(T))
        _check_tail_zero(y[b], n, f"vocoder T = {T}")


@pytest.mark.parametrize("L", LENS)
def test_oracle_fp32(states, refs, L, record_property):
    T = 1 + L // HOP
    y = _engine(states, "fp32").oracle(_dev(_item(L)))[0]
    assert y.shape[0] == (T + T % 2 + 4) * HOP
    check_fp32(record_property, "vocoder", "", y, refs.oracle(L))


def test_oracle_ragged_fp32(states, refs, record_property):
    x, lens = _batch([_item(L) for L in LENS], max(LENS))
    y = _engine(states, "fp32").oracle(x, lens=lens)
    for b, L in enumerate(LENS):
        T = 1 + L // HOP
        n = (T + T % 2 + 4) * HOP
        check_fp32(record_property, "vocoder", f"L{L}_", y[b, :n], refs.oracle(L))
        _check_tail_zero(y[b], n, f"oracle L = {L}")


@pytest.mark.parametrize("mode,L", [(0, L) for L in LENS] + [(1, L) for L in LENS[1:]] + [(2, L) for L in LENS_M2])
def test_restore_fp32(states, refs, mode, L, record_property):
    eng = _engine(states, "fp32")
    wav = _item(L)
    if mode == 1:
        from voicefixer_b200.api import VoiceFixer
        from oracle import vf_oracle as O
        # the cut bin: the fp32 and float64 pre-filters must agree, or the comparison below measures that instead
        _, cut32 = O.remove_higher_frequency(wav, return_cut=True)
        _, cut64 = O.remove_higher_frequency(wav, dtype=np.float64, return_cut=True)
        assert cut32 == cut64
        y = VoiceFixer.from_engine(eng).restore_inmem(wav, cuda=True, mode=1)[0]
    else:
        y = eng.restore(_dev(wav), mode=mode, drop_masks=_item_mask(L) if mode == 2 else None)[0]
    check_fp32(record_property, "restore" if mode == 0 else "restore_m12", "", y, refs.restore(L, mode))


@pytest.mark.parametrize("mode", [0, 2])
def test_restore_ragged_fp32(states, refs, mode, record_property):
    lens = LENS if mode == 0 else LENS_M2
    x, lens_t = _batch([_item(L) for L in lens], max(lens))
    y = _engine(states, "fp32").restore(x, mode=mode, drop_masks=_ragged_masks(lens) if mode == 2 else None, lens=lens_t)
    for b, L in enumerate(lens):
        check_fp32(record_property, "restore" if mode == 0 else "restore_m12", f"L{L}_", y[b, :L], refs.restore(L, mode))
        _check_tail_zero(y[b], L, f"restore mode {mode} L = {L}")


@pytest.mark.timeout(900)
def test_restore_many_two_segments_fp32(states, states64, record_property):
    """33 s: one full 30 s segment and a 3 s one, cut, restored and joined by restore_many."""
    from voicefixer_b200.api import VoiceFixer
    from oracle import vf_oracle as O
    wav = _item(33 * SR)
    y = VoiceFixer.from_engine(_engine(states, "fp32")).restore_many([wav])[0][0]
    with torch.no_grad():
        ref = _f64(O.restore_inmem(wav, *states64, mode=0))
    seg = 30 * SR
    record_property("segment0_rel_rms", rel_rms(y[:seg], ref[:seg]))
    record_property("segment1_rel_rms", rel_rms(y[seg:], ref[seg:]))
    check_fp32(record_property, "restore", "", y, ref)
    assert rel_rms(y[seg:], ref[seg:]) < FP32_TOL["restore"]


# ============================================================================ B. tensor-core modes against the model
@pytest.mark.parametrize("prec", TC_PRECS)
def test_restore_10s_tensor_core_vs_rounding_model(states, refs, prec, record_property):
    L = LENS[-1]
    y = _engine(states, prec).restore(_dev(_item(L)))[0]
    ref, model = refs.restore(L), refs.restore(L, rounding=prec)
    check_ratio(record_property, "", rel_rms(y, ref), rel_rms(model, ref))
    w_e, w_m = worst_window(y, ref), worst_window(model, ref)
    record_property("worst_window_engine", w_e)
    record_property("worst_window_model", w_m)
    assert w_e <= WIN_FACTOR * w_m


@pytest.mark.parametrize("prec", TC_PRECS)
def test_restore_ragged_tensor_core_vs_rounding_model(states, refs, prec, record_property):
    x, lens_t = _batch([_item(L) for L in LENS], max(LENS))
    y = _engine(states, prec).restore(x, lens=lens_t)
    ys, refs64, models = [], [], []
    for b, L in enumerate(LENS):
        ys.append(y[b, :L])
        refs64.append(refs.restore(L))
        models.append(refs.restore(L, rounding=prec))
        _check_tail_zero(y[b], L, f"{prec} L = {L}")
    check_ratio(record_property, "pooled_", pooled_rel_rms(ys, refs64), pooled_rel_rms(models, refs64))
    for L, yb, rb, mb in zip(LENS, ys, refs64, models):
        w_e, w_m = worst_window(yb, rb), worst_window(mb, rb)
        record_property(f"L{L}_worst_window_engine", w_e)
        record_property(f"L{L}_worst_window_model", w_m)
        assert w_e <= WIN_FACTOR * w_m, f"L = {L}: worst window {w_e:.3e} against the model's {w_m:.3e}"
