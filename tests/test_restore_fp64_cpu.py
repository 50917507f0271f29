"""The float64 oracle (no GPU): how far the fp32 oracle is from it, and whether the bounds of
tests/test_restore_fp64_gpu.py separate a correct restore path from one with a wiring fault.

1. The oracle run in float64 (float64 copies of the checkpoints, on the same float32 samples) against the oracle in
   fp32: restore in modes 0 / 1 / 2, the vocoder at odd and even T, and Vocoder.oracle.  This pins what fp32
   arithmetic costs on this path, which the GPU file's fp32 bounds must sit just above.
2. Sensitivity: the GPU file asserts E_engine / E_model within 1 +- DELTA for the tensor-core modes and fp32-level
   bounds for the fp32 mode.  Faults of the kind the kernel tests cannot see are put into the operand-rounding model
   (a tensor the engine keeps in fp32 stored in the operand format instead) or into the fp32 oracle (a BatchNorm eps),
   and each must fall outside the GPU file's band or bounds, with the same metric functions.  Where each falls against
   the older whole-path tolerances (tests/test_parity_gpu.py) is recorded beside it.
3. Calibration of tests/test_tc_seams_fp64_gpu.py: on each of its pooled sets, the rounding model with fp32 sums
   against the same model with float64 sums, three input seeds per format, within half that file's band.
4. Sensitivity of tests/test_tc_seams_fp64_gpu.py: operands left unrounded at one named rounding point of the model
   (OperandRounding.operand's `where`), and an item's end read one sample or frame early.

Each test records its statistics as pytest properties (written by --junitxml with -o junit_family=legacy).
"""
import contextlib

import numpy as np
import pytest
import torch

from test_restore_fp64_gpu import (DELTA, FP32_TOL, LENS, LENS_M2, VOC_T, WIN_FACTOR, _f64, _mask, pooled_rel_rms,
                                   rel_rms, worst_frame, worst_window)
from test_tc_seams_fp64_gpu import M2_DELTA, M2_UNPOOLED
from oracle import vf_oracle as O

SR, HOP = 44100, 441
# float64 oracle against the fp32 oracle, both metrics; measured 1.3e-6 .. 2.6e-6 (seeded, so these repeat)
FP64_FP32_TOL = 1e-5
# the whole-path tolerances of tests/test_parity_gpu.py (FULL_TOL), for the record
TODAY_TOL = {"fp32": 2e-4, "tf32": 2e-3, "fp16": 2e-3, "bf16": 3e-2}
FMTS = ["tf32", "fp16", "bf16"]


def _to(sd, dtype):
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}


@pytest.fixture(scope="module")
def st(states):
    return states[0], states[1], _to(states[0], torch.float64), _to(states[1], torch.float64)


def _utt(seconds, seed):
    from voicefixer_b200 import synthetic
    return synthetic.make_utterances(1, seconds=seconds, seed=seed)[0]


def _check(record_property, y32, y64):
    rel, win = rel_rms(y32, y64), worst_window(y32, y64)
    record_property("rel_rms", rel)
    record_property("worst_window", win)
    assert rel < FP64_FP32_TOL and win < FP64_FP32_TOL, f"fp32 oracle against float64: rel {rel:.3e}, window {win:.3e}"


# ============================================================================ 1. float64 oracle against fp32 oracle
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_restore_fp64_vs_fp32(st, mode, record_property):
    ana32, voc32, ana64, voc64 = st
    wav = _utt(0.7, 77)                                              # T = 71: mode 2 needs more than 64 frames
    if mode == 1:
        _, cut32 = O.remove_higher_frequency(wav, return_cut=True)
        _, cut64 = O.remove_higher_frequency(wav, dtype=np.float64, return_cut=True)
        record_property("cut_bin", cut32)
        assert cut32 == cut64, "the fp32 and float64 pre-filters cut at different bins"
    masks = _masks(1 + wav.shape[0] // HOP) if mode == 2 else None
    fn = (lambda T: masks) if mode == 2 else None
    y32 = O.restore_inmem(wav, ana32, voc32, mode=mode, drop_masks_fn=fn)
    y64 = O.restore_inmem(wav, ana64, voc64, mode=mode, drop_masks_fn=fn)
    assert y32.dtype == np.float32 and y64.dtype == np.float64 and y32.shape == y64.shape
    _check(record_property, y32, y64)


def _masks(T):
    return torch.rand(2, 1, T, 512, generator=torch.Generator().manual_seed(T)) >= 0.5


@pytest.mark.parametrize("T", [20, 21])
def test_vocoder_fp64_vs_fp32(st, T, record_property):
    ana32, voc32, _, voc64 = st
    mel = O.frontend(torch.from_numpy(_utt(0.6, 5)[: HOP * (T - 1) + 100])[None], ana32)[1]
    assert mel.shape[2] == T
    y32 = O.vocoder_forward(mel, voc32)
    y64 = O.vocoder_forward(mel.double(), voc64)
    assert y64.dtype == torch.float64 and y32.shape == y64.shape == (1, 1, (T + T % 2 + 4) * HOP)
    _check(record_property, y32, y64)


def test_oracle_wave_fp64_vs_fp32(st, record_property):
    _, voc32, _, voc64 = st
    wav = _utt(0.5, 9)
    y32, y64 = O.oracle_wave(wav, voc32), O.oracle_wave(wav, voc64)
    assert y32.dtype == np.float32 and y64.dtype == np.float64 and y32.shape == y64.shape
    _check(record_property, y32, y64)


# ============================================================================ 2. sensitivity of the GPU bounds
class _StoredInOperandFormat(O.OperandRounding):
    """Wiring fault: a tensor the engine keeps in fp32 ("vocoder.residual" or "unet.block") stored in the operand format."""

    def __init__(self, fmt, where):
        super().__init__(fmt)
        self.where = where

    def stored(self, x, where):
        return self.round(x) if where == self.where else x


class _Sens:
    """restore mode 0 of one 1 s utterance in float64: the plain oracle, and the rounding model with or without a fault"""

    def __init__(self, ana64, voc64):
        self.ana, self.voc, self.wav, self.cache = ana64, voc64, _utt(1.0, 1234), {}
        self.ref = self.run(None)

    def run(self, model):
        if model is None:
            return O.restore_inmem(self.wav, self.ana, self.voc, mode=0)
        with O.operand_rounding(model):
            return O.restore_inmem(self.wav, self.ana, self.voc, mode=0)

    def error(self, fmt, where=None):
        key = (fmt, where)
        if key not in self.cache:
            y = self.run(fmt if where is None else _StoredInOperandFormat(fmt, where))
            self.cache[key] = (rel_rms(y, self.ref), worst_window(y, self.ref))
        return self.cache[key]


@pytest.fixture(scope="module")
def sens(st):
    return _Sens(st[2], st[3])


def _fault_ratio(sens, fmt, where, record_property):
    e_model, w_model = sens.error(fmt)
    e_fault, w_fault = sens.error(fmt, where)
    ratio = e_fault / e_model
    record_property("E_model", e_model)
    record_property("E_fault", e_fault)
    record_property("ratio", ratio)
    record_property("worst_window_ratio", w_fault / w_model)
    record_property("outside_band", not (1 - DELTA <= ratio <= 1 + DELTA))
    record_property("passes_parity_tolerance", e_fault < TODAY_TOL[fmt])
    return ratio


@pytest.mark.parametrize("fmt", FMTS)
def test_resstack_residual_in_operand_format_is_outside_band(sens, fmt, record_property):
    """The vocoder's ResStack stream x kept in the operand format: what the tf32 encoded stream and the 16-bit pair
    outputs exist to avoid.  About x1.23 .. x1.25 in every format; in bf16 it stays under the parity tolerance (3e-2)."""
    ratio = _fault_ratio(sens, fmt, "vocoder.residual", record_property)
    assert not (1 - DELTA <= ratio <= 1 + DELTA), f"{fmt}: the fault gives E / E_model = {ratio:.4f}, inside the band"


@pytest.mark.parametrize("fmt", FMTS)
def test_unet_block_outputs_in_operand_format_recorded(sens, fmt, record_property):
    """Every UNet ConvBlockRes output kept in the operand format: about x1.07 .. x1.09, so near the band's edge; the
    ratio and which side of the band it falls on are recorded, not asserted."""
    ratio = _fault_ratio(sens, fmt, "unet.block", record_property)
    assert ratio > 1.0


def test_bn_eps_fault_is_outside_fp32_bounds(sens, st, monkeypatch, record_property):
    """An fp32 path with every BatchNorm's eps at 2e-5 instead of 1e-5 (fp32 arithmetic otherwise)."""
    ana32, voc32 = st[0], st[1]
    y_ok = O.restore_inmem(sens.wav, ana32, voc32, mode=0)
    monkeypatch.setattr(O, "BN_EPS", 2e-5)
    y = O.restore_inmem(sens.wav, ana32, voc32, mode=0)
    rel, win = rel_rms(y, sens.ref), worst_window(y, sens.ref)
    record_property("correct_rel_rms", rel_rms(y_ok, sens.ref))
    record_property("correct_worst_window", worst_window(y_ok, sens.ref))
    record_property("fault_rel_rms", rel)
    record_property("fault_worst_window", win)
    record_property("passes_parity_tolerance", rel < TODAY_TOL["fp32"])
    tol = FP32_TOL["restore"]
    assert rel_rms(y_ok, sens.ref) < tol and worst_window(y_ok, sens.ref) < tol
    assert rel > tol or win > tol, f"the fault gives rel {rel:.3e}, window {win:.3e}"


# ============================================================================ 3. calibration of the seams' band
# tests/test_tc_seams_fp64_gpu.py asserts E_engine / E_model within 1 +- DELTA, pooled over each set of items below.
# Here the engine is stood in for by the rounding model with fp32 sums (fp32 checkpoints), which rounds the same
# operands and sums in another precision, as the engine's kernels sum in another order; for three input seeds per
# format its pooled ratio to the float64-sum model must stay within 1 +- DELTA / 2, so that the GPU band is not flaky by
# construction (the mode-2 pools: within 1 +- M2_DELTA / 2, see M2_DELTA).  For run time, the 10 s item of LENS is
# left out of the sets whose pool does not need it (it is no edge: they keep every padding and L % 441 edge), and
# shortened to 3 s in the restore mode-2 set, where it dilutes the ill-conditioned T = 129 item; the 10 s and 33 s
# restores of the GPU file (engine options, two segments) are stood in for by one 1 s restore in mode 0.  Seed 1 is the
# GPU file's input (_item, _item_mask, _voc_mel).
CAL_SEEDS = (1, 2, 3)
_M2_POOL = [L for L in LENS_M2 if L != M2_UNPOOLED]
CAL_SETS = {
    "analysis_mode0": LENS[:-1],
    "analysis_mode2": _M2_POOL,
    "vocoder": VOC_T,
    "oracle": LENS[:-1],
    "restore_mode1": LENS[1:-1],
    "restore_mode2": _M2_POOL[:-1] + [441 * 300],
    "restore_mode0": [SR],
}


def _band(name):
    return M2_DELTA if name.endswith("mode2") else DELTA


def _cal_item(L, seed):
    from voicefixer_b200 import synthetic
    return synthetic.make_utterances(1, seconds=L / SR + 0.01, seed=L % 9973 + seed)[0, :L].copy()


def _cal_mask(L, seed):
    return _mask(1 + L // HOP, L + 1000 * (seed - 1))


def _seam(name, n, seed, ana, voc, fe):
    """item n of set `name` for input seed `seed`, in the dtype of (ana, voc); the vocoder and analysis read the fp32
    mel of the front end `fe` (fp32 checkpoints), as the GPU file's do"""
    dt = ana["mel.fb"].dtype
    if name == "vocoder":
        mel = O.frontend(torch.from_numpy(_cal_item(SR, seed))[None], fe)[1]
        return O.vocoder_forward(mel[:, :, :n].to(dt), voc)
    wav = _cal_item(n, seed)
    if name.startswith("analysis"):
        mel = O.frontend(torch.from_numpy(wav)[None], fe)[1]
        train = name == "analysis_mode2"
        return O.analysis(mel.to(dt), ana, train, _cal_mask(n, seed) if train else None)[0, 0]
    if name == "oracle":
        return O.oracle_wave(wav, voc)
    mode = int(name[-1])
    fn = (lambda T: _cal_mask(n, seed)) if mode == 2 else None
    return O.restore_inmem(wav, ana, voc, mode=mode, drop_masks_fn=fn)


class _Cal:
    """each set's items in float64, under the rounding model with float64 sums, and with fp32 sums (or a fault model)"""

    def __init__(self, st):
        self.st, self.cache = st, {}

    def items(self, name, seed, rounding=None, sums="float64"):
        key = (name, seed, rounding, sums)
        if key not in self.cache:
            ana, voc = (self.st[2], self.st[3]) if sums == "float64" else (self.st[0], self.st[1])
            model = O.operand_rounding(rounding) if rounding is not None else contextlib.nullcontext()
            with torch.no_grad(), model:
                self.cache[key] = [_f64(_seam(name, n, seed, ana, voc, self.st[0])) for n in CAL_SETS[name]]
        return self.cache[key]


@pytest.fixture(scope="module")
def cal(st):
    return _Cal(st)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("name", list(CAL_SETS))
def test_seam_band_calibration(cal, name, fmt, record_property):
    ratios = []
    for seed in CAL_SEEDS:
        ref = cal.items(name, seed)
        e64 = pooled_rel_rms(cal.items(name, seed, fmt), ref)
        e32 = pooled_rel_rms(cal.items(name, seed, fmt, sums="fp32"), ref)
        record_property(f"seed{seed}_E_model", e64)
        record_property(f"seed{seed}_ratio", e32 / e64)
        ratios.append(e32 / e64)
    record_property("spread", f"{min(ratios):.4f} .. {max(ratios):.4f}")
    record_property("half_band", _band(name) / 2)
    assert all(abs(r - 1) <= _band(name) / 2 for r in ratios), f"{name} {fmt}: fp32-sum / float64-sum model = {ratios}"


# ============================================================================ 4. sensitivity of the seams' checks
# Faults only the tensor-core seams can have, put into the float64-sum model of one set (seed 1, the GPU file's input),
# against the correct model with the GPU file's two checks: the pooled ratio against 1 +- DELTA, and each item's worst
# window / frame against WIN_FACTOR x the model's.
class _LeftUnrounded(O.OperandRounding):
    """Wiring fault: the operands at the rounding points `where` left in fp32 (a layer that silently runs unrounded)."""

    def __init__(self, fmt, where):
        super().__init__(fmt)
        self.where = where

    def operand(self, x, where):
        return x if where in self.where else self.round(x)


def _unrounded_ratio(cal, name, fmt, where, record_property):
    ref = cal.items(name, 1)
    e_model = pooled_rel_rms(cal.items(name, 1, fmt), ref)
    e_fault = pooled_rel_rms(cal.items(name, 1, _LeftUnrounded(fmt, where)), ref)
    ratio = e_fault / e_model
    record_property("E_model", e_model)
    record_property("E_fault", e_fault)
    record_property("ratio", ratio)
    record_property("outside_band", not (1 - _band(name) <= ratio <= 1 + _band(name)))
    return ratio


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("name", ["vocoder", "oracle"])
def test_vocoder_conditions_unrounded_recorded(cal, name, fmt, record_property):
    """The conditions condnet.0 reads (voc_normalize's output, or the oracle front end's) left in fp32: the input of one
    of the vocoder's 74 convolutions, about x0.985 .. x0.991 in every format, inside the band; recorded, and asserted
    only on the side it falls on."""
    ratio = _unrounded_ratio(cal, name, fmt, ("vocoder.cond",), record_property)
    assert ratio < 1.0


@pytest.mark.parametrize("fmt", FMTS)
def test_mode2_bn_act_unrounded_is_below_band(cal, fmt, record_property):
    """Mode 2: the UNet conv blocks' operands written by bn_act (train-mode statistics, nothing folded) left in fp32:
    about x0.77 .. x0.81."""
    ratio = _unrounded_ratio(cal, "analysis_mode2", fmt, ("unet.bn_act",), record_property)
    assert ratio < 1 - M2_DELTA, f"{fmt}: the fault gives E / E_model = {ratio:.4f}, not below the band"


@pytest.mark.parametrize("fmt", FMTS)
def test_gru_input_projections_unrounded_recorded(cal, fmt, record_property):
    """The GRU input projections (bn(x) or layer 0's output, and w_ih) left in fp32: the denoiser's mask carries a
    small part of the log-mel's error (6.5e-5 of 1.2e-3 in tf32), and the fault moves the pooled error by x0.993 ..
    x1.005, inside the band; recorded, and asserted only to change the result."""
    ratio = _unrounded_ratio(cal, "analysis_mode0", fmt, ("gru.input", "gru.weight"), record_property)
    assert ratio != 1.0


def _end_fault(y, log_mel):
    """Wiring fault at an item's end: its last frame, or its last 441 samples, read one frame / sample early"""
    y = y.copy()
    if log_mel:
        y = y.reshape(-1, 128)
        y[-1] = y[-2]
        return y.reshape(-1)
    y[-HOP:] = y[-HOP - 1:-1]
    return y


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("name", list(CAL_SETS))
def test_error_at_item_end_fails_worst_window(cal, name, fmt, record_property):
    """The fault on each item of the set in turn: the item's worst window / frame must exceed WIN_FACTOR x the model's
    (it gives x19 .. x1120).  Whether the pooled ratio catches it too is recorded (x1.25 .. x115)."""
    log_mel = name.startswith("analysis")
    loc = worst_frame if log_mel else worst_window
    ref, model = cal.items(name, 1), cal.items(name, 1, fmt)
    e_model = pooled_rel_rms(model, ref)
    for k, n in enumerate(CAL_SETS[name]):
        faulty = list(model)
        faulty[k] = _end_fault(model[k], log_mel)
        ratio = pooled_rel_rms(faulty, ref) / e_model
        w_fault, w_model = loc(faulty[k], ref[k]), loc(model[k], ref[k])
        record_property(f"n{n}_pooled_ratio", ratio)
        record_property(f"n{n}_worst_ratio", w_fault / w_model)
        assert w_fault > WIN_FACTOR * w_model, f"{name} {fmt} n = {n}: worst {w_fault:.3e}, the model's {w_model:.3e}"
