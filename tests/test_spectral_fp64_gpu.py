"""The kernels built on the shared FFT (csrc/fft.cuh) against float64 references of the same operation: the restore
front end (vfx_frontend_mel), the mode-1 pre-filter (vfx_hf_cut, vfx_hf_cut_ragged) and the front end of
Vocoder.oracle (vfx_oracle_cond, and the operand-format conditions inside vfx_oracle).

The other tests compare these kernels with fp32 results over whole signals, so an error confined to a few hundred
samples, one bin or the edge of a frame passes them.  Here every reference is computed in float64 on the float32
operands the kernel reads (the wav, the engine's float32 Hann values, the mel basis it was given), and the error is
measured locally: per frame or per sample, normalised by the RMS of that frame or item.  Outputs start NaN-filled, so
memory a kernel fails to write is caught.  The thresholds are at least 3x the worst value measured on an H100 80GB
HBM3 (700 W power limit); every input is seeded, so those values repeat.  Each test records its statistics as pytest
properties (written by --junitxml with -o junit_family=legacy).
"""
import ctypes
import math
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
NAN = float("nan")
SR = 44100
SEG = 30 * SR                           # one 30 s segment of restore_inmem / restore_many
DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "tf32": torch.float32}

# A. restore front end.  Per frame: max_k |sp - sp64| / rms_k(sp64); measured worst 5.6e-6 (30 s, tone halfway
# between bins: the frame's energy sits in two bins, so its RMS is small against the peak's rounding).
SP_FRAME_TOL = 2e-5
# whole tensor: relative RMS of sp; measured worst 1.4e-7 (L = 1323, impulse at L - 1)
SP_REL_TOL = 5e-7
# per element: |mel - mel64| / rms(mel64 of the frame); measured worst 6.8e-6 (dense random basis, tone halfway)
MEL_FRAME_TOL = 2.5e-5
# B. mode-1 pre-filter: max |y - y64| / rms(y64) in every region of the item; measured worst 1.24e-6 (middle of a 30 s
# segment of white noise; [512, 1024): 7.9e-7).  With the truncating overlap-add index, [512, 1024) was 9e-4 .. 9e-3.
HF_TOL = 4e-6
# the cut bin must satisfy the float64 decision up to this fraction of the total energy (see _check_cut).  Measured:
# the cut always equals the float64 one; the nearest partial sum lay 1.6e-6 x total from the threshold.
CUT_MARGIN = 1e-6
# C. oracle front end, fp32 conditions: max |cond - cond64|; measured worst 3.1e-7.  A float32 window product gives
# 4.9e-4 on the 1 kHz tone, a float32 FFT 3.3e-3.
ORACLE_TOL = 1e-6


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from voicefixer_b200 import _lib
    _lib.check(rc, what)


def _hann32():
    """the engine's window: periodic Hann computed in double and rounded to float32 (engine.cu)"""
    n = torch.arange(2048, dtype=F64)
    return (0.5 - 0.5 * torch.cos(2 * math.pi * n / 2048)).float().to(DEV)


def _signal(kind, L, seed):
    """float32 (L,) test signals"""
    g = np.random.default_rng(seed)
    n = np.arange(L, dtype=np.float64)
    if kind == "noise":
        x = 0.5 * g.standard_normal(L)
    elif kind == "tone_on":                        # exactly on bin 100 of the 2048-point transform
        x = 0.8 * np.sin(2 * np.pi * 100.0 * n / 2048 + 0.3)
    elif kind == "tone_half":                      # halfway between bins 100 and 101: Z[k], Z[1024 - k] nearly cancel
        x = 0.8 * np.sin(2 * np.pi * 100.5 * n / 2048 + 0.3)
    elif kind == "dc":
        x = np.full(L, 0.7)
    elif kind == "alt":                            # +-1 alternation: all energy in the Nyquist bin
        x = 0.6 * (1.0 - 2.0 * (n % 2))
    elif kind == "imp0":
        x = np.zeros(L)
        x[0] = 1.0
    elif kind == "impL":
        x = np.zeros(L)
        x[L - 1] = 1.0
    elif kind == "zeros":
        x = np.zeros(L)
    elif kind == "utt":
        from voicefixer_b200 import synthetic
        x = synthetic.make_utterances(1, seconds=L / SR + 0.01, seed=seed)[0, :L]
    elif kind.startswith("white"):                 # white_0.1, white_3
        x = float(kind.split("_")[1]) * g.standard_normal(L)
    elif kind == "lowpass":                        # white noise with nothing above bin 100 of the STFT
        X = np.fft.rfft(g.standard_normal(L))
        X[int(100 / 2048 * L):] = 0
        x = np.fft.irfft(X, n=L)
        x *= 0.3 / max(float(np.sqrt(np.mean(x ** 2))), 1e-30)
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(x, dtype=np.float32)


def _frame_err(got, ref):
    """per row (last axis): max |got - ref| / rms(ref)"""
    return (got.to(F64) - ref).abs().amax(-1) / ref.pow(2).mean(-1).sqrt()


def _rel(got, ref):
    got, ref = got.to(F64), ref.to(F64)
    return float((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())


# ============================================================================ A. restore front end
_FE = {}


def _fe_engine(states, basis):
    """an fp32 engine whose mel.fb (1025, 128) is `basis` ("model": the checkpoint's own)"""
    if basis not in _FE:
        from voicefixer_b200.engine import Engine
        ana = dict(states[0])
        fb = ana["mel.fb"].float().clone()
        g = torch.Generator().manual_seed(7)
        if basis == "dense":                       # every band is all 1025 bins
            fb = torch.rand(1025, 128, generator=g) + 0.01
        elif basis == "one_bin_and_zero":          # band of length 1 (row 5) and of length 0 (row 7)
            fb[:, 5] = 0
            fb[300, 5] = 0.7
            fb[:, 7] = 0
        elif basis == "gap":                       # row 9: non-zeros at 200..210 and 400..420, zeros between
            fb[:, 9] = 0
            fb[200:211, 9] = torch.rand(11, generator=g) + 0.1
            fb[400:421, 9] = torch.rand(21, generator=g) + 0.1
        ana["mel.fb"] = fb
        _FE[basis] = (Engine(ana, states[1], precision="fp32"), fb.to(DEV, F64))
    return _FE[basis]


def _fe_run(eng, wav):
    B, L = wav.shape
    T = 1 + L // 441
    mel = torch.full((B, T, 128), NAN, device=DEV)
    sp = torch.full((B, T, 1025), NAN, device=DEV)
    _check(eng.lib.vfx_frontend_mel(eng.h, _ptr(wav), B, L, _ptr(mel), _ptr(sp), _stream()), "vfx_frontend_mel")
    torch.cuda.synchronize()
    return mel, sp


def _fe_ref(wav, fb64):
    """reflect pad, the float32 Hann values, rFFT, sqrt(max(|X|^2, 1e-8)) and the dense mel product, in float64"""
    x = F.pad(wav.to(F64)[:, None], (1024, 1024), mode="reflect")[:, 0]
    X = torch.fft.rfft(x.unfold(-1, 2048, 441) * _hann32().to(F64), dim=-1)
    sp = (X.real ** 2 + X.imag ** 2).clamp_min(1e-8).sqrt()
    return sp, sp @ fb64


def _fe_check(rec, eng, fb64, wav):
    mel, sp = _fe_run(eng, wav)
    assert bool(torch.isfinite(sp).all()) and bool(torch.isfinite(mel).all()), "unwritten or non-finite output"
    sp64, mel64 = _fe_ref(wav, fb64)
    assert sp.shape == sp64.shape and mel.shape == mel64.shape
    e_sp = float(_frame_err(sp, sp64).max())
    e_rel = _rel(sp, sp64)
    e_mel = float(((mel.to(F64) - mel64).abs() / mel64.pow(2).mean(-1, keepdim=True).sqrt()).max())
    rec("sp_frame_max", e_sp)
    rec("sp_rel_rms", e_rel)
    rec("mel_frame_max", e_mel)
    assert e_sp < SP_FRAME_TOL
    assert e_rel < SP_REL_TOL
    assert e_mel < MEL_FRAME_TOL
    return mel, sp


FE_LENS = [1025, 1026, 1322, 1323, 1324, 44099, 44100, SEG]
FE_KINDS = ["noise", "tone_on", "tone_half", "dc", "alt", "imp0", "impL", "zeros", "utt"]


@pytest.mark.parametrize("kind", FE_KINDS)
@pytest.mark.parametrize("L", FE_LENS)
def test_frontend_vs_fp64(states, L, kind, record_property):
    """One item: lengths from the shortest allowed (1025: frame 0's reflection reaches the item's far end) through
    3 x 441 +- 1 to a 30 s segment; a tone halfway between bins, the Nyquist bin (+-1) and impulses where the
    reflection happens.  All zeros: every magnitude is exactly sqrtf(1e-8f)."""
    eng, fb64 = _fe_engine(states, "model")
    wav = torch.from_numpy(_signal(kind, L, seed=L % 997 + FE_KINDS.index(kind))).to(DEV)[None]
    mel, sp = _fe_check(record_property, eng, fb64, wav)
    if kind == "zeros":
        floor = torch.tensor(1e-8, dtype=torch.float32).sqrt().item()
        assert bool((sp == floor).all())
        rows = fb64.sum(0) * floor
        assert float(((mel[0].to(F64) - rows).abs() / rows.max()).max()) < MEL_FRAME_TOL


@pytest.mark.parametrize("L", [1025, 44100])
def test_frontend_batch_of_different_items(states, L, record_property):
    """B = 3 with different items: each row is its own item's transform."""
    eng, fb64 = _fe_engine(states, "model")
    wav = torch.stack([torch.from_numpy(_signal(k, L, seed=i)) for i, k in enumerate(["noise", "utt", "tone_half"])])
    _fe_check(record_property, eng, fb64, wav.to(DEV))


@pytest.mark.parametrize("kind", ["noise", "tone_half"])
@pytest.mark.parametrize("basis", ["dense", "one_bin_and_zero", "gap"])
def test_frontend_filterbank_bands(states, basis, kind, record_property):
    """weights.pack_analysis turns each basis row into one (start, len) band of bins: a dense basis (len 1025), a
    one-bin row and an all-zero row (len 0), a row with zeros inside its band.  The banded product must equal the
    dense one."""
    eng, fb64 = _fe_engine(states, basis)
    wav = torch.from_numpy(_signal(kind, 44100, seed=3)).to(DEV)[None]
    mel, _ = _fe_check(record_property, eng, fb64, wav)
    if basis == "one_bin_and_zero":
        assert bool((mel[..., 7] == 0).all())


# ============================================================================ B. mode-1 pre-filter
def _hf_run(eng, wav, ratio, lens=None):
    B, L = wav.shape
    ws = torch.empty(eng.hf_cut_workspace_bytes(B, L), dtype=torch.uint8, device=DEV)
    cut = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    lens_out = None
    if lens is None:
        out = torch.full((B, 512 * (L // 512)), NAN, device=DEV)
        _check(eng.lib.vfx_hf_cut(eng.h, _ptr(wav), B, L, float(ratio), _ptr(out), _ptr(cut), _ptr(ws), ws.numel(),
                                  _stream()), "vfx_hf_cut")
    else:
        out = torch.full((B, L), NAN, device=DEV)
        lens_out = torch.full((B,), -7, dtype=torch.int32, device=DEV)
        _check(eng.lib.vfx_hf_cut_ragged(eng.h, _ptr(wav), B, L, _ptr(lens), float(ratio), _ptr(out), _ptr(lens_out),
                                         _ptr(cut), _ptr(ws), ws.numel(), _stream()), "vfx_hf_cut_ragged")
    torch.cuda.synchronize()
    return out, cut, lens_out


def _hf_spectrum(x):
    """librosa.stft(n_fft 2048, hop 512, center, zero padding) of the float32 item x in float64, with the engine's
    float32 window values: (frames, 1025) complex128"""
    xp = F.pad(x.to(F64), (1024, 1024))
    return torch.fft.rfft(xp.unfold(0, 2048, 512) * _hann32().to(F64), dim=-1)


def _check_cut(rec, S, ratio, cut):
    """base.py:94-99 in float64 on float32 features: cut = the first bin whose running energy sum reaches
    ratio x total.  The kernel adds the same features in double, in an order that varies from run to run, from its
    own fp32 spectrum.  So `cut` must be consistent with the float64 running sum cs up to a margin m:
    cs[cut - 1] < thr + m and cs[cut] >= thr - m.  Wherever no partial sum lies within m of thr, this is equality."""
    feat = torch.log10(S.abs() + 1e-8).clamp_min(0).float().to(F64)
    cs = torch.cumsum(feat.sum(0), 0)
    total = float(cs[-1])
    thr = total * float(np.float32(ratio))
    m = CUT_MARGIN * total
    hit = torch.nonzero(cs >= thr).flatten()
    ref = int(hit[0]) if hit.numel() else 1024
    rec("cut", cut)
    rec("cut_ref", ref)
    rec("cut_gap", min(abs(float(cs[ref]) - thr), abs(float(cs[ref - 1]) - thr) if ref > 0 else math.inf) / max(total, 1e-300))
    assert cut == 1024 or float(cs[cut]) >= thr - m, f"cut {cut} (float64: {ref}): the running sum is short of thr"
    assert cut == 0 or float(cs[cut - 1]) < thr + m, f"cut {cut} (float64: {ref}): the sum reached thr earlier"


def _hf_wave(S, cut):
    """the float64 remainder of base.py:100-104 with the given cut: S |S| / (|S| + 1e-8) below the cut, irFFT,
    window, overlap-add, divide by the window sum-square where it exceeds float32's tiny, trim center padding to
    512 * (frames - 1) samples"""
    nfr = S.shape[0]
    mag = S.abs()
    Sp = S * (mag / (mag + 1e-8))
    Sp[:, cut:] = 0
    w = _hann32().to(F64)
    fr = torch.fft.irfft(Sp, n=2048, dim=-1) * w
    y = torch.zeros(nfr + 3, 512, dtype=F64, device=DEV)
    wss = torch.zeros_like(y)
    for q in range(4):
        y[q:q + nfr] += fr[:, q * 512:(q + 1) * 512]
        wss[q:q + nfr] += (w * w)[q * 512:(q + 1) * 512]
    y, wss = y.flatten(), wss.flatten()
    y = torch.where(wss > torch.finfo(torch.float32).tiny, y / wss, y)
    return y[1024:1024 + 512 * (nfr - 1)]


def _check_wave(rec, got, ref):
    """max per-sample error over the item's RMS, in [0, 512), [512, 1024), the middle and the last 2048 samples"""
    n = ref.numel()
    assert got.numel() == n
    assert bool(torch.isfinite(got).all()), "unwritten or non-finite output"
    rms = float(ref.pow(2).mean().sqrt())
    if rms == 0.0:
        assert bool((got == 0).all())
        return
    err = (got.to(F64) - ref).abs() / rms
    regions = {"head": (0, 512), "edge": (512, 1024), "middle": (1024, n - 2048), "tail": (max(0, n - 2048), n)}
    for name, (a, b) in regions.items():
        a, b = max(0, a), min(n, b)
        if b > a:
            e = float(err[a:b].max())
            rec(f"err_{name}", e)
            assert e < HF_TOL, f"{name} [{a}, {b}): max error {e:.3e} x RMS"


HF_LENS = [512, 513, 1023, 1024, 1025, 1536, 2047, 2048, 2049, 35280, SEG]
HF_KINDS = ["white_0.1", "white_3", "utt", "lowpass", "zeros"]


def _hf_case(rec, engine, x, ratio):
    out, cut, _ = _hf_run(engine, x[None], ratio)
    S = _hf_spectrum(x)
    c = int(cut[0])
    if not bool((x != 0).any()):
        assert c == 0 and bool((out == 0).all())
        return
    _check_cut(rec, S, ratio, c)
    _check_wave(rec, out[0], _hf_wave(S, c))


@pytest.mark.parametrize("kind", HF_KINDS)
@pytest.mark.parametrize("L", HF_LENS)
def test_hf_cut_vs_fp64(engine, L, kind, record_property):
    """vfx_hf_cut at ratio 0.95 from the minimum length (512: two frames) through the frame-count steps around
    multiples of 512 to a 30 s segment.  Samples 512..1023 take frame 0 into their overlap-add, whose truncating
    index once dropped it (an error of 3e-2 on white noise of sigma 3)."""
    x = torch.from_numpy(_signal(kind, L, seed=L % 991 + 17 * HF_KINDS.index(kind))).to(DEV)
    _hf_case(record_property, engine, x, 0.95)


@pytest.mark.parametrize("kind", HF_KINDS)
@pytest.mark.parametrize("ratio", [0.5, 0.999])
def test_hf_cut_ratio(engine, ratio, kind, record_property):
    x = torch.from_numpy(_signal(kind, 35280, seed=5 + HF_KINDS.index(kind))).to(DEV)
    _hf_case(record_property, engine, x, ratio)


def test_hf_cut_ragged_vs_fp64(engine, record_property):
    """vfx_hf_cut_ragged on a NaN-filled output: an item below 512 samples (filtered as its row's first 512), items
    of L_cap and beyond it (clamped to L_cap), and mixed lengths.  Every row holds its item's filtered samples, then
    exact zeros up to L_cap; lens_out = 512 (len // 512) of the clamped length.  Samples past an item's length are
    loud noise that must not leak in."""
    L_cap = 35280
    lens_in = [300, L_cap, 9000, 2047, 513, L_cap + 4000, 1536]
    g = torch.Generator().manual_seed(77)
    wav = (torch.randn(len(lens_in), L_cap, generator=g) * 0.1).to(DEV)
    for b, n in enumerate(lens_in):
        wav[b, min(n, L_cap):] *= 30.0
    lens = torch.tensor(lens_in, dtype=torch.int32, device=DEV)
    out, cut, lens_out = _hf_run(engine, wav, 0.95, lens)
    for b, n in enumerate(lens_in):
        Lb = min(max(n, 512), L_cap)
        nb = 512 * (Lb // 512)
        assert int(lens_out[b]) == nb
        assert bool((out[b, nb:] == 0).all()), f"row {b}: not zero after its {nb} samples"
        S = _hf_spectrum(wav[b, :Lb])
        _check_cut(record_property, S, 0.95, int(cut[b]))
        _check_wave(record_property, out[b, :nb], _hf_wave(S, int(cut[b])))


# ============================================================================ C. oracle front end
_HANN64 = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(2048) / 2048)


def _oracle_ref(a):
    """librosa 0.10.1's arithmetic for vocoder/base.py:61-73: float32 wav / max|wav|, zero center padding, the float64
    periodic Hann times the float32 frames, float64 rFFT rounded to complex64, |.| in float32, the Slaney basis in
    float64, dB - 20, normalise and clip, the -4 tail.  Returns (conditions (Tc, 128) float64, T, Tc)."""
    from voicefixer_b200 import wavio
    w = a / np.max(np.abs(a))
    x = np.pad(w, (1024, 1024))
    T = 1 + (len(x) - 2048) // 441
    idx = np.arange(2048)[None, :] + 441 * np.arange(T)[:, None]
    mag = np.abs(np.fft.rfft(x[idx] * _HANN64[None, :], axis=1).astype(np.complex64))
    mel = mag.astype(np.float64) @ wavio.slaney_htk_mel_basis().astype(np.float64).T
    min_level = np.exp(-100 / 20 * np.log(10))
    S = 20 * np.log10(np.maximum(min_level, np.abs(mel))) - 20
    S = np.clip(8.0 * ((S + 115.0) / 115.0) - 4.0, -4.0, 4.0)
    Tc = T + T % 2 + 4
    return np.concatenate([S, np.full((Tc - T, 128), -4.0)]), T, Tc


def _oracle_items():
    g = np.random.default_rng(31)
    t = np.arange(2 * SR) / SR
    bin_hz = SR / 2048
    tone = lambda f: np.sin(2 * np.pi * f * t + 0.2).astype(np.float32)
    neg = (0.1 * g.standard_normal(SR)).astype(np.float32)
    neg[12345] = -0.9                                         # the peak is one negative sample
    items = {"tone_1k": tone(1000.0), "tone_1k_on_bin": tone(46 * bin_hz), "tone_440": tone(440.0),
             "tone_440_on_bin": tone(20 * bin_hz), "noise": g.standard_normal(3 * SR).astype(np.float32),
             "negative_peak": neg}
    for n in (1, 440, 441, 442, 2048):
        items[f"len_{n}"] = (0.3 * g.standard_normal(n)).astype(np.float32)
    from voicefixer_b200 import synthetic
    items["utt_10s"] = synthetic.make_utterances(1, seconds=10.0, seed=33)[0]
    return items


@pytest.fixture(scope="module")
def oracle_case():
    """every item in one ragged batch, rows padded with loud noise past each item, plus one row whose lens exceeds
    L_cap (clamped); with the float64 reference of every item"""
    items = _oracle_items()
    names = list(items)
    L_cap = max(a.shape[0] for a in items.values()) + 777
    g = torch.Generator().manual_seed(5)
    wav = torch.randn(len(names) + 1, L_cap, generator=g) * 4.0
    lens = []
    for b, k in enumerate(names):
        wav[b, :items[k].shape[0]] = torch.from_numpy(items[k])
        lens.append(items[k].shape[0])
    lens.append(L_cap + 1000)
    refs = [_oracle_ref(items[k]) for k in names] + [_oracle_ref(wav[-1].numpy())]
    return names + ["over_L_cap"], wav.to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV), refs


_VOC = {}


def _voc_engine(states, prec):
    if prec not in _VOC:
        from voicefixer_b200.engine import Engine
        from voicefixer_b200.weights import pack_vocoder
        _VOC[prec] = Engine(packed=pack_vocoder(states[1], prec), precision=prec)
    return _VOC[prec]


def test_oracle_cond_fp32_vs_fp64(states, oracle_case, record_property):
    """vfx_oracle_cond into a NaN-filled buffer: rows below T_b within ORACLE_TOL of librosa's arithmetic, rows
    T_b .. Tc_b - 1 exactly -4, rows from Tc_b on exactly 0 (oracle_fe.cu)."""
    names, wav, lens, refs = oracle_case
    eng = _voc_engine(states, "fp32")
    B, L_cap = wav.shape
    T_cap = 1 + L_cap // 441
    Tc_cap = T_cap + T_cap % 2 + 4
    cond = torch.full((B, Tc_cap, 128), NAN, device=DEV)
    ws = torch.empty((4 * B + 255) // 256 * 256, dtype=torch.uint8, device=DEV)
    _check(eng.lib.vfx_oracle_cond(eng.h, _ptr(wav), B, L_cap, _ptr(lens), _ptr(cond), _ptr(ws), ws.numel(),
                                   _stream()), "vfx_oracle_cond")
    torch.cuda.synchronize()
    cond = cond.cpu().numpy()
    worst = 0.0
    for b, (name, (ref, T, Tc)) in enumerate(zip(names, refs)):
        err = float(np.max(np.abs(cond[b, :T].astype(np.float64) - ref[:T])))
        record_property(f"max_abs_{name}", err)
        worst = max(worst, err)
        assert err < ORACLE_TOL, f"{name}: max-abs {err:.3e}"
        assert bool((cond[b, T:Tc] == -4.0).all()), f"{name}: tail rows are not -4"
        assert bool((cond[b, Tc:] == 0.0).all()), f"{name}: rows past Tc_b are not 0"
    record_property("max_abs", worst)


def _ordinal(q, prec):
    """consecutive values of the format -> consecutive integers (+0 and -0 -> 0)"""
    if prec == "tf32":
        i = q.contiguous().view(torch.int32)
        mag = (i & 0x7FFFFFFF) >> 13
    else:
        i = q.contiguous().view(torch.int16).to(torch.int32)
        mag = i & 0x7FFF
    return torch.where(i < 0, -mag, mag)


def _fmt_round(x64, prec):
    from voicefixer_b200.weights import round_tf32
    return round_tf32(x64.float()) if prec == "tf32" else x64.to(DT[prec])


@pytest.mark.parametrize("prec", ["bf16", "fp16", "tf32"])
def test_oracle_operand_conditions(states, oracle_case, prec, record_property):
    """The conditions vfx_oracle writes in the operand format, read from its workspace (a bump allocation after the
    per-item peaks, frame counts and extent table, each 256-byte aligned): every element below T_b is the float64
    reference rounded to the format or one of its two neighbours, every row from T_b on is -4."""
    names, wav, lens, refs = oracle_case
    eng = _voc_engine(states, prec)
    B, L_cap = wav.shape
    T_cap = 1 + L_cap // 441
    Tc_cap = T_cap + T_cap % 2 + 4
    nbytes = eng.oracle_workspace_bytes(B, L_cap)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)          # NaN in every format
    out = torch.empty(B, Tc_cap * 441, device=DEV)
    _check(eng.lib.vfx_oracle(eng.h, _ptr(wav), B, L_cap, _ptr(lens), 1.0, _ptr(out), _ptr(ws), nbytes, _stream()),
           "vfx_oracle")
    torch.cuda.synchronize()
    r256 = lambda n: (n + 255) // 256 * 256
    off = 2 * r256(4 * B) + r256(4 * 15 * B)
    esz = 2 if prec in ("bf16", "fp16") else 4
    op = ws[off:off + B * Tc_cap * 128 * esz].view(DT[prec]).view(B, Tc_cap, 128)
    worst = 0
    for b, (name, (ref, T, Tc)) in enumerate(zip(names, refs)):
        got = op[b, :T]
        if prec == "tf32":
            assert int((got.contiguous().view(torch.int32) & 0x1FFF).abs().max()) == 0
        want = _fmt_round(torch.from_numpy(ref[:T]).to(DEV), prec)
        steps = int((_ordinal(got, prec) - _ordinal(want, prec)).abs().max())
        worst = max(worst, steps)
        assert steps <= 1, f"{name}: {steps} steps from the rounded float64 reference"
        assert bool((op[b, T:].float() == -4.0).all()), f"{name}: rows from T_b on are not -4"
    record_property("max_steps", worst)
