"""The element-wise, batch-statistics and waveform-output kernels of elementwise.cu against float64 references, called
one kernel at a time through the C ABI's per-kernel entry points (vfx_bn_stats, vfx_voc_post, ...).

Every restore, vocoder and oracle call goes through these kernels, but the whole-path comparisons with the oracle
(relative RMS over a waveform) cannot see an error that stays local: one reflected row at the ends of an output, or
the statistics of one channel at one UNet level.  Here each reference is computed in float64 on exactly the float32
(or operand-format) values the kernel reads, the error is checked element by element, and outputs start filled with a
sentinel or NaN, so memory a kernel fails to write, or writes outside its region, is caught.  Checks marked exact
compare bits.  Measured thresholds are at least 3x the worst value measured on an H100 80GB HBM3 (700 W power limit);
every input is seeded, so those values repeat.  Each test records its statistics as pytest properties (written by
--junitxml with -o junit_family=legacy).  Every grid-stride kernel runs at least one case above grid_for's cap of
132 x 32 blocks x 256 threads (1 081 344 elements), so its loop turns more than once.
"""
import ctypes
import math
import zlib
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
NAN = float("nan")
SENT = -1920.0                  # sentinel: exact in fp32, bf16, fp16 and tf32, and no kernel result
DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "tf32": torch.float32, "fp32": torch.float32}
PREC = {"fp32": 0, "bf16": 1, "tf32": 2, "fp16": 3}
ACT = {"none": 0, "lrelu": 1}
GRID_CAP = 132 * 32 * 256

# A. bn_act(bn_stats(x)) against float64 F.batch_norm(training=True), relative RMS per item: kernel <= 2 x torch's fp32
# error + BN_CEIL x (1 + |mean| / sigma).  y = fmaf(x, s, t) carries the float32 rounding of t = beta - mean s, which
# grows with |mean| / sigma (torch subtracts the mean first).  Measured: kernel 3.5e-8 .. 9.8e-6, torch 3.9e-8 ..
# 8.5e-5; the largest excess over 2 x torch 7.2e-7 at |mean| / sigma = 300 (2.4e-9 per unit).
BN_CEIL = 1e-8
# C. max |xlog - xlog64| and |log10 mel - log10 mel64| (log10 domain); measured worst 8.3e-7.
LOG_TOL = 2.5e-6
# unet_head: |out - out64| / (|bias| + sum |w x| + |xlog|); measured worst 2.5e-7.
HEAD_TOL = 8e-7
# D. voc_normalize fp32: max |cond - cond64|; measured worst 1.2e-6.
NORM_TOL = 4e-6
# E. voc_post: |out / scale - tanh64| / (1 + sum of the magnitudes of the terms), see test_voc_post.
POST_TOL = 1.2e-7


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _call(name, *args):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    _lib.check(getattr(lib, name)(*args, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), name)
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ulp(v64):
    """the spacing of float32 at |v64| (the larger neighbour's, at a power of two), in float64"""
    a = v64.abs().float()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).to(F64)


def _ord(q, prec):
    """consecutive values of the format -> consecutive integers (+0 and -0 -> 0)"""
    if prec in ("fp32", "tf32"):
        i = q.contiguous().view(torch.int32).to(torch.int64)
        mag = i & 0x7FFFFFFF
        if prec == "tf32":
            mag = mag >> 13
    else:
        i = q.contiguous().view(torch.int16).to(torch.int64)
        mag = i & 0x7FFF
    return torch.where(i < 0, -mag, mag)


def _fmt_round(x64, prec):
    """float64 -> nearest value of the format, stored as the kernel stores it (tf32: ties away, cvt.rna)"""
    from voicefixer_b200.weights import round_tf32
    if prec == "tf32":
        return round_tf32(x64.float())
    return x64.to(DT[prec])


def _worst(t):
    """max of an error tensor; a NaN anywhere (a value read from a NaN-filled row) is infinitely bad"""
    return math.inf if bool(torch.isnan(t).any()) else float(t.max())


def _bits_equal(a, b):
    view = torch.int16 if a.element_size() == 2 else torch.int32
    return torch.equal(a.contiguous().view(view), b.contiguous().view(view))


# ============================================================================ A. train-mode BatchNorm
RATIOS = [0.0, 1.0, 30.0, 300.0, "const"]


def _channel_values(n, ratio, g):
    """n float32 values of one channel with |mean| / sigma = ratio (or constant)"""
    sigma = 0.5 + torch.rand(1, generator=g).item()
    sign = 1.0 if torch.rand(1, generator=g).item() < 0.5 else -1.0
    if ratio == "const":
        return torch.full((n,), sign * 3.0 * sigma)
    return sign * ratio * sigma + sigma * torch.randn(n, generator=g)


def _bn_input(B, P, pad, C, ldx, col, bn_C, ratio, seed):
    """x [B][P + pad][ldx] (NaN outside columns [col, col + C) and in the pad rows) and the item data view.
    bn_C = 1: item b's values have the ratio `ratio`; bn_C = C: channel c has RATIOS[c % 5] (ratio unused)."""
    g = _gen(seed)
    buf = torch.full((B, P + pad, ldx), NAN)
    for b in range(B):
        if bn_C == 1:
            buf[b, :P, col:col + C] = _channel_values(P * C, ratio, g).view(P, C)
        else:
            for c in range(C):
                buf[b, :P, col + c] = _channel_values(P, RATIOS[(c + b) % 5], g)
    buf = buf.to(DEV)
    return buf, buf[:, :, col:col + C]


def _bn_stats(x, B, P, C, bn_C, gamma, beta, seq=None, per_row=1):
    scale = torch.full((B, bn_C), NAN, device=DEV)
    shift = torch.full((B, bn_C), NAN, device=DEV)
    acc = torch.full((2 * B * bn_C,), NAN, dtype=F64, device=DEV)
    _call("vfx_bn_stats", _ptr(x), x.stride(0), x.stride(1), B, P, C, bn_C, _ptr(gamma), _ptr(beta), _ptr(scale),
          _ptr(shift), _ptr(acc), _ptr(seq), per_row)
    return scale, shift


def _bn_act(x, B, P, C, scale, shift, bn_C, stat_sB, act, p, prec, ldy):
    y = torch.full((B, P, ldy), SENT, dtype=DT[prec], device=DEV)
    _call("vfx_bn_act", PREC[prec], _ptr(x), x.stride(0), x.stride(1), B, P, C, _ptr(scale), _ptr(shift), bn_C, stat_sB,
          ACT[act], ctypes.c_float(p), _ptr(y), y.stride(0), y.stride(1))
    return y


def _check_stats(rec, xs, bn_C, gamma, beta, s, t):
    """one item's statistics: xs [Pb][C] float32 -> the bounds that follow from bn_stats_final's arithmetic"""
    x64 = xs.to(F64)
    if bn_C == 1:
        x64 = x64.reshape(-1, 1)
    mean = x64.mean(0)
    var = (x64 - mean).pow(2).mean(0)
    s64 = gamma.to(F64) / torch.sqrt(var + 1e-5)
    t64 = beta.to(F64) - mean * s64
    s_err = (s.to(F64) - s64).abs() / _ulp(s64)
    t_err = (t.to(F64) - t64).abs() / (_ulp(beta.to(F64)) + 4 * _ulp(mean * s64))
    return _worst(s_err), _worst(t_err)


def _item_positions(seq, b, per_row, P):
    return P if seq is None else min(P, seq[b] * per_row)


def _run_stats_case(rec, B, P, pad, C, ldx, col, bn_C, ratio, seq_list, per_row, seed):
    x_buf, x = _bn_input(B, P, pad, C, ldx, col, bn_C, ratio, seed)
    # rows past an item's extent (inside the capacity P) hold NaN: a statistic that reads them comes out NaN
    for b in range(B):
        x_buf[b, _item_positions(seq_list, b, per_row, P):P] = NAN
    g = _gen(seed + 1)
    gamma = (0.5 + torch.rand(bn_C, generator=g)).to(DEV)
    beta = (0.5 * torch.randn(bn_C, generator=g)).to(DEV)
    seq = None if seq_list is None else torch.tensor(seq_list, dtype=torch.int32, device=DEV)
    scale, shift = _bn_stats(x, B, P, C, bn_C, gamma, beta, seq, per_row)
    worst_s = worst_t = 0.0
    for b in range(B):
        Pb = _item_positions(seq_list, b, per_row, P)
        es, et = _check_stats(rec, x[b, :Pb], bn_C, gamma, beta, scale[b], shift[b])
        worst_s, worst_t = max(worst_s, es), max(worst_t, et)
    rec("scale_err_over_2ulp", worst_s / 2)
    rec("shift_err_over_bound", worst_t)
    assert worst_s <= 2, f"scale {worst_s:.3g} ulp from float64"
    assert worst_t <= 1, f"shift error {worst_t:.3g} x its bound"
    return x, scale, shift, gamma, beta


@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("C", [128, 256, 512])
def test_bn_stats_denoiser(C, ratio, record_property):
    """The denoiser's single-channel norms (bn_C = 1): P = T frames of C features, count P_b x C.  Ragged seq
    (per_row 1): item 0 asks for more frames than the capacity (clamped to P; the rows past P are NaN), item 1 ends
    inside a 256-row block of the reduction, item 2 is one frame.  |mean| / sigma up to 300, where E[x^2] - mean^2
    cancels, and a constant item (variance 0, the var < 0 -> 0 clamp).  Bounds from bn_stats_final's arithmetic:
    |s - s64| <= 2 ulp(s64), |t - t64| <= ulp(beta) + 4 ulp(mean64 s64).  Measured on the H100, denoiser and UNet
    norms alike: s within 1.24 ulp, t within 0.61 of its bound, at |mean| / sigma = 300 as well."""
    B, T = 3, 301
    _run_stats_case(record_property, B, T, 300, C, C, 0, 1, ratio, [T + 5, 200, 1], 1, seed=C + 7 * RATIOS.index(ratio))


UNET = [(2, 127), (32, 127), (64, 63), (128, 31), (256, 15), (384, 7), (384, 3), (384, 1)]


@pytest.mark.parametrize("C,W", UNET)
def test_bn_stats_unet(C, W, record_property):
    """The UNet's per-channel norms: C = 2 with ldx = 2 (the first encoder block), otherwise the pitch-2C concat
    buffer read at column offset C; W = 127 .. 1 with H = 128 >> k rows.  Channel c has |mean| / sigma from
    RATIOS[(c + b) % 5].  Ragged seq with per_row = W: item 0 beyond the capacity, item 1 ending inside a 256-row block,
    item 2 one row (at W = 1 a single position: the 1 x 1 centre, variance 0)."""
    H = {127: 128, 63: 64, 31: 32, 15: 16, 7: 8, 3: 4, 1: 2}[W]
    B, P = 3, H * W
    ldx, col = (2, 0) if C == 2 else (2 * C, C)
    _run_stats_case(record_property, B, P, 256 + 2 * W, C, ldx, col, C, None, [H + 2, H // 2 + 1, 1], W, seed=C * W)


@pytest.mark.parametrize("prec", ["fp32", "bf16", "fp16", "tf32"])
@pytest.mark.parametrize("path", ["float4", "scalar"])
@pytest.mark.parametrize("stats", ["per_channel", "single", "shared"])
@pytest.mark.parametrize("act,p", [("lrelu", 0.01), ("lrelu", 0.0), ("none", 0.0)])
def test_bn_act(act, p, stats, path, prec, record_property):
    """y = act(fmaf(x, s, t)) in every operand format, on both the float4 path (C % 4 == 0, aligned) and the scalar one
    (x read at an odd column), with per-item statistics (stat_sB = bn_C), one shared set (stat_sB = 0) and the
    single-channel form.  fp32: within 1 step of float64 where the activation is the identity, 2 on LeakyReLU's
    negative side (the fma, then the product with the float32 slope, round).  16-bit / tf32: within one step of the
    float64 value rounded to the format; tf32 has its low 13 bits clear.  Columns >= C of the wider ldy keep the
    sentinel.  B x P x C / 4 = 1.15M: the grid-stride loop turns twice.  Measured on the H100: at most 1 step in every
    format, on both sides of the activation."""
    B, P, C = 3, 24000, 64
    ldy = C + 8
    col = 4 if path == "float4" else 1
    g = _gen(zlib.crc32(repr((act, p, stats, path, prec)).encode()))
    xbuf = (2 * torch.randn(B, P, C + 8, generator=g)).to(DEV)
    x = xbuf[:, :, col:col + C]
    bn_C = 1 if stats == "single" else C
    stat_sB = 0 if stats == "shared" else bn_C
    nsets = 1 if stat_sB == 0 else B
    scale = (0.5 + torch.rand(nsets, bn_C, generator=g)).to(DEV)
    shift = (0.5 * torch.randn(nsets, bn_C, generator=g)).to(DEV)
    assert B * P * C // (4 if path == "float4" else 1) > GRID_CAP
    y = _bn_act(x, B, P, C, scale, shift, bn_C, stat_sB, act, p, prec, ldy)
    s = scale.to(F64)[torch.arange(B) % nsets].view(B, 1, bn_C)
    t = shift.to(F64)[torch.arange(B) % nsets].view(B, 1, bn_C)
    z = x.to(F64) * s + t
    p32 = float(torch.tensor(p, dtype=torch.float32))
    ref = torch.where(z > 0, z, z * p32) if act == "lrelu" else z
    got = y[:, :, :C]
    assert bool((y[:, :, C:].float() == SENT).all())
    if prec == "tf32":
        assert int((got.contiguous().view(torch.int32) & 0x1FFF).abs().max()) == 0
    steps = (_ord(got, prec) - _ord(_fmt_round(ref, prec), prec)).abs()
    record_property("max_steps", int(steps.max()))
    if prec == "fp32":
        neg = (z <= 0) & (act == "lrelu")
        assert int(steps[~neg].max()) <= 1
        if bool(neg.any()):
            assert int(steps[neg].max()) <= 2
    else:
        assert int(steps.max()) <= 1


def _rel(got, ref):
    got, ref = got.to(F64), ref.to(F64)
    return float((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())


@pytest.mark.parametrize("ratio", [0.0, 1.0, 30.0, 300.0])
@pytest.mark.parametrize("kind", ["denoiser", "unet"])
def test_bn_end_to_end(kind, ratio, record_property):
    """bn_act(bn_stats(x)) (fp32, identity) on each item against float64 F.batch_norm(training=True), next to torch's
    own fp32 F.batch_norm on the same item: the kernel's relative RMS error must stay within twice torch's plus
    BN_CEIL per unit of |mean| / sigma (see BN_CEIL)."""
    if kind == "denoiser":
        B, P, C, bn_C, W, seq_list = 3, 301, 512, 1, 1, [301, 200, 37]
    else:
        B, P, C, bn_C, W, seq_list = 3, 64 * 63, 64, 64, 63, [64, 33, 2]
    x_buf, x = _bn_input(B, P, 0, C, C, 0, bn_C, ratio, seed=int(ratio) + len(kind))
    if bn_C != 1:          # every channel at the ratio of this case
        g = _gen(5)
        x_buf.copy_(torch.stack([torch.stack([_channel_values(P, ratio, g) for _ in range(C)], 1)
                                 for _ in range(B)]).to(DEV))
    g = _gen(9)
    gamma = (0.5 + torch.rand(bn_C, generator=g)).to(DEV)
    beta = (0.5 * torch.randn(bn_C, generator=g)).to(DEV)
    seq = torch.tensor(seq_list, dtype=torch.int32, device=DEV)
    scale, shift = _bn_stats(x, B, P, C, bn_C, gamma, beta, seq, W)
    y = _bn_act(x, B, P, C, scale, shift, bn_C, bn_C, "none", 0.0, "fp32", C)
    worst = 0.0
    for b in range(B):
        Pb = seq_list[b] * W
        xi, yi = x[b, :Pb], y[b, :Pb]
        if bn_C == 1:
            shape = (1, 1, Pb * C)
            ref = F.batch_norm(xi.to(F64).reshape(shape), None, None, gamma.to(F64), beta.to(F64), True, 0.0, 1e-5)
            t32 = F.batch_norm(xi.reshape(shape), None, None, gamma, beta, True, 0.0, 1e-5)
        else:
            ref = F.batch_norm(xi.to(F64), None, None, gamma.to(F64), beta.to(F64), True, 0.0, 1e-5)
            t32 = F.batch_norm(xi, None, None, gamma, beta, True, 0.0, 1e-5)
        ref = ref.reshape(Pb, C)
        err, err_t = _rel(yi, ref), _rel(t32.reshape(Pb, C), ref)
        record_property(f"item{b}_kernel_rel_rms", err)
        record_property(f"item{b}_torch_fp32_rel_rms", err_t)
        worst = max(worst, (err - 2 * err_t) / (1 + ratio))
        assert err <= 2 * err_t + BN_CEIL * (1 + ratio), f"item {b}: kernel {err:.3g} against torch fp32 {err_t:.3g}"
    record_property("worst_excess_per_unit_ratio", worst)


# ============================================================================ B. exact kernels
def test_dropout_apply_exact():
    """x[i] = keep[i] ? 2 x[i] : 0 (any non-zero keep byte keeps), bit for bit, over 1.3M elements."""
    n = 1_300_003
    g = _gen(31)
    x0 = torch.randn(n, generator=g).to(DEV)
    keep = torch.randint(0, 4, (n,), generator=g, dtype=torch.uint8)
    keep[keep == 3] = 255
    keep = keep.to(DEV)
    x = x0.clone()
    _call("vfx_dropout_apply", _ptr(x), _ptr(keep), n)
    assert _bits_equal(x, torch.where(keep != 0, x0 * 2, torch.zeros_like(x0)))


@pytest.mark.parametrize("B,H,W,C", [(3, 128, 127, 384), (2, 8, 127, 32), (2, 5, 3, 384), (1, 2, 2, 4)])
def test_avgpool2x2_exact(B, H, W, C):
    """((a + b) + c) + d) * 0.25 in float32, bit for bit, from the pitch-2C concat buffer at column offset C, odd W
    (the last column dropped) and odd H (the last row dropped).  The first case runs 1.16M float4 threads."""
    g = _gen(B * H * W + C)
    buf = torch.randn(B, H, W, 2 * C, generator=g).to(DEV)
    x = buf[..., C:]
    Ho, Wo = H // 2, W // 2
    y = torch.full((B * Ho * Wo * C + 64,), SENT, device=DEV)
    _call("vfx_avgpool2x2", _ptr(x), x.stride(0), x.stride(1), x.stride(2), B, H, W, C, _ptr(y))
    a, b = x[:, 0:2 * Ho:2, 0:2 * Wo:2], x[:, 0:2 * Ho:2, 1:2 * Wo:2]
    c, d = x[:, 1:2 * Ho:2, 0:2 * Wo:2], x[:, 1:2 * Ho:2, 1:2 * Wo:2]
    ref = (((a + b) + c) + d) * 0.25
    assert _bits_equal(y[:-64].view(B, Ho, Wo, C), ref)
    assert bool((y[-64:] == SENT).all())


@pytest.mark.parametrize("prec", ["fp32", "bf16", "fp16", "tf32"])
@pytest.mark.parametrize("case", ["ragged", "equal", "big"])
def test_reflect_pad3_exact(case, prec):
    """ReflectionPad1d(3) in place on [B][L + 6][C], in the 2-byte (bf16 / fp16) and 4-byte forms, bit for bit; with
    ragged ext_len each item reflects at its own end, and rows past L_b + 5 keep the sentinel.  The big case runs
    1.23M threads."""
    B, L, C = {"ragged": (3, 50, 512), "equal": (2, 37, 128), "big": (400, 10, 512)}[case]
    g = _gen(B + L + C)
    lens = [L, 4, 17] if case == "ragged" else [L] * B
    buf = torch.full((B, L + 6, C), SENT, dtype=DT[prec], device=DEV)
    ref = buf.clone()
    for b, Lb in enumerate(lens):
        inner = torch.randn(Lb, C, generator=g).to(DEV).to(DT[prec])
        buf[b, 3:3 + Lb] = inner
        ref[b, :Lb + 6] = F.pad(inner.float().t()[None], (3, 3), mode="reflect")[0].t().to(DT[prec])
    ext = torch.tensor(lens, dtype=torch.int32, device=DEV) if case == "ragged" else None
    _call("vfx_reflect_pad3", _ptr(buf), B, L, C, _ptr(ext), PREC[prec])
    assert _bits_equal(buf, ref)


def _tie_inputs(prec, g):
    """float32 values exactly halfway between two neighbours of the format, with even and odd last kept bits"""
    if prec in ("tf32", "bf16"):
        low = 0x1000 if prec == "tf32" else 0x8000
        mag = torch.randint(0x00800000, 0x7F000000, (20000,), generator=g, dtype=torch.int32)
        sign = torch.randint(0, 2, (20000,), generator=g, dtype=torch.int32) << 31
        return (sign | (mag & ~(2 * low - 1)) | low).view(torch.float32)
    h = torch.randint(0, 0x7BFF, (20000,), generator=g, dtype=torch.int16)
    lo = h.view(torch.float16).float()
    hi = (h + 1).view(torch.float16).float()
    sign = torch.where(torch.rand(20000, generator=g) < 0.5, -1.0, 1.0)
    return sign * (lo + hi) / 2                    # exact in float32


@pytest.mark.parametrize("prec", ["bf16", "fp16", "tf32", "fp32"])
def test_cast_rows_exact(prec):
    """fp32 -> bf16 / fp16 with round-to-nearest-even (torch's .to), tf32 with ties away from zero (cvt.rna,
    weights.round_tf32), bit for bit, over 1.1M elements: normal values, ties where the two rules differ, subnormals,
    zeros of both signs, and values beyond fp16's range (to inf)."""
    from voicefixer_b200.weights import round_tf32
    g = _gen(41 + PREC[prec])
    parts = [torch.randn(1_100_000, generator=g) * 10, _tie_inputs(prec, g),
             torch.tensor([0.0, -0.0, 1e-40, -3e-39, 6e-8, 65519.0, 65520.0, 7e4, -1e6, 3e38])]
    x = torch.cat(parts).to(DEV)
    n = x.numel()
    y = torch.full((n + 64,), SENT, dtype=DT[prec], device=DEV)
    _call("vfx_cast_rows", _ptr(x), n, _ptr(y), PREC[prec])
    ref = round_tf32(x) if prec == "tf32" else x.to(DT[prec])
    assert _bits_equal(y[:n], ref)
    assert bool((y[n:].float() == SENT).all())


def _ext_rows(L, T):
    Tp = (T + 63) // 64 * 64
    Tc = T + T % 2 + 4
    return [L, T] + [Tp >> k for k in range(7)] + [Tc, Tc + 6, Tc * 7, Tc * 49, Tc * 147, Tc * 441]


@pytest.mark.parametrize("L_cap", [1025, 44100 * 3 + 17, 30 * 44100])
def test_ragged_extents_exact(L_cap):
    """ext[15][B] against DESIGN 3's table: L_b clamped into [1025, L_cap] (lengths below 1025, negative, exactly at
    and above L_cap), T_b = 1 + L_b // 441, Tp_b >> k, Tc_b = T_b + T_b % 2 + 4, Tc_b + 6, Tc_b x (7, 49, 147, 441).
    B = 300 spans three blocks."""
    g = _gen(L_cap)
    lens = torch.randint(-2000, L_cap + 5000, (300,), generator=g, dtype=torch.int32)
    lens[:8] = torch.tensor([0, -5, 1, 1024, 1025, L_cap, L_cap + 1, 2 ** 31 - 1], dtype=torch.int32)
    ext = torch.full((15, 300), -7, dtype=torch.int32, device=DEV)
    _call("vfx_ragged_extents", _ptr(lens.to(DEV)), 300, L_cap, _ptr(ext))
    want = []
    for L in lens.tolist():
        Lb = min(max(L, 1025), L_cap)
        want.append(_ext_rows(Lb, 1 + Lb // 441))
    assert ext.cpu().t().tolist() == want


@pytest.mark.parametrize("T_cap", [1, 7, 3001])
def test_frame_extents_exact(T_cap):
    """The vocoder's table: frames clamped into [1, T_cap] (below 1, negative, at and above T_cap), samples S_b =
    Tc_b x 441, the other rows as in ragged_extents."""
    g = _gen(T_cap)
    frames = torch.randint(-10, T_cap + 50, (300,), generator=g, dtype=torch.int32)
    frames[:6] = torch.tensor([0, -3, 1, T_cap, T_cap + 1, 2 ** 31 - 1], dtype=torch.int32)
    ext = torch.full((15, 300), -7, dtype=torch.int32, device=DEV)
    _call("vfx_frame_extents", _ptr(frames.to(DEV)), 300, T_cap, _ptr(ext))
    want = []
    for f in frames.tolist():
        T = min(max(f, 1), T_cap)
        Tc = T + T % 2 + 4
        want.append(_ext_rows(Tc * 441, T))
    assert ext.cpu().t().tolist() == want


# ============================================================================ C. analysis tail
def _mask_inputs(B, T, seed):
    g = _gen(seed)
    lin = 3 * torch.randn(B, T, 128, generator=g)
    mel = torch.rand(B, T, 128, generator=g) * 10 ** (4 * torch.rand(B, T, 128, generator=g) - 3)
    special_lin = torch.tensor([30.0, -30.0, 100.0, -100.0, 0.0, 88.0, -88.0, 104.0])
    special_mel = torch.tensor([0.0, 1e-8, 0.5e-8, 0.99e-8, 1.01e-8, 2e-8, 1e-9, 1.0])
    idx = torch.randint(0, B * T * 128, (4000,), generator=g)
    lin.view(-1)[idx] = special_lin[torch.arange(4000) % 8]
    idx = torch.randint(0, B * T * 128, (4000,), generator=g)
    mel.view(-1)[idx] = special_mel[torch.arange(4000) % 8]
    return lin.to(DEV), mel.to(DEV)


@pytest.mark.parametrize("ragged", [False, True])
def test_mask_log_pack(ragged, record_property):
    """xlog = log10(max(sigmoid(lin) mel, 1e-8)) and log10(max(mel, 1e-8)) against float64, with lin at +-30, +-88,
    +-100 (sigmoid saturates; expf overflows to inf), mel = 0 and values around 1e-8, T = 2900 (not a multiple of 64;
    1.13M threads) and ragged ext_frames.  Exact: unet_in rows t >= T_b are zero, unet_in[f] holds mel column f (column
    127 is never packed, nothing is written past the tensor), and xlog rows past T_b keep the sentinel."""
    B, T = 3, 2900
    Tp = (T + 63) // 64 * 64
    lin, mel = _mask_inputs(B, T, seed=51 + ragged)
    frames = [T, 1000, 1] if ragged else [T] * B
    ext = torch.tensor(frames, dtype=torch.int32, device=DEV) if ragged else None
    xlog = torch.full((B, T, 128), SENT, device=DEV)
    unet = torch.full((B * Tp * 127 * 2 + 64,), SENT, device=DEV)
    assert B * Tp * 128 > GRID_CAP
    _call("vfx_mask_log_pack", _ptr(lin), _ptr(mel), B, T, Tp, _ptr(ext), _ptr(xlog), _ptr(unet))
    floor = float(torch.tensor(1e-8, dtype=torch.float32))
    lin64, mel64 = lin.to(F64), mel.to(F64)
    lx = torch.log10(torch.clamp(mel64 / (1 + torch.exp(-lin64)), min=floor))
    lm = torch.log10(torch.clamp(mel64, min=floor))
    u = unet[:-64].view(B, Tp, 127, 2)
    assert bool((unet[-64:] == SENT).all())
    worst_x = worst_m = 0.0
    for b, Tb in enumerate(frames):
        assert bool((xlog[b, Tb:] == SENT).all())
        assert bool((u[b, Tb:] == 0).all()) and not bool(torch.signbit(u[b, Tb:]).any())
        ex = (xlog[b, :Tb].to(F64) - lx[b, :Tb]).abs()
        eu = (u[b, :Tb, :, 1].to(F64) - lx[b, :Tb, :127]).abs()
        em = (u[b, :Tb, :, 0].to(F64) - lm[b, :Tb, :127]).abs()
        assert torch.equal(u[b, :Tb, :, 1], xlog[b, :Tb, :127])
        worst_x, worst_m = max(worst_x, _worst(ex), _worst(eu)), max(worst_m, _worst(em))
    record_property("xlog_max_abs", worst_x)
    record_property("logmel_max_abs", worst_m)
    assert worst_x < LOG_TOL and worst_m < LOG_TOL


def test_unet_head(record_property):
    """out = bias + sum_c w[c] x[b][t][f][c] + xlog for f < 127 against float64, relative to the sum of the terms'
    magnitudes; column 127 is xlog exactly.  x has the UNet's padded Tp rows (never read past T); 1.11M threads."""
    B, T = 3, 2900
    Tp = (T + 63) // 64 * 64
    g = _gen(61)
    x = torch.randn(B, Tp, 127, 32, generator=g).to(DEV)
    x[:, T:] = NAN
    w = (torch.randn(32, generator=g) / 4).to(DEV)
    bias = torch.randn(1, generator=g).to(DEV)
    xlog = (8 * torch.rand(B, T, 128, generator=g) - 8).to(DEV)
    out = torch.full((B * T * 128 + 64,), SENT, device=DEV)
    _call("vfx_unet_head", _ptr(x), B, T, Tp, _ptr(w), _ptr(bias), _ptr(xlog), _ptr(out))
    o = out[:-64].view(B, T, 128)
    assert bool((out[-64:] == SENT).all())
    assert torch.equal(o[..., 127], xlog[..., 127])
    x64 = x[:, :T].to(F64)
    ref = bias.to(F64) + x64 @ w.to(F64) + xlog[..., :127].to(F64)
    mag = bias.to(F64).abs() + x64.abs() @ w.to(F64).abs() + xlog[..., :127].to(F64).abs()
    err = float(((o[..., :127].to(F64) - ref).abs() / mag).max())
    record_property("rel_max", err)
    assert err < HEAD_TOL


# ============================================================================ D. vocoder conditions
def _mel_tab():
    """voc.mel_tab as weights.pack_vocoder builds it"""
    k = torch.linspace(1, 128, 128)
    w = 18.8927416350036 * torch.exp(0.0269863588184314 * k)
    min_level = torch.exp(torch.tensor(-100.0) / 20 * torch.log(torch.tensor(10.0)))
    return torch.cat([w, min_level.reshape(1)]).float().to(DEV)


def _norm_inputs(B, T, is_log, tab, seed):
    """c = 8 (S + 115) / 115 - 4 is inside (-4, 4) for log10(|mel| / w) in (-4.75, 1): u spans both sides"""
    g = _gen(seed)
    u = 7.5 * torch.rand(B, T, 128, generator=g) - 6
    lw = torch.log10(tab[:128].cpu().to(F64))
    if is_log:
        mel = (lw + u).float()
        idx = torch.randint(0, B * T * 128, (3000,), generator=g)
        mel.view(-1)[idx] = torch.tensor([5.5, 40.0, -50.0, -1e4, 5.0, 4.9999])[torch.arange(3000) % 6]
    else:
        sign = torch.where(torch.rand(B, T, 128, generator=g) < 0.5, -1.0, 1.0)
        mel = (sign * 10 ** (lw + u)).float()
        idx = torch.randint(0, B * T * 128, (3000,), generator=g)
        mel.view(-1)[idx] = torch.tensor([0.0, -0.0, 1e-30, -1e30, 3e38])[torch.arange(3000) % 5]
    return mel.to(DEV)


@pytest.mark.parametrize("prec", ["fp32", "bf16", "fp16", "tf32"])
@pytest.mark.parametrize("is_log", [1, 0])
@pytest.mark.parametrize("T", [2900, 2901])
@pytest.mark.parametrize("ragged", [False, True])
def test_voc_normalize(ragged, T, is_log, prec, record_property):
    """Vocoder.forward's conditions against float64: log input (from_log, values above 5 clipped, very negative ones
    down to the min_level clamp) and linear input (negative mels through fabsf), on both sides of the +-4 clip; even and
    odd T (pre()'s tail of 4 or 5 rows); ragged ext_frames.  fp32 within NORM_TOL; an operand-format value lies between
    the roundings of cond64 - NORM_TOL and cond64 + NORM_TOL: it is the float64 value rounded to the format except
    within NORM_TOL of a rounding midpoint (or of zero, where the format's steps are finer than NORM_TOL).  Exact: clipped values are +-4, and tail and ragged rows are -4, in every format.  B x Tc x 128 = 1.11M threads."""
    B = 3
    Tc = T + T % 2 + 4
    tab = _mel_tab()
    mel = _norm_inputs(B, T, is_log, tab, seed=T + 2 * is_log + ragged)
    frames = [T, 1001, 1] if ragged else [T] * B
    ext = torch.tensor(frames, dtype=torch.int32, device=DEV) if ragged else None
    cond = torch.full((B * Tc * 128 + 64,), SENT, dtype=DT[prec], device=DEV)
    _call("vfx_voc_normalize", _ptr(mel), B, T, Tc, _ptr(ext), is_log, _ptr(tab), _ptr(cond), PREC[prec])
    assert bool((cond[-64:].float() == SENT).all())
    c = cond[:-64].view(B, Tc, 128)
    v = mel.to(F64)
    if is_log:
        v = 10 ** torch.clamp(v, max=5.0)
    tab64 = tab.to(F64)
    S = 20 * torch.log10(torch.clamp((v / tab64[:128]).abs(), min=float(tab64[128]))) - 20
    ref = torch.clamp(8 * ((S + 115) / 115) - 4, -4, 4)
    worst = 0.0
    for b, Tb in enumerate(frames):
        assert bool((c[b, Tb:].float() == -4).all())                    # pre()'s tail and the ragged rows
        got, r = c[b, :Tb], ref[b, :Tb]
        beyond = (8 * ((S[b, :Tb] + 115) / 115) - 4).abs() > 4 + NORM_TOL
        assert bool((got[beyond].float().abs() == 4).all())
        if prec == "fp32":
            worst = max(worst, _worst((got.to(F64) - r).abs()))
        else:
            if prec == "tf32":
                assert int((got.contiguous().view(torch.int32) & 0x1FFF).abs().max()) == 0
            lo, hi = _fmt_round(r - NORM_TOL, prec), _fmt_round(r + NORM_TOL, prec)
            ok = (_ord(lo, prec) <= _ord(got, prec)) & (_ord(got, prec) <= _ord(hi, prec))
            assert bool(ok.all()), f"{int((~ok).sum())} {prec} conditions differ from float64 rounded"
    record_property("fp32_max_abs", worst)
    assert worst < NORM_TOL


# ============================================================================ E. the waveform
POST_CASES = {
    # name: (S_b per item, out_len, trim L_b per item or None, lo, scale, input scale)
    "smallest_Tc6": ([2646], 2646, None, 0, 1.0, 1.0),
    "untrimmed_lo0": ([8820, 8820], 8820, None, 0, 32768.0, 1.0),
    "trim_even_diff": ([8820, 8820], 8818, None, 1, 1.0, 1.0),
    "trim_odd_diff": ([8820, 8820], 8813, None, 3, 32768.0, 1.0),
    "trim_5s": ([220500 + 441 * 4], 220500, None, 882, 32768.0, 1.0),
    "saturating": ([8820, 8820], 8805, None, 7, 1.0, 20.0),
    "linear": ([8820], 8820, None, 0, 32768.0, 1e-3),
    "ragged": ([13230, 8820, 2646], 13000, [13000, 8001, 2646], 0, 1.0, 1.0),
    "ragged_lo0": ([13230, 8820, 2646], 13230, [13230, 8820, 2646], 0, 32768.0, 1.0),
}


def _post_ref(x64, w64, b64, lo, n):
    """tanh(conv1d(reflect_pad3(lrelu(x, 0.2)), w) + b)[lo : lo + n] in float64, x64 [S][64], and the sum of the
    magnitudes of the 449 terms inside the tanh (the scale of the kernel's fp32 rounding; tanh' <= 1)"""
    a = torch.where(x64 > 0, x64, x64 * float(torch.tensor(0.2, dtype=torch.float32)))
    a = F.pad(a.t()[None], (3, 3), mode="reflect")
    y = F.conv1d(a, w64.t()[None]) + b64
    mag = F.conv1d(a.abs(), w64.abs().t()[None]) + b64.abs()
    return torch.tanh(y[0, 0, lo:lo + n]), mag[0, 0, lo:lo + n]


@pytest.mark.parametrize("case", sorted(POST_CASES))
def test_voc_post(case, record_property):
    """LeakyReLU 0.2, ReflectionPad1d(3), Conv1d(64 -> 1, k7), tanh, the centred trim and x scale against float64:
    the smallest generated length (Tc = 6, 2646 samples), lo = 0 with reflection at both ends (as vfx_vocoder /
    vfx_oracle use it), trims with odd and even S - out_len, out_len not a multiple of 16 or of 1024, ragged ext_gen /
    ext_len with per-item centred trims, scale 1 and 2^15, inputs that saturate tanh and inputs that keep it linear.
    The error |out / scale - ref| / (1 + sum of the terms' magnitudes) is checked over each item and separately in its
    first and last 8 samples, where the reflected rows enter (the 1 covers tanhf's own rounding).  Measured on the H100:
    at most 3.8e-8 over the items (saturating inputs, an absolute 1.2e-5), 1.9e-8 at the edges.  Reflecting one row off
    at the start gives 1.4e-3 and more.  Exact: samples from L_b to out_len are 0, and
    nothing past B x out_len is written."""
    gen, out_len, trims, lo, scale, xs = POST_CASES[case]
    B, S = len(gen), max(gen)
    g = _gen(len(case) * 13 + S)
    x = (xs * torch.randn(B, S, 64, generator=g)).to(DEV)
    w = (torch.randn(7, 64, generator=g) / math.sqrt(448) * 2).to(DEV)
    bias = (0.1 * torch.randn(1, generator=g)).to(DEV)
    for b, Sb in enumerate(gen):
        x[b, Sb:] = NAN                                   # rows past an item's generated length are never read
    ragged = trims is not None
    ext_gen = torch.tensor(gen, dtype=torch.int32, device=DEV) if ragged else None
    ext_len = torch.tensor(trims, dtype=torch.int32, device=DEV) if ragged else None
    out = torch.full((B * out_len + 64,), SENT, device=DEV)
    _call("vfx_voc_post", _ptr(x), B, S, _ptr(w), _ptr(bias), lo, out_len, _ptr(ext_gen), _ptr(ext_len),
          ctypes.c_float(scale), _ptr(out))
    assert bool((out[-64:] == SENT).all())
    o = out[:-64].view(B, out_len)
    worst = worst_edge = 0.0
    for b, Sb in enumerate(gen):
        Lb = trims[b] if ragged else out_len
        lo_b = (Sb - Lb) // 2 if ragged else lo
        ref, mag = _post_ref(x[b, :Sb].to(F64), w.to(F64), bias.to(F64), lo_b, Lb)
        err = (o[b, :Lb].to(F64) / scale - ref).abs() / (1 + mag)
        assert bool((o[b, Lb:] == 0).all())
        worst = max(worst, _worst(err))
        worst_edge = max(worst_edge, _worst(err[:8]), _worst(err[-8:]))
    record_property("max_err", worst)
    record_property("edge_max_err", worst_edge)
    assert worst < POST_TOL and worst_edge < POST_TOL
