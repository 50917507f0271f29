"""The wgmma convolution, the fused ResStack pair, the conv-GEMM epilogues and the GRU recurrence against float64
references of the same operation.

The other GPU tests compare with an fp32 torch result, whose rounding error is of the same order as the kernel's, so
a slightly wrong kernel passes them.  Here the reference is computed in float64 on exactly the operands the kernel
reads (bf16 / fp16 values, tf32-rounded fp32, fp32 bias and residual), so what remains is the kernel's own
accumulation and epilogue rounding.  Each convolution test asserts
  (a) raw fp32 output: relative RMS against float64 under a threshold set at least 3x above the worst value measured
      on an H100 80GB HBM3 (400 W power limit);
  (b) operand output (bf16 / fp16 / tf32): wherever the activation's input z is not tiny (|z| > CUT * RMS(z)), every
      element is the float64 result rounded to the format, or one of its two neighbours in that format;
  (c) memory the kernel must not write (the other half of a concat buffer, padding rows) still holds a sentinel.
The measured values quoted below come from that card; every input is seeded, so they repeat exactly.  Each test
records its statistics as pytest properties (written by --junitxml with -o junit_family=legacy).
"""
import ctypes
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "tf32": torch.float32, "fp32": torch.float32}
SENT = -1920.0                  # sentinel: exact in fp32, bf16, fp16 and tf32, and no kernel result
TC = ["bf16", "tf32", "fp16"]
# the epilogue tests run the wgmma kernel (impl 1) in every tensor-core format and the SIMT kernel (impl 0) in fp32 and bf16
EPI = [(1, "bf16"), (1, "tf32"), (1, "fp16"), (0, "fp32"), (0, "bf16")]

# (a) raw output, relative RMS against float64.  Worst measured: wgmma 2.2e-7 (vocoder pre-conv, tf32, K = 3584; the
# fused pair's update 1.5e-7), SIMT 7.2e-7 (fp32 operands, UNet 384 -> 384 3x3).
RAW_TOL = {"tc": 1e-6, "simt": 2.5e-6}
# (b) |z| / RMS(z) above which every operand element must be within one step of the rounded float64 result.  Below it
# the kernel's fp32 error can exceed a step of the format.  Measured: all elements are within one step above 5.9e-4
# (tf32 condnet ELU); 16-bit pair outputs above 4.1e-4.
CUT = 1e-3
# Group A: |mean((y - ref) sign(ref))| / mean|ref|.  Measured 4.8e-8 .. 8.9e-8 (all negative: the truncating adds
# inside one K slice); accumulating the whole K in the tensor core gives 2.4e-6 .. 7.3e-6.
BIAS_MAX = 5e-7
# Group D: kernel error <= 2 x torch's fp32 GRU error + GRU_CEIL (relative RMS against float64).  Measured: the kernel
# 6.7e-8 .. 8.0e-8, torch's fp32 GRU 6.7e-8 .. 9.8e-8; the largest ratio 1.003 (B = 1, T = 1).
GRU_CEIL = 1e-8


@pytest.fixture(autouse=True)
def _fp32_torch():
    """torch's own fp32 results (the GRU comparison) must not run in TF32."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _rnd(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _op(t, prec):
    """t (fp32) in the operand format of `prec`: the stored tensor and the exact value it holds, in float64."""
    from voicefixer_b200.weights import round_tf32
    if prec in ("bf16", "fp16"):
        q = t.to(DT[prec])
    elif prec == "tf32":
        q = round_tf32(t)
    else:
        q = t.clone()
    return q, q.to(F64)


def _rel(got, ref):
    """relative RMS of got against the float64 reference"""
    got, ref = got.to(F64), ref.to(F64)
    return float((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())


def _fmt_round(x64, prec):
    """float64 -> nearest value of the operand format, stored as the kernel stores it (tf32: ties away, cvt.rna)."""
    from voicefixer_b200.weights import round_tf32
    return round_tf32(x64.float()) if prec == "tf32" else x64.to(DT[prec])


def _ordinal(q, prec):
    """consecutive values of the format -> consecutive integers (+0 and -0 -> 0)"""
    if prec == "tf32":
        i = q.contiguous().view(torch.int32)
        mag = (i & 0x7FFFFFFF) >> 13
    else:
        i = q.contiguous().view(torch.int16).to(torch.int32)
        mag = i & 0x7FFF
    return torch.where(i < 0, -mag, mag)


def _check_operand(rec, got, z64, act64, prec, fp32_tol=None):
    """(b) for the operand output `got` of act64 = act(z64).  An fp32 operand (SIMT fp32) carries the raw output's
    error, so it is held to the raw tolerance instead."""
    if prec == "fp32":
        err = _rel(got, act64)
        rec("act_rel_rms", err)
        assert err < fp32_tol
        return
    if prec == "tf32":          # a tf32 operand has its low 13 mantissa bits clear
        assert int((got.contiguous().view(torch.int32) & 0x1FFF).abs().max()) == 0
    steps = (_ordinal(got, prec) - _ordinal(_fmt_round(act64, prec), prec)).abs()
    zrel = z64.abs() / z64.pow(2).mean().sqrt()
    bad = steps > 1
    rec("clean_cut", float(zrel[bad].max()) if bool(bad.any()) else 0.0)
    mask = zrel > CUT
    n_bad = int((bad & mask).sum())
    assert n_bad == 0, f"{n_bad} of {int(mask.sum())} {prec} elements are more than one step from float64"


def _conv(**kw):
    from gpu_util import conv_gemm
    return conv_gemm(**kw)


# ============================================================================ A. accumulation bias at the largest K
def _largest_k_case(shape, prec):
    """raw output of the wgmma kernel and its float64 reference, channels-last"""
    if shape.startswith("unet"):        # UNet 384 -> 384 3x3 at the last two levels (K = 9 x 384 = 3456)
        W = int(shape[-1])
        B, H, C = 2, 64 if W == 3 else 32, 384
        x, x64 = _op(_rnd(B, H, W, C, seed=101), prec)
        w, w64 = _op(_rnd(9, C, C, seed=102, scale=(9 * C) ** -0.5), prec)          # [tap][Cout][Cin]
        taps = [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)]
        raw, _ = _conv(a=x, w=w, taps=taps, precision=prec, impl=1)
        ref = F.conv2d(x64.permute(0, 3, 1, 2), w64.view(3, 3, C, C).permute(2, 3, 0, 1), padding=1)
        return raw, ref.permute(0, 2, 3, 1)
    # vocoder pre-conv: Conv1d(512, 1024, k7) on the reflect-padded condition (K = 7 x 512 = 3584)
    B, L = 2, 150
    x, x64 = _op(_rnd(B, L + 6, 512, seed=103), prec)
    w, w64 = _op(_rnd(7, 1024, 512, seed=104, scale=(7 * 512) ** -0.5), prec)
    raw, _ = _conv(a=x[:, None].contiguous(), w=w, taps=[(0, k) for k in range(7)], Wq=L, OW=L, precision=prec, impl=1)
    ref = F.conv1d(x64.permute(0, 2, 1), w64.permute(1, 2, 0))
    return raw[:, 0], ref.permute(0, 2, 1)


@pytest.mark.parametrize("prec", TC)
@pytest.mark.parametrize("shape", ["unet384_W3", "unet384_W7", "voc_pre"])
def test_accumulation_is_unbiased(shape, prec, record_property):
    """The tensor core's accumulator adds truncate; the kernel sums each 128-byte K slice's result into the running
    fp32 sum with round-to-nearest adds.  Accumulating the whole K in the tensor core instead shrinks every output
    systematically, which the relative RMS alone does not reveal: the signed statistic mean((y - ref) sign(ref)) /
    mean|ref| does.  Measured on the H100: at most 8.9e-8 in size with the split, at least 2.4e-6 without it
    (BIAS_MAX = 5e-7 lies about 5x from both)."""
    raw, ref = _largest_k_case(shape, prec)
    err = _rel(raw, ref)
    bias = float(((raw.to(F64) - ref) * ref.sign()).mean() / ref.abs().mean())
    record_property("raw_rel_rms", err)
    record_property("bias", bias)
    assert err < RAW_TOL["tc"]
    assert abs(bias) < BIAS_MAX


# ============================================================================ B. fused ResStack pair
_SCRATCH = {}


def _pair(prec, form, a, x, w1, b1, w2, b2, dil, write_raw=1, out_act=None, act="lrelu", act_param=0.01, x_out=None,
          stream_enc=0, stream_enc_out=0):
    """vfx_resstack_pair in form "fused" or "blocked"; weights [3][C][C] (tap, out, in)"""
    from voicefixer_b200 import _lib
    lib = _lib.load()
    B, L, C = x.shape
    d = _lib.PairDesc()
    d.a, d.x = a.data_ptr(), x.data_ptr()
    d.w1, d.b1, d.dilation, d.w2, d.b2 = w1.data_ptr(), b1.data_ptr(), dil, w2.data_ptr(), b2.data_ptr()
    d.B, d.L, d.C, d.write_raw = B, L, C, write_raw
    d.out_act = None if out_act is None else out_act.data_ptr()
    d.act, d.act_param = _lib.ACT[act], act_param
    d.precision, d.form = _lib.PREC[prec], _lib.PAIR_FORM[form]
    d.x_out = None if x_out is None else x_out.data_ptr()
    d.stream_enc, d.stream_enc_out = stream_enc, stream_enc_out
    if form == "blocked":
        n = int(lib.vfx_resstack_pair_scratch_bytes())
        if "buf" not in _SCRATCH:
            _SCRATCH["buf"] = torch.empty(n, dtype=torch.uint8, device=DEV)
        d.scratch, d.scratch_bytes = _SCRATCH["buf"].data_ptr(), n
    _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "vfx_resstack_pair")
    torch.cuda.synchronize()


def _pair_operands(B, L, C, prec, seed):
    """a and W1 / b1 are small integers (times 2^-6): every partial sum of conv1 is exact in fp32, in any order, so the
    kernel's intermediate h = lrelu(conv1 + b1) rounds to the operand format exactly as the reference's does.  (With
    arbitrary operands an h within the kernel's error of a rounding midpoint flips by one step, and those flips, not
    the accumulation, would set the error.)  W2, b2 and x are continuous."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lim, *s: torch.randint(-lim, lim + 1, s, generator=g).float()
    a = ri(8, B, L, C).to(DEV).to(DT[prec])
    w1 = (ri(8, 3, C, C) / 64).to(DEV).to(DT[prec])
    b1 = (ri(64, C) / 64).to(DEV)
    w2 = (torch.randn(3, C, C, generator=g) * (0.3 / (3 * C) ** 0.5)).to(DEV).to(DT[prec])
    b2 = (torch.randn(C, generator=g) * 0.1).to(DEV)
    x = torch.randn(B, L, C, generator=g).to(DEV)
    return a, x, w1, b1, w2, b2


def _tw(w):
    """[tap][Cout][Cin] -> torch (Cout, Cin, tap), float64"""
    return w.to(F64).permute(1, 2, 0)


def _pair_ref(a, x, w1, b1, w2, b2, dil, prec):
    v = F.conv1d(a.to(F64).permute(0, 2, 1), _tw(w1), b1.to(F64), dilation=dil, padding=dil)
    v32 = v.float()
    assert torch.equal(v32.to(F64), v)                                   # conv1 + b1 is exact in fp32
    h = torch.where(v32 > 0, v32, v32 * torch.tensor(0.01, device=DEV)).to(DT[prec]).to(F64)
    return x.to(F64) + F.conv1d(h, _tw(w2), b2.to(F64), padding=1).permute(0, 2, 1)


def _act64(z, act, p):
    if act == "lrelu":
        return torch.where(z > 0, z, z * p)
    if act == "lrelu_xsinx":
        u = torch.where(z > 0, z, z * p)
        return u + torch.sin(u)
    if act == "elu":
        return torch.where(z > 0, z, torch.expm1(z))
    if act == "sigmoid":
        return 1.0 / (1.0 + torch.exp(-z))
    return z


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("dil", [1, 3, 243, 2187])
@pytest.mark.parametrize("L", [1, 125, 126, 127, 252, 253, 1000, 20000])
def test_pair128_fused(L, dil, B, prec, record_property):
    """Width 128, the fused form: tile edges at 126 rows, dilations up to beyond L, in place.  Measured on the H100:
    the update within 1.2e-7 .. 1.5e-7 relative RMS of float64."""
    C = 128
    a, x, w1, b1, w2, b2 = _pair_operands(B, L, C, prec, seed=L * 7 + dil * 3 + B)
    ref = _pair_ref(a, x, w1, b1, w2, b2, dil, prec)
    xin = x.clone()
    act = torch.full((B, L, C), SENT, dtype=DT[prec], device=DEV)
    _pair(prec, "fused", a, xin, w1, b1, w2, b2, dil, out_act=act)
    x64 = x.to(F64)
    err = _rel(xin.to(F64) - x64, ref - x64)              # the update itself, not masked by the residual
    record_property("raw_rel_rms", err)
    _check_operand(record_property, act, ref, _act64(ref, "lrelu", 0.01), prec)
    assert err < RAW_TOL["tc"]


@pytest.mark.parametrize("dest", ["in_place", "x_out"])
@pytest.mark.parametrize("act", ["lrelu", "lrelu_xsinx", "none", None])
@pytest.mark.parametrize("write_raw", [1, 0])
@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_pair128_output_variants(prec, write_raw, act, dest, record_property):
    """write_raw 0 / 1 x operand output (lrelu 0.01, x + sin x after lrelu 0.2, identity, none) x result in place / in
    x_out.  Whatever is not an output keeps its contents."""
    if act is None and not write_raw:
        pytest.skip("no output at all")
    C, L, B, dil = 128, 1000, 3, 27
    a, x, w1, b1, w2, b2 = _pair_operands(B, L, C, prec, seed=5)
    ref = _pair_ref(a, x, w1, b1, w2, b2, dil, prec)
    xin = x.clone()
    xout = torch.full_like(x, SENT) if dest == "x_out" else None
    out_act = None if act is None else torch.full((B, L, C), SENT, dtype=DT[prec], device=DEV)
    p = {"lrelu": 0.01, "lrelu_xsinx": 0.2}.get(act, 0.0)
    _pair(prec, "fused", a, xin, w1, b1, w2, b2, dil, write_raw=write_raw, out_act=out_act, act=act or "none",
          act_param=p, x_out=xout)
    x64 = x.to(F64)
    if write_raw:
        got = xout if dest == "x_out" else xin
        err = _rel(got.to(F64) - x64, ref - x64)
        record_property("raw_rel_rms", err)
        assert err < RAW_TOL["tc"]
    if dest == "x_out" or not write_raw:
        assert torch.equal(xin, x)                                      # x is only read
    if dest == "x_out" and not write_raw:
        assert bool((xout == SENT).all())
    if act is not None:
        _check_operand(record_property, out_act, ref, _act64(ref, act, p), prec)


def _enc(x, slope=0.01):
    """host form of the encoded tf32 stream: S = bits(lrelu(x)) + 0x1000 (include/vfx_b200.h)"""
    y = F.leaky_relu(x, slope).contiguous()
    return (y.view(torch.int32) + 0x1000).view(torch.float32)


def _dec(s, slope=0.01):
    y = (s.contiguous().view(torch.int32) - 0x1000).view(torch.float32)
    return torch.where(y > 0, y, y / slope)


@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("prec", ["bf16", "fp16"])
def test_pair_fused_and_blocked_are_bit_identical(prec, C):
    """The fused form (one kernel, h in shared memory) and the blocked form (two conv-GEMM launches, h in the scratch)
    use the same instruction shape, the same K order and the same epilogue expression order: their results are the same
    bits."""
    B, L, dil = 2, 3000, 9
    x = _rnd(B, L, C, seed=61)
    a = F.leaky_relu(x, 0.01).to(DT[prec])
    w1, _ = _op(_rnd(3, C, C, seed=62, scale=0.08), prec)
    w2, _ = _op(_rnd(3, C, C, seed=63, scale=0.08), prec)
    b1, b2 = _rnd(C, seed=64, scale=0.1), _rnd(C, seed=65, scale=0.1)
    outs = []
    for form in ("fused", "blocked"):
        xin = x.clone()
        act = torch.full((B, L, C), SENT, dtype=DT[prec], device=DEV)
        _pair(prec, form, a, xin, w1, b1, w2, b2, dil, out_act=act)
        outs.append((xin, act))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1].view(torch.int16), outs[1][1].view(torch.int16))


@pytest.mark.parametrize("enc_out", [1, 0])
def test_pair_tf32_fused_and_blocked_are_bit_identical(enc_out):
    """tf32 on the encoded stream: the fused and the blocked form give the same bits (the blocked form
    decodes the residual with 1 / 0.01f, which is 100.0f exactly as the fused one)."""
    from voicefixer_b200.weights import round_tf32
    B, L, C, dil = 2, 5000, 64, 27
    S = _enc(_rnd(B, L, C, seed=71))
    w1, w2 = round_tf32(_rnd(3, C, C, seed=72, scale=0.08)), round_tf32(_rnd(3, C, C, seed=73, scale=0.08))
    b1, b2 = _rnd(C, seed=74, scale=0.1), _rnd(C, seed=75, scale=0.1)
    outs = []
    for form in ("fused", "blocked"):
        out = torch.full_like(S, SENT)
        _pair("tf32", form, S, S, w1, b1, w2, b2, dil, x_out=out, stream_enc=1, stream_enc_out=enc_out)
        outs.append(out)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))


# ============================================================================ C. epilogues at the engine's layouts
def _raw_tol(impl):
    return RAW_TOL["tc"] if impl == 1 else RAW_TOL["simt"]


@pytest.mark.parametrize("impl,prec", EPI)
@pytest.mark.parametrize("slope", [0.01, 0.0])
@pytest.mark.parametrize("C,W", [(32, 127), (32, 63), (32, 3), (384, 127), (384, 63), (384, 3)])
def test_unet_conv2_epilogue(C, W, slope, impl, prec, record_property):
    """ConvBlockRes conv2 as the engine runs it: residual read from the second half of a pitch-2C concat buffer, raw
    result into column C of a pitch-2C buffer, and the next block's eval BatchNorm (act_scale / act_shift) with
    LeakyReLU 0.01 or ReLU (slope 0) fused into the dense operand output."""
    B, H = 2, {127: 8, 63: 16, 3: 64}[W]
    x, x64 = _op(_rnd(B, H, W, C, seed=81), prec)
    w, w64 = _op(_rnd(9, C, C, seed=82, scale=(9 * C) ** -0.5), prec)
    resbuf = _rnd(B, H, W, 2 * C, seed=83)
    scale, shift = 0.5 + _rnd(C, seed=84).abs(), _rnd(C, seed=85, scale=0.3)
    out = torch.full((B, H, W, 2 * C), SENT, device=DEV)
    act = torch.full((B, H, W, C), SENT, dtype=DT[prec], device=DEV)
    taps = [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)]
    _conv(a=x, w=w, taps=taps, residual=resbuf[..., C:], out_ld=2 * C, out_col=C, out_raw=out, want_act=True,
          out_act=act, act_ld=C, act_col=0, act="lrelu", act_param=slope, act_scale=scale, act_shift=shift,
          precision=prec, impl=impl)
    z = F.conv2d(x64.permute(0, 3, 1, 2), w64.view(3, 3, C, C).permute(2, 3, 0, 1), padding=1).permute(0, 2, 3, 1)
    z = z + resbuf[..., C:].to(F64)
    err = _rel(out[..., C:], z)
    record_property("raw_rel_rms", err)
    assert bool((out[..., :C] == SENT).all())                            # (c) the other half of the concat buffer
    zb = z * scale.to(F64) + shift.to(F64)
    _check_operand(record_property, act, zb, _act64(zb, "lrelu", slope), prec, fp32_tol=2 * _raw_tol(impl))
    assert err < _raw_tol(impl)


@pytest.mark.parametrize("impl,prec", EPI)
@pytest.mark.parametrize("Cin", [128, 512])
def test_condnet_elu_into_padded_buffer(Cin, impl, prec, record_property):
    """Condnet Conv1d(k3) + ELU written at row 3 of a [B][Tc + 6][512] reflect-pad buffer (item stride (Tc + 6) x 512):
    the three padding rows at each end stay untouched."""
    B, Tc, N = 2, 200, 512
    x, x64 = _op(_rnd(B, 1, Tc, Cin, seed=91), prec)
    w, w64 = _op(_rnd(3, N, Cin, seed=92, scale=(3 * Cin) ** -0.5), prec)
    b = _rnd(N, seed=93, scale=0.5)
    buf = torch.full((B, Tc + 6, N), SENT, dtype=DT[prec], device=DEV)
    _conv(a=x, w=w, taps=[(0, -1), (0, 0), (0, 1)], bias=b, want_raw=False, want_act=True, out_act=buf[:, 3:],
          act="elu", act_sB=(Tc + 6) * N, precision=prec, impl=impl)
    z = F.conv1d(x64[:, 0].permute(0, 2, 1), _tw(w64), b.to(F64), padding=1).permute(0, 2, 1)
    assert bool((buf[:, :3] == SENT).all()) and bool((buf[:, Tc + 3:] == SENT).all())      # (c)
    _check_operand(record_property, buf[:, 3:Tc + 3], z, _act64(z, "elu", 0.0), prec, fp32_tol=2 * _raw_tol(impl))


@pytest.mark.parametrize("impl,prec", EPI)
@pytest.mark.parametrize("Ci,Co,u,Lin", [(1024, 512, 7, 64), (128, 64, 3, 1000)])
def test_upsampler_engine_formulation(Ci, Co, u, Lin, impl, prec, record_property):
    """ConvTranspose1d(k = 2u, stride u) as the engine runs it: the output seen as [B][Lin][u * Co], each phase group
    a stride-1 GEMM into columns [r0 * Co, (r0 + nph) * Co) of pitch u * Co.  tf32 writes the encoded stream
    (raw_enc), which is decoded and compared, and whose tf32 operand view is checked as an operand output."""
    B = 2
    enc = prec == "tf32"
    x, x64 = _op(_rnd(B, 1, Lin, Ci, seed=111), prec)
    w, w64 = _op(_rnd(2 * u, Co, Ci, seed=112, scale=(2 * Ci) ** -0.5), prec)        # [k][Co][Ci]
    b = _rnd(Co, seed=113, scale=0.5)
    raw = torch.full((B, 1, Lin, u * Co), SENT, device=DEV)
    act = None if enc else torch.full((B, 1, Lin, u * Co), SENT, dtype=DT[prec], device=DEV)
    pad = u // 2 + u % 2
    nA, mat = u - pad, Co * Ci
    for grp in range(2):
        if grp == 0:
            taps, offs, r0, nph = [(0, 0), (0, -1)], [pad * mat, (pad + u) * mat], 0, nA
        else:
            taps, offs, r0, nph = [(0, 1), (0, 0)], [0, u * mat], nA, u - nA
        _conv(a=x, w=w, taps=taps, N=nph * Co, w_off=offs, bias=b, bias_mod=Co, out_ld=u * Co, out_col=r0 * Co,
              out_raw=raw, want_act=not enc, out_act=act, act="lrelu", act_param=0.01, raw_enc=int(enc),
              enc_slope=0.01 if enc else 0.0, precision=prec, impl=impl)
    z = F.conv_transpose1d(x64[:, 0].permute(0, 2, 1), w64.permute(2, 1, 0), b.to(F64), stride=u, padding=pad,
                           output_padding=u % 2).permute(0, 2, 1)                   # (B, u * Lin, Co)
    got = (_dec(raw) if enc else raw).reshape(B, Lin * u, Co)
    err = _rel(got, z)
    record_property("raw_rel_rms", err)
    assert err < _raw_tol(impl)
    if enc:     # the operand conv1 reads from the stream: its low 13 bits ignored = round-to-nearest(lrelu(x))
        opnd = (raw.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)
        _check_operand(record_property, opnd.reshape(B, Lin * u, Co), z, _act64(z, "lrelu", 0.01), "tf32")
    else:
        _check_operand(record_property, act.reshape(B, Lin * u, Co), z, _act64(z, "lrelu", 0.01), prec,
                       fp32_tol=2 * _raw_tol(impl))


@pytest.mark.parametrize("impl,prec", EPI)
@pytest.mark.parametrize("act,p", [("sigmoid", 0.0), ("lrelu_xsinx", 0.2)])
def test_linear_sigmoid_and_xsinx(act, p, impl, prec, record_property):
    """1-tap linear layer with the sigmoid and x + sin x epilogues; N = 192 leaves a partial N tile."""
    B, L, Cin, N = 2, 500, 256, 192
    x, x64 = _op(_rnd(B, 1, L, Cin, seed=121), prec)
    w, w64 = _op(_rnd(1, N, Cin, seed=122, scale=2 * Cin ** -0.5), prec)
    b = _rnd(N, seed=123, scale=0.5)
    out = torch.full((B, 1, L, N), SENT, dtype=DT[prec], device=DEV)
    raw, _ = _conv(a=x, w=w, taps=[(0, 0)], bias=b, want_act=True, out_act=out, act=act, act_param=p,
                   precision=prec, impl=impl)
    z = (x64 @ w64[0].t() + b.to(F64))
    err = _rel(raw, z)
    record_property("raw_rel_rms", err)
    assert err < _raw_tol(impl)
    _check_operand(record_property, out, z, _act64(z, act, p), prec, fp32_tol=2 * _raw_tol(impl))


# ============================================================================ D. GRU recurrence
def _torch_gru(gi, whh, bhh, dtype):
    """torch.nn.GRU driven by the given input projections: the input weights are [I | 0] and [0 | I] on the input
    gi viewed as [B][T][1536], with zero input bias, so gi reaches the gates exactly."""
    B, T = gi.shape[:2]
    m = torch.nn.GRU(1536, 256, bidirectional=True, batch_first=True).to(DEV, dtype)
    eye, zero = torch.eye(768, dtype=dtype, device=DEV), torch.zeros(768, 768, dtype=dtype, device=DEV)
    with torch.no_grad():
        m.weight_ih_l0.copy_(torch.cat([eye, zero], 1))
        m.weight_ih_l0_reverse.copy_(torch.cat([zero, eye], 1))
        m.bias_ih_l0.zero_()
        m.bias_ih_l0_reverse.zero_()
        m.weight_hh_l0.copy_(whh[0])
        m.weight_hh_l0_reverse.copy_(whh[1])
        m.bias_hh_l0.copy_(bhh[0])
        m.bias_hh_l0_reverse.copy_(bhh[1])
        y, _ = m(gi.reshape(B, T, 1536).to(dtype))
    return y


def _gru_kernel(gi, whh_t, bhh):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    B, T = gi.shape[:2]
    out = torch.full((B, T, 512), SENT, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(lib.vfx_gru_layer(p(gi), p(whh_t), p(bhh), B, T, p(out), None), "vfx_gru_layer")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("T", [1, 2, 1001])
@pytest.mark.parametrize("B", [1, 16, 17, 32, 33, 64])
def test_gru_layer_fp64(B, T, record_property):
    """All three cluster tiers (G = 2 up to B = 16, 4 up to 32, 8 above) with full and partial last groups, and the
    shortest sequences (T = 1, 2: the prefetch ring and the last step).  The kernel's error against float64 must stay
    within twice torch's own fp32 GRU's, and every item must come out bit-identical to the same item run alone:
    a sequence's FMA order depends neither on G nor on its place in the group.  Measured on the H100: kernel 6.7e-8 ..
    8.0e-8 relative RMS against float64, torch's fp32 GRU 6.7e-8 .. 9.8e-8."""
    g = torch.Generator().manual_seed(1000 + B + T)
    gi = torch.randn(B, T, 2, 768, generator=g).to(DEV)
    whh = ((torch.rand(2, 768, 256, generator=g) * 2 - 1) / 16).to(DEV)          # torch's GRU init range
    bhh = ((torch.rand(2, 768, generator=g) * 2 - 1) / 16).to(DEV)
    whh_t = whh.transpose(1, 2).contiguous()
    out = _gru_kernel(gi, whh_t, bhh)
    with torch.backends.cudnn.flags(enabled=False):
        ref = _torch_gru(gi.to(F64), whh.to(F64), bhh.to(F64), F64)
    t32 = _torch_gru(gi, whh, bhh, torch.float32)
    err, err_t = _rel(out, ref), _rel(t32, ref)
    record_property("gru_rel_rms", err)
    record_property("torch_fp32_rel_rms", err_t)
    assert err <= 2 * err_t + GRU_CEIL
    for b in range(B):
        alone = _gru_kernel(gi[b:b + 1].contiguous(), whh_t, bhh)
        assert torch.equal(alone[0], out[b]), f"item {b} of {B} differs from the same item run alone"
