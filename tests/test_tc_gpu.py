"""GPU tests of the wgmma conv-GEMM kernel (impl=1) through the C ABI, in every operand format
(bf16 / fp16; tf32 on fp32 storage pre-rounded to tf32).

bf16 x bf16 and tf32 x tf32 products are exact in fp32, so against an fp32 torch conv of the SAME rounded
operands only the accumulation order differs: tolerance 2e-5 relative RMS on the fp32 output; the activated
operand output carries one more rounding: bf16 4e-3, tf32 5e-4."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conftest import golden, rel_rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _op(t, prec):
    """Operand in the storage format of `prec` (rounded), and its exact fp32 value."""
    if prec == "bf16":
        q = t.bfloat16()
        return q, q.float()
    if prec == "fp16":
        q = t.half()
        return q, q.float()
    from voicefixer_b200.weights import round_tf32
    q = round_tf32(t.cpu()).to(DEV)
    return q, q


ACT_TOL = {"bf16": 4e-3, "tf32": 5e-4, "fp16": 5e-4}
PRECS = ["bf16", "tf32", "fp16"]


@pytest.mark.parametrize("C,L,dil,B", [(64, 128, 1, 1), (64, 700, 3, 2), (128, 1000, 27, 1), (256, 333, 243, 2),
                                       (512, 200, 2187, 1), (64, 5000, 81, 3)])
@pytest.mark.parametrize("prec", PRECS)
def test_tc_conv1d_dilated(C, L, dil, B, prec):
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x, xf = _op(_rnd(B, C, L, seed=1), prec)
    w, wf = _op(_rnd(C, C, 3, seed=2, scale=0.1), prec)
    b = _rnd(C, seed=3)
    res = _rnd(B, L, C, seed=4)
    ref = F.conv1d(xf, wf, b, dilation=dil, padding=dil) + res.permute(0, 2, 1)
    a = x.permute(0, 2, 1).contiguous()[:, None]
    wp = w.permute(2, 0, 1).contiguous()
    raw, act = conv_gemm(a, wp, [(0, -dil), (0, 0), (0, dil)], bias=b, residual=res[:, None].contiguous(),
                         want_act=True, act="lrelu", act_param=0.01, precision=prec, impl=1)
    assert rel_rms(raw[:, 0].permute(0, 2, 1).cpu(), ref.cpu()) < 2e-5
    assert rel_rms(act[:, 0].permute(0, 2, 1).float().cpu(), F.leaky_relu(ref, 0.01).cpu()) < ACT_TOL[prec]
    if prec == "tf32":      # the operand output is exactly representable in tf32 (low 13 mantissa bits zero)
        assert int((act.view(torch.int32) & 0x1FFF).abs().max()) == 0


@pytest.mark.parametrize("prec", PRECS)
def test_tc_conv1d_act_only_output(prec):
    """conv1 of a ResStack pair: activated operand out only (no raw / residual): exercises the double-buffered
    operand staging of the TMA epilogue."""
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    C, L, dil, B = 64, 3000, 9, 2
    x, xf = _op(_rnd(B, C, L, seed=21), prec)
    w, wf = _op(_rnd(C, C, 3, seed=22, scale=0.1), prec)
    b = _rnd(C, seed=23)
    ref = F.leaky_relu(F.conv1d(xf, wf, b, dilation=dil, padding=dil), 0.01)
    a = x.permute(0, 2, 1).contiguous()[:, None]
    _, act = conv_gemm(a, w.permute(2, 0, 1).contiguous(), [(0, -dil), (0, 0), (0, dil)], bias=b, want_raw=False,
                       want_act=True, act="lrelu", act_param=0.01, precision=prec, impl=1)
    assert rel_rms(act[:, 0].permute(0, 2, 1).float().cpu(), ref.cpu()) < ACT_TOL[prec]


@pytest.mark.parametrize("Cin,Cout,H,W", [(32, 32, 64, 127), (64, 64, 32, 63), (128, 64, 16, 31), (64, 128, 24, 15),
                                          (256, 256, 16, 7), (384, 384, 32, 3)])
@pytest.mark.parametrize("prec", PRECS)
def test_tc_conv2d_3x3(Cin, Cout, H, W, prec):
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    x, xf = _op(_rnd(2, Cin, H, W, seed=5), prec)
    w, wf = _op(_rnd(Cout, Cin, 3, 3, seed=6, scale=0.1), prec)
    ref = F.conv2d(xf, wf, padding=1)
    a = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    taps = [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)]
    raw, _ = conv_gemm(a, wp, taps, precision=prec, impl=1)
    assert rel_rms(raw.permute(0, 3, 1, 2).cpu(), ref.cpu()) < 2e-5


@pytest.mark.parametrize("u,Cin,Cout,L", [(7, 128, 64, 300), (3, 64, 64, 1000)])
@pytest.mark.parametrize("prec", PRECS)
def test_tc_conv_transpose1d(u, Cin, Cout, L, prec):
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    x, xf = _op(_rnd(2, Cin, L, seed=7), prec)
    w, wf = _op(_rnd(Cin, Cout, 2 * u, seed=8, scale=0.1), prec)
    b = _rnd(Cout, seed=9)
    pad = u // 2 + u % 2
    ref = F.conv_transpose1d(xf, wf, b, stride=u, padding=pad, output_padding=u % 2)
    a = x.permute(0, 2, 1).contiguous()[:, None]
    wp = w.permute(2, 1, 0).contiguous()
    mat, nA = Cout * Cin, u - pad
    out = torch.zeros(2, 1, u * L, Cout, device=DEV)
    conv_gemm(a, wp, [(0, 0), (0, -1)], N=nA * Cout, w_off=[pad * mat, (pad + u) * mat], bias=b, bias_mod=Cout,
              sw=u, rw=0, OW=u * L, out_ld=Cout, out_raw=out, precision=prec, impl=1)
    conv_gemm(a, wp, [(0, 1), (0, 0)], N=(u - nA) * Cout, w_off=[0, u * mat], bias=b, bias_mod=Cout,
              sw=u, rw=nA, OW=u * L, out_ld=Cout, out_raw=out, precision=prec, impl=1)
    assert rel_rms(out[:, 0].permute(0, 2, 1).cpu(), ref.cpu()) < 2e-5


@pytest.mark.parametrize("prec", PRECS)
def test_tc_conv_transpose2d_into_concat_buffer(prec):
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    Cin, Cout, H, W = 128, 64, 16, 31
    x, xf = _op(_rnd(2, Cin, H, W, seed=10), prec)
    w, wf = _op(_rnd(Cin, Cout, 3, 3, seed=11, scale=0.1), prec)
    ref = F.conv_transpose2d(xf, wf, stride=2)[:, :, :-1, :]
    OH, OW = 2 * H, 2 * W + 1
    a = x.permute(0, 2, 3, 1).contiguous()
    wp = w.permute(2, 3, 1, 0).reshape(9, Cout, Cin).contiguous()
    out = torch.zeros(2, OH, OW, 2 * Cout, device=DEV)          # first half of a concat buffer
    for rh in range(2):
        for rw in range(2):
            taps, offs = [], []
            for kh in ([1] if rh else [0, 2]):
                for kw in ([1] if rw else [0, 2]):
                    taps.append((-1 if kh == 2 else 0, -1 if kw == 2 else 0))
                    offs.append((kh * 3 + kw) * Cout * Cin)
            conv_gemm(a, wp, taps, Hq=H, Wq=W + 1, N=Cout, w_off=offs, sh=2, rh=rh, sw=2, rw=rw, OH=OH, OW=OW,
                      out_ld=2 * Cout, out_raw=out, precision=prec, impl=1)
    assert rel_rms(out[..., :Cout].permute(0, 3, 1, 2).cpu(), ref.cpu()) < 2e-5
    assert float(out[..., Cout:].abs().max()) == 0.0


@pytest.mark.parametrize("prec", PRECS)
def test_tc_wide_n_and_k7_valid_conv(prec):
    """N = 1024 (4 N-tiles of 256), 7 taps, 'valid' window on a padded input (vocoder pre-conv)."""
    from gpu_util import conv_gemm
    torch.backends.cudnn.allow_tf32 = False
    Cin, Cout, L = 512, 1024, 150
    x, xf = _op(_rnd(1, Cin, L + 6, seed=12), prec)
    w, wf = _op(_rnd(Cout, Cin, 7, seed=13, scale=0.05), prec)
    ref = F.conv1d(xf, wf)
    a = x.permute(0, 2, 1).contiguous()[:, None]
    wp = w.permute(2, 0, 1).contiguous()
    raw, _ = conv_gemm(a, wp, [(0, k) for k in range(7)], Wq=L, OW=L, precision=prec, impl=1)
    assert rel_rms(raw[:, 0].permute(0, 2, 1).cpu(), ref.cpu()) < 2e-5


def _enc(x, slope=0.01):
    """host form of the encoded tf32 stream: S = bits(lrelu(x)) + 0x1000 (include/vfx_b200.h)."""
    y = F.leaky_relu(x, slope).contiguous()
    return (y.view(torch.int32) + 0x1000).view(torch.float32)


def _dec(s, slope=0.01):
    y = (s.contiguous().view(torch.int32) - 0x1000).view(torch.float32)
    return torch.where(y > 0, y, y / slope)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("C,L,dil", [(64, 3000, 3), (128, 1000, 1), (256, 500, 243)])
def test_tf32_encoded_stream(C, L, dil, impl):
    """One fp32 tensor S as tf32 operand AND lossless residual carrier.  The UN-rounded S goes to the tensor core: this
    passes only if the tf32 tensor core ignores the low 13 mantissa bits (then the operand it sees is round-to-nearest(lrelu(x)))."""
    from gpu_util import conv_gemm
    from voicefixer_b200.weights import round_tf32
    torch.backends.cudnn.allow_tf32 = False
    B = 2
    x = _rnd(B, L, C, seed=31)
    S = _enc(x)
    assert torch.equal((S.view(torch.int32) & ~0x1FFF).view(torch.float32), round_tf32(F.leaky_relu(x, 0.01).cpu()).to(DEV))
    assert rel_rms(_dec(S).cpu(), x.cpu()) < 2e-7                       # the residual survives the encoding
    w, wf = _op(_rnd(C, C, 3, seed=32, scale=0.1), "tf32")
    b = _rnd(C, seed=33)
    a_ref = round_tf32(F.leaky_relu(x, 0.01).cpu()).to(DEV)
    ref = F.conv1d(a_ref.permute(0, 2, 1), wf, b, dilation=dil, padding=dil).permute(0, 2, 1) + x
    buf = S.clone()[:, None].contiguous()
    raw, _ = conv_gemm(buf, w.permute(2, 0, 1).contiguous(), [(0, -dil), (0, 0), (0, dil)], bias=b, residual=buf,
                       out_raw=torch.empty_like(buf), res_enc=1, raw_enc=1, enc_slope=0.01, precision="tf32", impl=impl)
    assert rel_rms(_dec(raw[:, 0]).cpu(), ref.cpu()) < 2e-5
    # and as the next operand it is exactly round-to-nearest(lrelu(result))
    got_op = (raw[:, 0].contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)
    assert rel_rms(got_op.cpu(), F.leaky_relu(ref, 0.01).cpu()) < 5e-4


# ---------------------------------------------------------------------------- tf32, width 128: the ResStack output forms
@pytest.mark.parametrize("mode", ["act", "enc", "xsinx", "plain"])
@pytest.mark.parametrize("L,dil,B", [(1000, 1, 2), (64, 3, 1), (63, 1, 1), (777, 9, 2), (5000, 27, 1), (3000, 81, 2),
                                     (9000, 2187, 1), (20000, 243, 3), (130, 729, 1)])
def test_tf32_c128_weights_in_tmem(L, dil, B, mode):
    """The C = 128 ResStack convolutions of the tf32 mode.  The four output forms the vocoder uses: activated operand only (conv1), encoded residual
    in / encoded stream out in place (conv2), encoded residual in / x + sin x operand out (last conv2 of a stack), plain
    residual / plain raw.  Against torch on the same tf32-rounded operands (fp32 accumulation: only the order differs)."""
    from gpu_util import conv_gemm
    from voicefixer_b200.weights import round_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    C = 128
    x = _rnd(B, L, C, seed=51)
    w, wf = _op(_rnd(C, C, 3, seed=52, scale=0.08), "tf32")
    b = _rnd(C, seed=53, scale=0.1)
    wp = w.permute(2, 0, 1).contiguous()
    taps = [(0, -dil), (0, 0), (0, dil)]
    if mode == "act":           # S stream in as the operand (un-rounded bits: the tensor core truncates), lrelu operand out
        S = _enc(x)
        a_ref = round_tf32(F.leaky_relu(x, 0.01).cpu()).to(DEV)
        ref = F.leaky_relu(F.conv1d(a_ref.permute(0, 2, 1), wf, b, dilation=dil, padding=dil), 0.01).permute(0, 2, 1)
        _, act = conv_gemm(S[:, None].contiguous(), wp, taps, bias=b, want_raw=False, want_act=True, act="lrelu",
                           act_param=0.01, precision="tf32", impl=1)
        assert rel_rms(act[:, 0].cpu(), ref.cpu()) < ACT_TOL["tf32"]
        assert int((act.view(torch.int32) & 0x1FFF).abs().max()) == 0
        return
    h, hf = _op(_rnd(B, L, C, seed=54), "tf32")                 # conv2's operand: the rounded intermediate
    conv = F.conv1d(hf.permute(0, 2, 1), wf, b, dilation=dil, padding=dil).permute(0, 2, 1)
    ref = x + conv
    a = h[:, None].contiguous()
    if mode == "enc":
        buf = _enc(x)[:, None].contiguous()
        raw, _ = conv_gemm(a, wp, taps, bias=b, residual=buf, out_raw=buf, res_enc=1, raw_enc=1, enc_slope=0.01,
                           precision="tf32", impl=1)
        assert rel_rms((_dec(raw[:, 0]) - x).cpu(), conv.cpu()) < 1e-4
    elif mode == "xsinx":
        buf = _enc(x)[:, None].contiguous()
        _, act = conv_gemm(a, wp, taps, bias=b, residual=buf, want_raw=False, want_act=True, act="lrelu_xsinx", act_param=0.2,
                           res_enc=1, enc_slope=0.01, precision="tf32", impl=1)
        u = F.leaky_relu(ref, 0.2)
        assert rel_rms(act[:, 0].cpu(), (u + torch.sin(u)).cpu()) < ACT_TOL["tf32"]
        assert torch.equal(buf[:, 0], _enc(x))                   # the residual stream is untouched
    else:
        res = x[:, None].contiguous()
        raw, _ = conv_gemm(a, wp, taps, bias=b, residual=res, precision="tf32", impl=1)
        assert rel_rms((raw[:, 0] - x).cpu(), conv.cpu()) < 2e-5
