"""GPU tests of the ResStack pair entry point (vfx_resstack_pair) through the C ABI: the fused kernel (h kept in shared
memory) and, where a test asks for it, the blocked form (conv1 -> h in the caller's scratch -> conv2 + residual, on the
tensor-core convolution), against the same arithmetic spelled out with torch ops: 16-bit (or tf32-rounded) operands
(a, h, weights), fp32 accumulation, fp32 residual stream.  Reference op: ResStack.forward
voicefixer/vocoder/model/modules.py:592-595.

Tolerances: fp32 output 1e-4 relative RMS (bf16 x bf16 products are exact in fp32; a rare bf16 rounding tie of the
intermediate h may flip against torch's), activated bf16 output 4e-3 (one bf16 rounding)."""
import ctypes
import pytest
import torch
import torch.nn.functional as F
from conftest import rel_rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _pair(x, a, w1, b1, w2, b2, dil, write_raw=True, act="lrelu", act_param=0.01, want_act=True, prec="bf16"):
    """x (B,L,C) fp32 [updated in place], a (B,L,C) bf16 / fp16, w (C,C,3) same format, torch layout."""
    from voicefixer_b200 import _lib
    lib = _lib.load()
    B, L, C = x.shape
    d = _lib.PairDesc()
    w1p, w2p = w1.permute(2, 0, 1).contiguous(), w2.permute(2, 0, 1).contiguous()
    out_act = torch.zeros(B, L, C, device=DEV, dtype=a.dtype) if want_act else None
    d.a, d.x = a.data_ptr(), x.data_ptr()
    d.w1, d.b1, d.dilation, d.w2, d.b2 = w1p.data_ptr(), b1.data_ptr(), dil, w2p.data_ptr(), b2.data_ptr()
    d.B, d.L, d.C, d.write_raw = B, L, C, int(write_raw)
    d.out_act = out_act.data_ptr() if want_act else None
    d.act, d.act_param = _lib.ACT[act], act_param
    d.precision = _lib.PREC[prec]
    d.scratch, d.scratch_bytes = _scratch(lib)
    _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "vfx_resstack_pair")
    torch.cuda.synchronize()
    return out_act


_SCRATCH = {}


def _scratch(lib):
    n = int(lib.vfx_resstack_pair_scratch_bytes())
    if "buf" not in _SCRATCH:
        _SCRATCH["buf"] = torch.empty(n, dtype=torch.uint8, device=DEV)
    return _SCRATCH["buf"].data_ptr(), n


def _ref(x, a, w1, b1, w2, b2, dil):
    h = F.leaky_relu(F.conv1d(a.float().permute(0, 2, 1), w1.float(), b1, dilation=dil, padding=dil), 0.01)
    h = h.to(a.dtype).float()
    return x + F.conv1d(h, w2.float(), b2, padding=1).permute(0, 2, 1)


@pytest.mark.parametrize("L,dil,B", [(1000, 1, 2), (5000, 3, 1), (300, 27, 2), (378, 9, 1), (4000, 81, 2),
                                     (9000, 2187, 1), (125, 1, 1), (127, 729, 1), (20000, 243, 3)])
def test_pair_matches_two_convolutions(L, dil, B):
    torch.backends.cudnn.allow_tf32 = False
    C = 64
    x = _rnd(B, L, C, seed=1)
    a = F.leaky_relu(x, 0.01).bfloat16()
    w1, w2 = _rnd(C, C, 3, seed=2, scale=0.08).bfloat16(), _rnd(C, C, 3, seed=3, scale=0.08).bfloat16()
    b1, b2 = _rnd(C, seed=4, scale=0.1), _rnd(C, seed=5, scale=0.1)
    ref = _ref(x, a, w1, b1, w2, b2, dil)
    xin = x.clone()
    act = _pair(xin, a, w1, b1, w2, b2, dil)
    assert rel_rms((xin - x).cpu(), (ref - x).cpu()) < 1e-4            # the update itself, not masked by the residual
    assert rel_rms(act.float().cpu(), F.leaky_relu(ref, 0.01).cpu()) < 4e-3


@pytest.mark.parametrize("L,dil,B", [(3000, 3, 2), (4000, 243, 1)])
def test_pair_fp16_operands(L, dil, B):
    """The other 16-bit operand format: fp16 a / h / weights (tf32's mantissa in 2 bytes)."""
    torch.backends.cudnn.allow_tf32 = False
    C = 64
    x = _rnd(B, L, C, seed=1)
    a = F.leaky_relu(x, 0.01).half()
    w1, w2 = _rnd(C, C, 3, seed=2, scale=0.08).half(), _rnd(C, C, 3, seed=3, scale=0.08).half()
    b1, b2 = _rnd(C, seed=4, scale=0.1), _rnd(C, seed=5, scale=0.1)
    ref = _ref(x, a, w1, b1, w2, b2, dil)
    xin = x.clone()
    act = _pair(xin, a, w1, b1, w2, b2, dil, prec="fp16")
    assert rel_rms((xin - x).cpu(), (ref - x).cpu()) < 1e-4
    assert rel_rms(act.float().cpu(), F.leaky_relu(ref, 0.01).cpu()) < 5e-4


def test_pair_output_variants():
    """operand-only output with the next up-sampler's activation (no raw write), and raw-only output (last pair)."""
    torch.backends.cudnn.allow_tf32 = False
    C, L, B, dil = 64, 3000, 2, 9
    x = _rnd(B, L, C, seed=11)
    a = F.leaky_relu(x, 0.01).bfloat16()
    w1, w2 = _rnd(C, C, 3, seed=12, scale=0.08).bfloat16(), _rnd(C, C, 3, seed=13, scale=0.08).bfloat16()
    b1, b2 = _rnd(C, seed=14, scale=0.1), _rnd(C, seed=15, scale=0.1)
    ref = _ref(x, a, w1, b1, w2, b2, dil)
    xin = x.clone()
    act = _pair(xin, a, w1, b1, w2, b2, dil, write_raw=False, act="lrelu_xsinx", act_param=0.2)
    assert torch.equal(xin, x)                                          # x untouched
    u = F.leaky_relu(ref, 0.2)
    assert rel_rms(act.float().cpu(), (u + torch.sin(u)).cpu()) < 4e-3
    xin = x.clone()
    assert _pair(xin, a, w1, b1, w2, b2, dil, want_act=False) is None
    assert rel_rms((xin - x).cpu(), (ref - x).cpu()) < 1e-4


def test_pair_rejects_other_widths():
    """Widths other than the vocoder's last two ResStacks (64, 128) are refused, not mis-computed."""
    from voicefixer_b200._lib import VfxError
    x = _rnd(1, 200, 256, seed=21)
    a = x.bfloat16()
    w = _rnd(256, 256, 3, seed=22).bfloat16()
    b = _rnd(256, seed=23)
    with pytest.raises(VfxError, match="unsupported"):
        _pair(x, a, w, b, w, b, 1)


# ---------------------------------------------------------------------------- width 128 and the scratch
def test_blocked_pair_needs_scratch():
    from voicefixer_b200 import _lib
    from voicefixer_b200._lib import VfxError
    lib = _lib.load()
    x = _rnd(1, 300, 128, seed=1)
    a = x.bfloat16()
    w = _rnd(3, 128, 128, seed=2).bfloat16()
    b = _rnd(128, seed=3)
    act = torch.zeros_like(a)
    d = _lib.PairDesc()
    d.a, d.x, d.w1, d.b1, d.dilation, d.w2, d.b2 = a.data_ptr(), x.data_ptr(), w.data_ptr(), b.data_ptr(), 1, w.data_ptr(), b.data_ptr()
    d.B, d.L, d.C, d.write_raw, d.out_act, d.act, d.act_param, d.precision = 1, 300, 128, 1, act.data_ptr(), 1, 0.01, 1
    d.form = _lib.PAIR_FORM["blocked"]
    with pytest.raises(VfxError, match="scratch"):
        _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), None), "pair2")


def _desc(lib_mod, **kw):
    d = lib_mod.PairDesc()
    for k, v in kw.items():
        setattr(d, k, v)
    d.scratch, d.scratch_bytes = _scratch(lib_mod.load())
    return d


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
@pytest.mark.parametrize("C,L,dil,B", [(128, 1000, 1, 2), (128, 5000, 27, 1), (128, 700, 243, 2), (128, 20000, 9, 3),
                                       (128, 9000, 2187, 1), (128, 125, 1, 1)])
def test_pair2_16bit_matches_two_convolutions(C, L, dil, B, prec):
    """Width 128: same arithmetic as width 64."""
    from voicefixer_b200 import _lib
    lib = _lib.load()
    torch.backends.cudnn.allow_tf32 = False
    dt = torch.bfloat16 if prec == "bf16" else torch.float16
    x = _rnd(B, L, C, seed=1)
    a = F.leaky_relu(x, 0.01).to(dt)
    w1, w2 = _rnd(C, C, 3, seed=2, scale=0.06).to(dt), _rnd(C, C, 3, seed=3, scale=0.06).to(dt)
    b1, b2 = _rnd(C, seed=4, scale=0.1), _rnd(C, seed=5, scale=0.1)
    ref = _ref(x, a, w1, b1, w2, b2, dil)
    xin = x.clone()
    w1p, w2p = w1.permute(2, 0, 1).contiguous(), w2.permute(2, 0, 1).contiguous()
    act = torch.zeros(B, L, C, device=DEV, dtype=dt)
    d = _desc(_lib, a=a.data_ptr(), x=xin.data_ptr(), w1=w1p.data_ptr(), b1=b1.data_ptr(), dilation=dil, w2=w2p.data_ptr(),
              b2=b2.data_ptr(), B=B, L=L, C=C, write_raw=1, out_act=act.data_ptr(), act=_lib.ACT["lrelu"], act_param=0.01,
              precision=_lib.PREC[prec], form=_lib.PAIR_FORM["blocked"])
    _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pair2")
    torch.cuda.synchronize()
    assert rel_rms((xin - x).cpu(), (ref - x).cpu()) < 1e-4
    assert rel_rms(act.float().cpu(), F.leaky_relu(ref, 0.01).cpu()) < (4e-3 if prec == "bf16" else 5e-4)


def _enc(x, slope=0.01):
    y = F.leaky_relu(x, slope).contiguous()
    return (y.view(torch.int32) + 0x1000).view(torch.float32)


def _dec(s, slope=0.01):
    y = (s.contiguous().view(torch.int32) - 0x1000).view(torch.float32)
    return torch.where(y > 0, y, y / slope)


@pytest.mark.parametrize("form", ["fused", "blocked"])
@pytest.mark.parametrize("L,dil,B,enc_out", [(1000, 1, 2, 1), (5000, 81, 1, 1), (3000, 9, 2, 0), (20000, 729, 2, 1),
                                             (125, 1, 1, 1), (127, 3, 2, 0), (4000, 27, 1, 1), (9000, 2187, 1, 1),
                                             (40000, 243, 3, 1), (378, 9, 1, 1)])
def test_pair_tf32_encoded_stream(L, dil, B, enc_out, form):
    """tf32, C = 64: the encoded stream S is operand and residual carrier; the result goes to the other buffer as S' (or as
    plain x' for the last pair of a stack), by the fused kernel and by the blocked form (the two convolutions per row
    block through the scratch).  Reference: tf32-rounded operands and intermediate, fp32 accumulation."""
    from voicefixer_b200 import _lib
    from voicefixer_b200.weights import round_tf32
    lib = _lib.load()
    torch.backends.cudnn.allow_tf32 = False
    C = 64
    rt = lambda t: round_tf32(t.cpu()).to(DEV)
    x = _rnd(B, L, C, seed=41)
    S = _enc(x)
    w1, w2 = rt(_rnd(C, C, 3, seed=42, scale=0.08)), rt(_rnd(C, C, 3, seed=43, scale=0.08))
    b1, b2 = _rnd(C, seed=44, scale=0.1), _rnd(C, seed=45, scale=0.1)
    a_ref = rt(F.leaky_relu(x, 0.01))
    h = rt(F.leaky_relu(F.conv1d(a_ref.permute(0, 2, 1), w1, b1, dilation=dil, padding=dil), 0.01))
    ref = _dec(S) + F.conv1d(h, w2, b2, padding=1).permute(0, 2, 1)
    out = torch.zeros_like(S)
    w1p, w2p = w1.permute(2, 0, 1).contiguous(), w2.permute(2, 0, 1).contiguous()
    d = _desc(_lib, a=S.data_ptr(), x=S.data_ptr(), w1=w1p.data_ptr(), b1=b1.data_ptr(), dilation=dil, w2=w2p.data_ptr(),
              b2=b2.data_ptr(), B=B, L=L, C=C, write_raw=1, precision=_lib.PREC["tf32"], form=_lib.PAIR_FORM[form],
              x_out=out.data_ptr(), stream_enc=1, stream_enc_out=enc_out)
    keep = S.clone()
    _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pair2")
    torch.cuda.synchronize()
    assert torch.equal(S, keep)                                            # the input stream is untouched
    got = _dec(out) if enc_out else out
    assert rel_rms((got - x).cpu(), (ref - x).cpu()) < 1e-4
