"""GPU tests of the epilogue of the wgmma conv-GEMM (conv_gemm_tc.cu) with everything the restore step asks of it: bias
(with bias_mod < N, as in a ConvTranspose phase group), an fp32 residual, the raw output, the BN affine (act_scale /
act_shift) and the activated operand, and the tf32 ResStack's second convolution, which reads the encoded stream as its
residual and overwrites it in place.

The epilogue issues every global load of a tile's row pass before the pass's first store.  Each case runs the same
convolution through both operand producers (TMA without per-item extents, cp.async with full-length extents; which one
ran is asserted through vfx_conv_tma_launch_count()), which walk different tiles, and requires their outputs to be equal
bit for bit, untouched buffer parts included; and it bounds the raw output against float64.  The widths cover the three
tile widths (N = 32, 64, 128), several N tiles (256, 512), an N tail (200) and, through a residual and outputs that start
at an odd column, the scalar path; 127-bin lines give tiles of fewer than 128 rows."""
import ctypes

import pytest
import torch

from voicefixer_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = 12345.0
SLOPE = 0.01
RAW_TOL = 1e-6


def _rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _op(t, prec):
    if prec == "bf16":
        return t.bfloat16()
    if prec == "fp16":
        return t.half()
    from voicefixer_b200.weights import round_tf32
    return round_tf32(t.cpu()).to(DEV)


def _enc(x):
    y = torch.where(x > 0, x, x * SLOPE).contiguous()
    return (y.view(torch.int32) + 0x1000).view(torch.float32)


def _dec(s):
    y = (s.contiguous().view(torch.int32) - 0x1000).view(torch.float32)
    return torch.where(y > 0, y, y / SLOPE)


def _launch(prec, a, w, taps, N, raw, act, res, col, bias, bias_mod, scale, shift, enc, extents):
    """raw / act / res: [B][H][W][ld] buffers from column `col` (res may be raw itself); returns 1 if TMA fed the launch."""
    lib = _lib.load()
    B, H, W, Cin = a.shape
    d = _lib.ConvDesc()
    d.a = a.data_ptr(); d.B, d.H, d.W, d.Cin = B, H, W, Cin
    d.a_sB, d.a_sH, d.a_sW = a.stride(0), a.stride(1), a.stride(2)
    d.w = w.data_ptr(); d.ntaps = len(taps)
    for i, (dh, dw) in enumerate(taps):
        d.dh[i], d.dw[i], d.w_off[i] = dh, dw, i * N * Cin
    d.Hq, d.Wq, d.OH, d.OW, d.N = H, W, H, W, N
    d.sh, d.rh, d.sw, d.rw = 1, 0, 1, 0
    d.out_raw = raw.data_ptr(); d.o_sB, d.o_sH, d.o_sW, d.o_col = raw.stride(0), raw.stride(1), raw.stride(2), col
    d.out_act = act.data_ptr(); d.oa_sB, d.oa_sH, d.oa_sW, d.oa_col = act.stride(0), act.stride(1), act.stride(2), col
    d.residual = res.data_ptr(); d.r_sB, d.r_sH, d.r_sW, d.r_col = res.stride(0), res.stride(1), res.stride(2), col
    d.bias = bias.data_ptr(); d.bias_mod = bias_mod
    d.act_scale, d.act_shift = scale.data_ptr(), shift.data_ptr()
    d.act, d.act_param = _lib.ACT["lrelu"], 0.2
    d.res_enc = d.raw_enc = int(enc)
    d.enc_slope = SLOPE
    keep = []
    if extents:
        axis = 1 if W > 1 else 0
        n = W if axis else H
        keep = [torch.full((B,), n, dtype=torch.int32, device=DEV) for _ in range(2)]
        d.seq_in, d.seq_out, d.seq_axis = keep[0].data_ptr(), keep[1].data_ptr(), axis
    n0 = lib.vfx_conv_tma_launch_count()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.vfx_conv_gemm(_lib.PREC[prec], 1, ctypes.byref(d), st), "vfx_conv_gemm")
    torch.cuda.synchronize()
    return lib.vfx_conv_tma_launch_count() - n0


def _case(prec, B, H, W, Cin, N, taps, col=0, bias_mod=None, enc=False, seed=0):
    ld = N + col + (1 if col else 0)
    a = _op(_rnd(B, H, W, Cin, seed=seed), prec)
    w = _op(_rnd(len(taps), N, Cin, seed=seed + 1, scale=(len(taps) * Cin) ** -0.5), prec)
    bias_mod = bias_mod or N
    bias = _rnd(bias_mod, seed=seed + 2, scale=0.1)
    scale, shift = 1.0 + _rnd(N, seed=seed + 3, scale=0.2), _rnd(N, seed=seed + 4, scale=0.1)
    res0 = _rnd(B, H, W, ld, seed=seed + 5)
    if enc:
        res0 = _enc(res0)
    outs = []
    for extents in (False, True):
        raw = res0.clone() if enc else torch.full((B, H, W, ld), SENTINEL, device=DEV)
        res = raw if enc else res0
        act = torch.full((B, H, W, ld), SENTINEL, device=DEV).to(a.dtype)
        tma = _launch(prec, a, w, taps, N, raw, act, res, col, bias, bias_mod, scale, shift, enc, extents)
        assert tma == (0 if extents else 1), "extents" if extents else "no extents"
        outs.append((raw, act))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])
    raw, act = outs[0]
    # columns outside [col, col + N) are untouched
    keep_raw = res0 if enc else torch.full_like(res0, SENTINEL)
    assert torch.equal(raw[..., :col], keep_raw[..., :col]) and torch.equal(raw[..., col + N:], keep_raw[..., col + N:])
    keep_act = torch.full_like(act, SENTINEL)                              # the sentinel as the operand format holds it
    assert torch.equal(act[..., :col], keep_act[..., :col]) and torch.equal(act[..., col + N:], keep_act[..., col + N:])
    # raw output against float64: conv + bias[n % bias_mod] + residual
    a64, w64 = a.double(), w.double()
    ref = torch.zeros(B, H, W, N, dtype=torch.float64, device=DEV)
    for t, (dh, dw) in enumerate(taps):
        sh = torch.zeros_like(a64)
        h0, h1, w0, w1 = max(0, -dh), min(H, H - dh), max(0, -dw), min(W, W - dw)
        sh[:, h0:h1, w0:w1] = a64[:, h0 + dh:h1 + dh, w0 + dw:w1 + dw]
        ref = ref + sh @ w64[t].T
    r = res0[..., col:col + N]
    ref = ref + bias.double()[torch.arange(N, device=DEV) % bias_mod] + (_dec(r) if enc else r).double()
    got = raw[..., col:col + N]
    got = (_dec(got) if enc else got).double()
    assert float((got - ref).norm() / ref.norm()) < (1e-5 if enc else RAW_TOL)
    # the operand: lrelu_0.2(v * scale + shift) in the operand format
    u = ref * scale.double() + shift.double()
    u = torch.where(u > 0, u, 0.2 * u)
    tol = {"tf32": 2e-3, "bf16": 8e-3, "fp16": 2e-3}[prec]
    assert float((act[..., col:col + N].double() - u).norm() / u.norm()) < tol


PRECS = ["tf32", "bf16", "fp16"]
K3 = [(0, -1), (0, 0), (0, 1)]


@pytest.mark.parametrize("N", [32, 64, 128, 200, 256, 512])
@pytest.mark.parametrize("prec", PRECS)
def test_full_epilogue_every_tile_width(prec, N):
    _case(prec, 2, 1, 300, 64, N, K3, seed=N)


@pytest.mark.parametrize("N", [32, 64, 128])
@pytest.mark.parametrize("prec", PRECS)
def test_encoded_stream_in_place(prec, N):
    # residual == out_raw, read as the encoded stream and overwritten with the encoded result
    _case(prec, 3, 1, 333, 64, N, K3, enc=True, seed=100 + N)


@pytest.mark.parametrize("N", [32, 96])
@pytest.mark.parametrize("prec", PRECS)
def test_scalar_path_at_an_odd_column_with_bias_mod(prec, N):
    # outputs and residual from column 1: no 16-byte row accesses; bias_mod < N as in a ConvTranspose phase group
    _case(prec, 2, 1, 250, 64, N, K3, col=1, bias_mod=N // 2, seed=200 + N)


@pytest.mark.parametrize("prec", PRECS)
def test_3x3_on_127_bin_lines(prec):
    # every TMA tile holds one 127-bin line: 127 of 128 rows exist
    _case(prec, 2, 9, 127, 32, 32, [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)], seed=300)
