"""GPU tests of the TMA-store epilogue of the wgmma conv-GEMM (conv_gemm_tc.cu).

A launch fed by TMA whose residual and outputs tensor maps can express loads the tile's residual through a map during the
K loop and stores the finished tile with TMA stores, while the next tile runs; every other launch keeps the row-loop
epilogue.  Each case runs the same convolution twice: without per-item extents (TMA producer, TMA-store epilogue) and
with extents equal to every item's full length (cp.async producer, row-loop epilogue), asserts through
vfx_conv_tma_launch_count() and vfx_conv_tma_store_launch_count() which epilogue ran, and requires the raw and the operand
buffers to be equal bit for bit, the columns and positions outside the outputs included.  The cases are what the maps'
clipping and the buffer's reuse have to get right: many tiles per CTA (the residual prefetch and the store of
consecutive tiles overlap), the encoded stream overwritten in place, N tails and several N tiles, 127-bin lines, a
strided transposed-convolution phase whose last position is dropped, a column offset inside a concat buffer, and each
combination of outputs in each precision.  An odd column offset is asserted to take the row-loop epilogue."""
import ctypes

import pytest
import torch

from voicefixer_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = 12345.0
SLOPE = 0.01
PRECS = ["tf32", "bf16", "fp16"]
K3 = [(0, -1), (0, 0), (0, 1)]


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


def _launch(prec, a, w, taps, N, phase, out_hw, raw, act, res, col, bias, bias_mod, scale, shift, enc, extents):
    """raw / act / res: [B][OH][OW][ld] buffers or None, from column `col`.  Returns (TMA launches, TMA-store launches)."""
    lib = _lib.load()
    B, H, W, Cin = a.shape
    d = _lib.ConvDesc()
    d.a = a.data_ptr(); d.B, d.H, d.W, d.Cin = B, H, W, Cin
    d.a_sB, d.a_sH, d.a_sW = a.stride(0), a.stride(1), a.stride(2)
    d.w = w.data_ptr(); d.ntaps = len(taps)
    for i, (dh, dw) in enumerate(taps):
        d.dh[i], d.dw[i], d.w_off[i] = dh, dw, i * N * Cin
    d.Hq, d.Wq, d.N = H, W, N
    d.sh, d.rh, d.sw, d.rw = phase
    d.OH, d.OW = out_hw
    if raw is not None:
        d.out_raw = raw.data_ptr(); d.o_sB, d.o_sH, d.o_sW, d.o_col = raw.stride(0), raw.stride(1), raw.stride(2), col
    if act is not None:
        d.out_act = act.data_ptr(); d.oa_sB, d.oa_sH, d.oa_sW, d.oa_col = act.stride(0), act.stride(1), act.stride(2), col
    if res is not None:
        d.residual = res.data_ptr(); d.r_sB, d.r_sH, d.r_sW, d.r_col = res.stride(0), res.stride(1), res.stride(2), col
    d.bias = bias.data_ptr(); d.bias_mod = bias_mod
    d.act_scale, d.act_shift = scale.data_ptr(), shift.data_ptr()
    d.act, d.act_param = _lib.ACT["lrelu"], 0.2
    d.res_enc = int(enc and res is not None)
    d.raw_enc = int(enc and raw is not None)
    d.enc_slope = SLOPE
    keep = []
    if extents:
        axis = 1 if W > 1 else 0
        keep = [torch.full((B,), n, dtype=torch.int32, device=DEV) for n in ((W, out_hw[1]) if axis else (H, out_hw[0]))]
        d.seq_in, d.seq_out, d.seq_axis = keep[0].data_ptr(), keep[1].data_ptr(), axis
    n0, s0 = lib.vfx_conv_tma_launch_count(), lib.vfx_conv_tma_store_launch_count()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.vfx_conv_gemm(_lib.PREC[prec], 1, ctypes.byref(d), st), "vfx_conv_gemm")
    torch.cuda.synchronize()
    return lib.vfx_conv_tma_launch_count() - n0, lib.vfx_conv_tma_store_launch_count() - s0


def _case(prec, B, H, W, Cin, N, taps, outs="both", res=True, enc=False, col=0, ld=None, phase=(1, 0, 1, 0),
          out_hw=None, bias_mod=None, expect_store=True, seed=0):
    """The convolution through both epilogues; outs: "raw", "act" or "both"; enc: the residual is the encoded stream and,
    with a raw output, is overwritten in place."""
    ld = ld or N + col
    out_hw = out_hw or (H, W)
    a = _op(_rnd(B, H, W, Cin, seed=seed), prec)
    w = _op(_rnd(len(taps), N, Cin, seed=seed + 1, scale=(len(taps) * Cin) ** -0.5), prec)
    bias_mod = bias_mod or N
    bias = _rnd(bias_mod, seed=seed + 2, scale=0.1)
    scale, shift = 1.0 + _rnd(N, seed=seed + 3, scale=0.2), _rnd(N, seed=seed + 4, scale=0.1)
    res0 = _rnd(B, *out_hw, ld, seed=seed + 5)
    if enc:
        res0 = _enc(res0)
    results = []
    for extents in (False, True):
        raw = None
        if outs in ("raw", "both"):
            raw = res0.clone() if enc else torch.full((B, *out_hw, ld), SENTINEL, device=DEV)
        act = torch.full((B, *out_hw, ld), SENTINEL, device=DEV).to(a.dtype) if outs in ("act", "both") else None
        r = (raw if enc and raw is not None else res0) if res else None
        tma, tst = _launch(prec, a, w, taps, N, phase, out_hw, raw, act, r, col, bias, bias_mod, scale, shift, enc, extents)
        if extents:
            assert (tma, tst) == (0, 0), "extents: cp.async producer, row-loop epilogue"
        else:
            assert (tma, tst) == (1, int(expect_store)), "no extents"
        results.append((raw, act))
    (raw0, act0), (raw1, act1) = results
    for x0, x1 in ((raw0, raw1), (act0, act1)):
        if x0 is None:
            continue
        assert torch.equal(x0, x1)
        sh, rh, sw, rw = phase
        written = x0[:, rh::sh, rw::sw, col:col + N]
        before = res0[:, rh::sh, rw::sw, col:col + N] if (enc and x0 is raw0) else torch.full_like(written, SENTINEL)
        assert bool((written != before).any()), "the output was written"
    return results[0]


@pytest.mark.parametrize("dil", [1, 2187])
@pytest.mark.parametrize("C", [128, 256])
@pytest.mark.parametrize("prec", PRECS)
def test_resstack_shapes_over_many_tiles(prec, C, dil):
    # 2 x 157 M tiles (x 2 N tiles at C = 256): several tiles per CTA, so the buffer is reused and the residual of each
    # tile is loaded while the stores of the one before are in flight
    _case(prec, 2, 1, 20000, C, C, [(0, -dil), (0, 0), (0, dil)], seed=C + dil)


@pytest.mark.parametrize("outs", ["raw", "act"])
@pytest.mark.parametrize("prec", PRECS)
def test_encoded_stream_in_place_over_many_tiles(prec, outs):
    # raw: the tf32 ResStack's second convolution (S' written over its residual S); act: the last ResStack's, which
    # reads S and writes only the next operand
    _case(prec, 2, 1, 30000, 128, 128, K3, outs=outs, enc=True, seed=10)


@pytest.mark.parametrize("N", [200, 512])
@pytest.mark.parametrize("prec", PRECS)
def test_n_tail_and_several_n_tiles(prec, N):
    _case(prec, 2, 1, 3000, 64, N, K3, seed=N)


@pytest.mark.parametrize("prec", PRECS)
def test_3x3_on_127_bin_lines(prec):
    # every tile is one 127-bin line: the box's 127 rows are stored, the tile's 128th does not exist
    _case(prec, 2, 40, 127, 32, 32, [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)], seed=20)


@pytest.mark.parametrize("prec", PRECS)
def test_strided_phase_with_bias_mod(prec):
    # a transposed-convolution phase: output positions 2 q + 1 of 2 W - 1, so the grid's last position lies outside the
    # output and is clipped; bias_mod < N as in an up-sampler phase group
    B, W, N = 2, 700, 64
    _case(prec, B, 1, W, 64, N, K3, phase=(1, 0, 2, 1), out_hw=(1, 2 * W - 1), bias_mod=N // 2, seed=30)


@pytest.mark.parametrize("prec", PRECS)
def test_aligned_column_offset_in_a_concat_buffer(prec):
    # outputs and residual in columns [C, 2C) of a pitch-2C buffer
    _case(prec, 2, 8, 63, 64, 64, [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)], col=64, ld=128, seed=40)


@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("outs", ["raw", "act", "both"])
@pytest.mark.parametrize("prec", PRECS)
def test_each_combination_of_outputs(prec, outs, res):
    _case(prec, 2, 1, 5000, 128, 96, K3, outs=outs, res=res, seed=50)


@pytest.mark.parametrize("prec", PRECS)
def test_odd_column_takes_the_row_loop_epilogue(prec):
    _case(prec, 2, 1, 2000, 64, 32, K3, col=1, bias_mod=16, expect_store=False, seed=60)
