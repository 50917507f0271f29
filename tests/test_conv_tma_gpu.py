"""GPU tests of the two operand producers of the wgmma conv-GEMM (conv_gemm_tc.cu): TMA and cp.async.

The library chooses the producer from the descriptor: a launch without per-item extents whose operands a tensor map can
express is fed by TMA and walks rectangular tiles of the output grid; a launch with extents (seq_in / seq_out) is fed by
cp.async and walks 128 consecutive rows of the flattened grid.  Extents equal to every item's full length change nothing
in what is computed, so every case launches the same convolution twice, with NULL extents (expected on TMA) and with full
extents (expected on cp.async), asserts through vfx_conv_tma_launch_count() that each took the producer it should, and
requires the raw and the operand outputs to be equal bit for bit, untouched parts of the buffers included.  The cases are
what the out-of-bounds fill of the tensor maps has to supply in place of the zero-fill copies: padding at any dilation,
the Cin tail of a slice, rows beyond the problem, tiles that end at an item's or a line's end, weight rows beyond N.
One case is bounded against float64 (RAW_TOL of tests/test_kernels_fp64_gpu.py), so that the pair cannot be wrong together."""
import ctypes

import pytest
import torch

from voicefixer_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RAW_TOL = 1e-6
SENTINEL = 12345.0
PRECS = ["tf32", "bf16", "fp16"]


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


def _launch(prec, a, w, taps, w_off, N, grid, out_hw, raw, act, col, phase=(1, 0, 1, 0), bias=None, bias_mod=None,
            res=None, extents=False):
    """a: [B][H][W][Cin] (any strides, channels contiguous); taps: [(dh, dw)]; grid = (Hq, Wq); out_hw = (OH, OW);
    raw / act / res: [B][OH][OW][ld] buffers, written / read from column `col`; phase = (sh, rh, sw, rw).
    extents: pass every item's full length on the W axis (H when W == 1) as seq_in / seq_out.
    Returns how many of the launches were fed by TMA (0 or 1)."""
    lib = _lib.load()
    B, H, W, Cin = a.shape
    d = _lib.ConvDesc()
    d.a = a.data_ptr(); d.B, d.H, d.W, d.Cin = B, H, W, Cin
    d.a_sB, d.a_sH, d.a_sW = a.stride(0), a.stride(1), a.stride(2)
    d.w = w.data_ptr(); d.ntaps = len(taps)
    for i, (dh, dw) in enumerate(taps):
        d.dh[i], d.dw[i], d.w_off[i] = dh, dw, w_off[i]
    d.Hq, d.Wq = grid
    d.N = N
    d.sh, d.rh, d.sw, d.rw = phase
    d.OH, d.OW = out_hw
    d.out_raw = raw.data_ptr(); d.o_sB, d.o_sH, d.o_sW, d.o_col = raw.stride(0), raw.stride(1), raw.stride(2), col
    d.out_act = act.data_ptr(); d.oa_sB, d.oa_sH, d.oa_sW, d.oa_col = act.stride(0), act.stride(1), act.stride(2), col
    d.act, d.act_param = _lib.ACT["lrelu"], 0.01
    if res is not None:
        d.residual = res.data_ptr(); d.r_sB, d.r_sH, d.r_sW, d.r_col = res.stride(0), res.stride(1), res.stride(2), col
    if bias is not None:
        d.bias = bias.data_ptr(); d.bias_mod = bias_mod or bias.numel()
    keep = []
    if extents:
        axis = 1 if W > 1 else 0
        keep = [torch.full((B,), n, dtype=torch.int32, device=DEV) for n in ((W, out_hw[1]) if axis else (H, out_hw[0]))]
        d.seq_in, d.seq_out, d.seq_axis = keep[0].data_ptr(), keep[1].data_ptr(), axis
    n0 = lib.vfx_conv_tma_launch_count()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.vfx_conv_gemm(_lib.PREC[prec], 1, ctypes.byref(d), st), "vfx_conv_gemm")
    torch.cuda.synchronize()
    return lib.vfx_conv_tma_launch_count() - n0


def _both(prec, a, w, taps, N, grid=None, out_hw=None, w_off=None, ld=None, col=0, phase=(1, 0, 1, 0), bias_mod=None,
          seed=0):
    """The convolution through both producers; returns the (equal) raw output [B][OH][OW][ld], the bias and the residual."""
    B, H, W, Cin = a.shape
    grid = grid or (H, W)
    out_hw = out_hw or grid
    w_off = w_off or [i * N * Cin for i in range(len(taps))]
    ld = ld or N
    bias = _rnd(bias_mod or N, seed=seed + 50)
    res = _rnd(B, *out_hw, ld, seed=seed + 51)
    outs = []
    for extents in (False, True):
        raw = torch.full((B, *out_hw, ld), SENTINEL, device=DEV)
        act = torch.full((B, *out_hw, ld), SENTINEL, device=DEV).to(a.dtype)
        tma = _launch(prec, a, w, taps, w_off, N, grid, out_hw, raw, act, col, phase, bias, bias_mod, res, extents)
        assert tma == (0 if extents else 1), "extents" if extents else "no extents"
        outs.append((raw, act))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])
    assert bool((outs[0][0][..., col:col + N] != SENTINEL).all())
    return outs[0][0], bias, res


def _conv1d(prec, B, L, Cin, N, offs, seed=0):
    a = _op(_rnd(B, 1, L, Cin, seed=seed), prec)
    w = _op(_rnd(len(offs), N, Cin, seed=seed + 1, scale=(len(offs) * Cin) ** -0.5), prec)
    return (a, w) + _both(prec, a, w, [(0, o) for o in offs], N, seed=seed)


@pytest.mark.parametrize("L", [1000, 5000])
@pytest.mark.parametrize("dil", [1, 27, 2187])
@pytest.mark.parametrize("prec", PRECS)
def test_k3_dilations_on_short_and_long_sequences(prec, dil, L):
    # dilation 2187 on 1000 rows: the outer taps lie wholly outside every item
    _conv1d(prec, 2, L, 64, 64, [-dil, 0, dil])


@pytest.mark.parametrize("prec", PRECS)
def test_k7_valid_on_a_padded_buffer(prec):
    B, L, Cin, N = 2, 700, 64, 128
    a = _op(_rnd(B, 1, L + 6, Cin, seed=3), prec)
    w = _op(_rnd(7, N, Cin, seed=4, scale=0.05), prec)
    _both(prec, a, w, [(0, k) for k in range(7)], N, grid=(1, L), seed=3)


@pytest.mark.parametrize("prec", PRECS)
def test_items_whose_length_is_no_multiple_of_the_tile(prec):
    # cp.async: tiles straddle items; TMA: every item ends in a partial tile
    _conv1d(prec, 5, 333, 64, 64, [-3, 0, 3], seed=5)


@pytest.mark.parametrize("Cin", [16, 48])
@pytest.mark.parametrize("prec", PRECS)
def test_channel_tail_inside_a_slice(prec, Cin):
    _conv1d(prec, 2, 500, Cin, 64, [-1, 0, 1], seed=7)


@pytest.mark.parametrize("N", [24, 96, 200])
@pytest.mark.parametrize("prec", PRECS)
def test_n_tails(prec, N):
    _conv1d(prec, 2, 500, 64, N, [-1, 0, 1], seed=9)


@pytest.mark.parametrize("grp", [0, 1])
@pytest.mark.parametrize("prec", PRECS)
def test_transposed_conv_phase_group(prec, grp):
    # ConvTranspose1d(k = 2u, stride u) as the engine runs it: the group's two taps start mid-array in w and its phases go
    # to columns [r0 Co, (r0 + nph) Co) of the output viewed as [B][Lin][u Co]
    u, Ci, Co, B, Lin = 7, 64, 32, 2, 300
    pad = u // 2 + u % 2
    nA = u - pad
    mat = Co * Ci
    a = _op(_rnd(B, 1, Lin, Ci, seed=11), prec)
    w = _op(_rnd(2 * u, Co, Ci, seed=12, scale=0.1), prec)
    if grp == 0:
        taps, w_off, nph, r0 = [(0, 0), (0, -1)], [pad * mat, (pad + u) * mat], nA, 0
    else:
        taps, w_off, nph, r0 = [(0, 1), (0, 0)], [0, u * mat], u - nA, nA
    _both(prec, a, w, taps, nph * Co, w_off=w_off, ld=u * Co, col=r0 * Co, bias_mod=Co, seed=11)


@pytest.mark.parametrize("prec", PRECS)
def test_3x3_on_127_bins_of_a_concat_buffer(prec):
    # the operand is the first C channels of a [B][H][127][2C] buffer; tiles end at every line's 127th bin
    B, H, W, C, N = 2, 20, 127, 32, 32
    buf = _op(_rnd(B, H, W, 2 * C, seed=13), prec)
    a = buf[..., :C]
    w = _op(_rnd(9, N, C, seed=14, scale=0.06), prec)
    _both(prec, a, w, [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)], N, seed=13)


@pytest.mark.parametrize("prec", PRECS)
def test_3x3_on_lines_shorter_than_a_tile(prec):
    # 15-wide lines: a TMA tile holds 8 whole lines of one item, 6 lines at the item's end
    B, H, W, C, N = 3, 22, 15, 64, 64
    a = _op(_rnd(B, H, W, C, seed=15), prec)
    w = _op(_rnd(9, N, C, seed=16, scale=0.04), prec)
    _both(prec, a, w, [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)], N, seed=15)


@pytest.mark.parametrize("prec", PRECS)
def test_1x1_on_items_smaller_than_a_tile(prec):
    # 5 x 7 positions per item: a TMA tile holds 3 whole items
    B, H, W, C, N = 7, 5, 7, 128, 96
    a = _op(_rnd(B, H, W, C, seed=17), prec)
    w = _op(_rnd(1, N, C, seed=18, scale=0.09), prec)
    _both(prec, a, w, [(0, 0)], N, seed=17)


@pytest.mark.parametrize("prec", PRECS)
def test_against_float64(prec):
    B, L, Cin, N, offs = 3, 777, 80, 96, [-27, 0, 27]
    a, w, raw, bias, res = _conv1d(prec, B, L, Cin, N, offs, seed=19)
    a64 = a[:, 0].double()
    ref = bias.double() + res[:, 0].double()
    for t, o in enumerate(offs):
        sh = torch.zeros_like(a64)
        lo, hi = max(0, -o), min(L, L - o)
        sh[:, lo:hi] = a64[:, lo + o:hi + o]
        ref = ref + sh @ w[t].double().T
    assert float((raw[:, 0].double() - ref).norm() / ref.norm()) < RAW_TOL
