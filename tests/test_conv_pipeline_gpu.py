"""GPU tests of the persistent, pipelined wgmma conv-GEMM (conv_gemm_tc.cu) where the tile schedule matters.

The kernel assigns output tiles to CTAs by a static stride, runs a K slice ring across tile boundaries, skips the tiles
of a ragged batch that store nothing and writes the epilogue with vector or scalar accesses.  None of these may change
a bit: every case compares two launches that put the same rows on different CTAs, at different positions of a CTA's
tile sequence or through different epilogue paths, and bounds one of them against float64 (RAW_TOL of the other conv
tests)."""
import ctypes

import pytest
import torch

from voicefixer_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RAW_TOL = 1e-6
SENTINEL = 12345.0


def _rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _op(t, prec):
    """Operand in the storage format of `prec` and its exact value."""
    if prec == "bf16":
        return t.bfloat16()
    if prec == "fp16":
        return t.half()
    from voicefixer_b200.weights import round_tf32
    return round_tf32(t.cpu()).to(DEV)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _conv(a, w, offs, N, prec, bias=None, bias_mod=None, res=None, raw=None, act=None, lens=None):
    """1-D convolution on the [B][1][L][Cin] layout: out[b, l, n] = sum_t sum_c w[t, n, c] a[b, l + offs[t], c] + bias +
    residual.  raw / act / res: (tensor [B][L][ld], first column); lens: per-item extents (seq_in = seq_out)."""
    B, L, Cin = a.shape
    d = _lib.ConvDesc()
    d.a = a.data_ptr(); d.B, d.H, d.W, d.Cin = B, 1, L, Cin
    d.a_sW, d.a_sH, d.a_sB = Cin, L * Cin, L * Cin
    d.w = w.data_ptr(); d.ntaps = len(offs)
    for i, o in enumerate(offs):
        d.dh[i], d.dw[i], d.w_off[i] = 0, o, i * N * Cin
    d.Hq, d.Wq, d.N = 1, L, N
    d.sh, d.rh, d.sw, d.rw = 1, 0, 1, 0
    d.OH, d.OW = 1, L
    if raw is not None:
        t, col = raw
        d.out_raw = t.data_ptr(); d.o_sW, d.o_sH, d.o_sB, d.o_col = t.stride(1), t.stride(0), t.stride(0), col
    if act is not None:
        t, col = act
        d.out_act = t.data_ptr(); d.oa_sW, d.oa_sH, d.oa_sB, d.oa_col = t.stride(1), t.stride(0), t.stride(0), col
        d.act, d.act_param = _lib.ACT["lrelu"], 0.01
    if res is not None:
        t, col = res
        d.residual = t.data_ptr(); d.r_sW, d.r_sH, d.r_sB, d.r_col = t.stride(1), t.stride(0), t.stride(0), col
    if bias is not None:
        d.bias = bias.data_ptr(); d.bias_mod = bias_mod or bias.numel()
    if lens is not None:
        d.seq_in = d.seq_out = lens.data_ptr(); d.seq_axis = 1
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.load().vfx_conv_gemm(_lib.PREC[prec], 1, ctypes.byref(d), st), "vfx_conv_gemm")
    torch.cuda.synchronize()


def _ref(a, w, offs, N, bias=None, bias_mod=None, res=None, lens=None):
    """float64 reference of _conv's raw output (zero input outside each item's extent)."""
    B, L, _ = a.shape
    a64 = a.double()
    if lens is not None:
        a64 = a64 * (torch.arange(L, device=DEV)[None, :, None] < lens[:, None, None]).double()
    out = torch.zeros(B, L, N, dtype=torch.float64, device=DEV)
    for t, o in enumerate(offs):
        sh = torch.zeros_like(a64)
        lo, hi = max(0, -o), min(L, L - o)
        if hi > lo:
            sh[:, lo:hi] = a64[:, lo + o:hi + o]
        out += sh @ w[t].double().T
    if bias is not None:
        out += bias.double()[torch.arange(N, device=DEV) % (bias_mod or bias.numel())]
    if res is not None:
        out += res.double()
    return out


def _rel(x, ref):
    return float((x.double() - ref).norm() / ref.norm())


def _case(B, L, Cin, N, offs, prec, seed=0, bias_mod=None):
    a = _op(_rnd(B, L, Cin, seed=seed), prec)
    w = _op(_rnd(len(offs), N, Cin, seed=seed + 1, scale=Cin ** -0.5), prec)
    bias = _rnd(bias_mod or N, seed=seed + 2)
    res = _rnd(B, L, N, seed=seed + 3)
    return a, w, bias, res


def _batched_vs_alone(B, L, Cin, N, offs, prec, bias_mod=None):
    a, w, bias, res = _case(B, L, Cin, N, offs, prec, bias_mod=bias_mod)
    raw = torch.zeros(B, L, N, device=DEV)
    _conv(a, w, offs, N, prec, bias=bias, bias_mod=bias_mod, res=(res, 0), raw=(raw, 0))
    for b in range(B):
        one = torch.zeros(1, L, N, device=DEV)
        _conv(a[b:b + 1].contiguous(), w, offs, N, prec, bias=bias, bias_mod=bias_mod, res=(res[b:b + 1].contiguous(), 0),
              raw=(one, 0))
        assert torch.equal(one[0], raw[b]), f"item {b}"
    assert _rel(raw, _ref(a, w, offs, N, bias, bias_mod, res)) < RAW_TOL


@pytest.mark.parametrize("per_sm", [0.5, 1, 5])
@pytest.mark.parametrize("prec", ["tf32", "bf16"])
def test_tile_counts_around_the_sm_count(per_sm, prec):
    # N = 128: one N tile; B = 2 items of L rows make 2L / 128 tiles, each item alone half of them
    tiles = max(2, int(per_sm * _sms()) // 2 * 2)
    _batched_vs_alone(2, tiles * 64, 64, 128, [-3, 0, 3], prec)


@pytest.mark.parametrize("taps,Cin", [(1, 32), (2, 32), (1, 128), (9, 384)])
@pytest.mark.parametrize("prec", ["tf32", "bf16", "fp16"])
def test_k_loops_shorter_equal_and_longer_than_the_ring(taps, Cin, prec):
    # K slices = taps * Cin / (32 tf32 or 64 16-bit channels): 1, 2, 4 (the BN = 128 ring) and 9 x 12 in tf32
    if prec != "tf32":
        Cin *= 2
    offs = [2 * (t - taps // 2) for t in range(taps)]
    _batched_vs_alone(3, 1500, Cin, 128, offs, prec)


@pytest.mark.parametrize("N,bias_mod", [(96, None), (200, None), (1024, 128)])
@pytest.mark.parametrize("prec", ["tf32", "bf16"])
def test_n_tails_and_wide_n(N, bias_mod, prec):
    _batched_vs_alone(2, 700, 64, N, [-1, 0, 1], prec, bias_mod=bias_mod)


@pytest.mark.parametrize("prec", ["tf32", "bf16", "fp16"])
def test_ragged_batch_with_interleaved_skipped_tiles(prec):
    # alternating lengths: the short items' tail tiles store nothing and are skipped between live tiles of one CTA
    B, L, C = 8, 40 * 128, 64
    lens_l = [L if b % 2 == 0 else 300 + 37 * b for b in range(B)]
    lens = torch.tensor(lens_l, dtype=torch.int32, device=DEV)
    a, w, bias, res = _case(B, L, C, C, [-2, 0, 2], prec, seed=7)
    raw = torch.full((B, L, C), SENTINEL, device=DEV)
    act = torch.full((B, L, C), SENTINEL, device=DEV).to(a.dtype)
    act_sentinel = act[0, 0, 0].clone()
    _conv(a, w, [-2, 0, 2], C, prec, bias=bias, res=(res, 0), raw=(raw, 0), act=(act, 0), lens=lens)
    for b, n in enumerate(lens_l):
        one = torch.zeros(1, n, C, device=DEV)
        one_act = torch.zeros(1, n, C, device=DEV).to(a.dtype)
        _conv(a[b:b + 1, :n].contiguous(), w, [-2, 0, 2], C, prec, bias=bias, res=(res[b:b + 1, :n].contiguous(), 0),
              raw=(one, 0), act=(one_act, 0))
        assert torch.equal(raw[b, :n], one[0]), f"item {b}"
        assert torch.equal(act[b, :n], one_act[0]), f"item {b}"
        assert bool((raw[b, n:] == SENTINEL).all()) and bool((act[b, n:] == act_sentinel).all()), f"item {b}"
    ref = _ref(a, w, [-2, 0, 2], C, bias, None, res, lens)
    keep = torch.arange(L, device=DEV)[None, :, None] < lens[:, None, None]
    assert _rel(torch.where(keep, raw, 0.0), torch.where(keep, ref, 0.0)) < RAW_TOL


@pytest.mark.parametrize("N", [64, 128, 200])
@pytest.mark.parametrize("prec", ["tf32", "bf16", "fp16"])
def test_vector_and_scalar_epilogues_agree(N, prec):
    # the same convolution into dense buffers (16-byte epilogue accesses) and into buffers whose rows start at an odd
    # column (element accesses); the residual is read from the same kind of buffer
    B, L, Cin = 2, 900, 64
    a, w, bias, res = _case(B, L, Cin, N, [-1, 0, 1], prec, seed=11)
    raw_v, act_v = torch.zeros(B, L, N, device=DEV), torch.zeros(B, L, N, device=DEV).to(a.dtype)
    _conv(a, w, [-1, 0, 1], N, prec, bias=bias, res=(res, 0), raw=(raw_v, 0), act=(act_v, 0))
    ld = N + 3
    res_s = torch.zeros(B, L, ld, device=DEV)
    res_s[:, :, 1:N + 1] = res
    raw_s, act_s = torch.zeros(B, L, ld, device=DEV), torch.zeros(B, L, ld, device=DEV).to(a.dtype)
    _conv(a, w, [-1, 0, 1], N, prec, bias=bias, res=(res_s, 1), raw=(raw_s, 1), act=(act_s, 1))
    assert torch.equal(raw_v, raw_s[:, :, 1:N + 1])
    assert torch.equal(act_v, act_s[:, :, 1:N + 1])
    assert bool((raw_s[:, :, 0] == 0).all()) and bool((raw_s[:, :, N + 1:] == 0).all())
    assert _rel(raw_v, _ref(a, w, [-1, 0, 1], N, bias, None, res)) < RAW_TOL
