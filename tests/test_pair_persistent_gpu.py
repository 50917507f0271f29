"""The fused ResStack pair (vfx_resstack_pair, VFX_PAIR_FUSED: the persistent, warp-specialised kernel) against the blocked
form (the two tensor-core convolutions per row block through a scratch), bit for bit, in all five fused variants:
tf32 C = 64 on the encoded stream (S' or plain x' out), bf16 / fp16 at C = 64 and 128.  The shapes cover a single row,
the edges of the 126-row tile (125, 126, 127, 252, 253), fewer tiles than SMs, a tile count above the SM count and not a
multiple of it with item boundaries inside a CTA's stride, and a dilation longer than the item.  Ragged batches (the
cp.async producer) must give, row for row, what the same pair gives each item alone (the TMA producer), and leave the
rows past each item's length untouched."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = 7.0            # sentinel, exact in every operand format

# (precision, C, stream_enc_out): the pairs the fused kernel runs (pair_supported)
VARIANTS = [("tf32", 64, 1), ("tf32", 64, 0), ("bf16", 64, 0), ("bf16", 128, 0), ("fp16", 64, 0), ("fp16", 128, 0)]
VID = [f"{p}-C{c}" + ("-enc" if p == "tf32" and e else "-plain" if p == "tf32" else "") for p, c, e in VARIANTS]


def _scratch(lib, cache={}):
    n = int(lib.vfx_resstack_pair_scratch_bytes())
    if "buf" not in cache:
        cache["buf"] = torch.empty(n, dtype=torch.uint8, device=DEV)
    return cache["buf"].data_ptr(), n


def _operands(prec, C, B, L, seed):
    from voicefixer_b200.weights import round_tf32
    g = torch.Generator().manual_seed(seed)
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(prec, torch.float32)
    q = (lambda t: round_tf32(t)) if prec == "tf32" else (lambda t: t.to(dt))
    x = torch.randn(B, L, C, generator=g)
    w1 = q(torch.randn(3, C, C, generator=g) / (3 * C) ** 0.5).to(DEV)
    w2 = q(torch.randn(3, C, C, generator=g) * 0.3 / (3 * C) ** 0.5).to(DEV)
    b1 = (torch.randn(C, generator=g) * 0.1).to(DEV)
    b2 = (torch.randn(C, generator=g) * 0.1).to(DEV)
    y = torch.where(x > 0, x, x * 0.01).contiguous()
    if prec == "tf32":     # the encoded stream S = bits(lrelu(x)) + 0x1000 is operand and residual
        s = (y.view(torch.int32) + 0x1000).view(torch.float32).to(DEV)
        return s, s, w1, b1, w2, b2, torch.float32
    return y.to(dt).to(DEV), x.to(DEV), w1, b1, w2, b2, dt


def _run(prec, C, enc_out, a, x, w1, b1, w2, b2, dil, form="fused", write_raw=1, act="lrelu", act_param=0.01,
         lens=None):
    """One pair; returns (raw output, activated output or None).  x is not modified (copied first)."""
    from voicefixer_b200 import _lib
    lib = _lib.load()
    B, L, _ = x.shape
    enc = prec == "tf32"
    xin = x.clone()
    out = torch.full_like(x, SENT) if enc else None
    act_out = None if act is None else torch.full((B, L, C), SENT, device=DEV, dtype=a.dtype)
    d = _lib.PairDesc()
    d.a, d.x = (xin.data_ptr(), xin.data_ptr()) if enc else (a.data_ptr(), xin.data_ptr())
    d.w1, d.b1, d.dilation, d.w2, d.b2 = w1.data_ptr(), b1.data_ptr(), dil, w2.data_ptr(), b2.data_ptr()
    d.B, d.L, d.C, d.write_raw = B, L, C, write_raw
    d.out_act = None if act is None else act_out.data_ptr()
    d.act, d.act_param = (_lib.ACT[act], act_param) if act else (0, 0.0)
    d.precision, d.form = _lib.PREC[prec], _lib.PAIR_FORM[form]
    d.x_out = out.data_ptr() if enc else None
    d.stream_enc, d.stream_enc_out = (1, enc_out) if enc else (0, 0)
    d.lens = None if lens is None else lens.data_ptr()
    d.scratch, d.scratch_bytes = _scratch(lib)
    _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "vfx_resstack_pair")
    torch.cuda.synchronize()
    if enc:
        assert torch.equal(xin, x), "the input stream was written"
    return (out if enc else xin), act_out


SHAPES = [(1, 1, 1), (2, 125, 3), (2, 126, 1), (1, 127, 9), (2, 252, 27), (1, 253, 1), (2, 1000, 243), (1, 1000, 1),
          (3, 40001, 1), (3, 40001, 81), (1, 2000, 2187)]


@pytest.mark.parametrize("B,L,dil", SHAPES)
@pytest.mark.parametrize("prec,C,enc_out", VARIANTS, ids=VID)
def test_fused_equals_blocked(prec, C, enc_out, B, L, dil):
    a, x, w1, b1, w2, b2, _ = _operands(prec, C, B, L, seed=L + dil)
    fr, fa = _run(prec, C, enc_out, a, x, w1, b1, w2, b2, dil)
    br, ba = _run(prec, C, enc_out, a, x, w1, b1, w2, b2, dil, form="blocked")
    assert torch.equal(fr, br), "raw output differs from the blocked form"
    assert torch.equal(fa, ba), "activated output differs from the blocked form"


OUTPUTS = [(1, "lrelu"), (1, None), (0, "lrelu_xsinx"), (1, "lrelu_xsinx")]


@pytest.mark.parametrize("write_raw,act", OUTPUTS, ids=[f"raw{r}-{a}" for r, a in OUTPUTS])
@pytest.mark.parametrize("prec,C,enc_out", VARIANTS, ids=VID)
def test_fused_output_variants(prec, C, enc_out, write_raw, act):
    B, L, dil = 3, 1000, 9
    a, x, w1, b1, w2, b2, _ = _operands(prec, C, B, L, seed=5)
    p = 0.2 if act == "lrelu_xsinx" else 0.01
    fr, fa = _run(prec, C, enc_out, a, x, w1, b1, w2, b2, dil, write_raw=write_raw, act=act, act_param=p)
    br, ba = _run(prec, C, enc_out, a, x, w1, b1, w2, b2, dil, form="blocked", write_raw=write_raw, act=act, act_param=p)
    assert torch.equal(fr, br)
    if act is None:
        assert fa is None
    else:
        assert torch.equal(fa, ba)
    if not write_raw:
        assert torch.equal(fr, torch.full_like(x, SENT) if prec == "tf32" else x), "raw output written"


@pytest.mark.parametrize("dil", [1, 27, 2187])
@pytest.mark.parametrize("prec,C,enc_out", VARIANTS, ids=VID)
def test_fused_ragged_equals_items_alone(prec, C, enc_out, dil):
    L_cap = 1000
    lens_l = [1, 125, 126, 127, L_cap]
    B = len(lens_l)
    a, x, w1, b1, w2, b2, _ = _operands(prec, C, B, L_cap, seed=70 + dil)
    lens = torch.tensor(lens_l, dtype=torch.int32, device=DEV)
    raw, act = _run(prec, C, enc_out, a, x, w1, b1, w2, b2, dil, lens=lens)
    for b, n in enumerate(lens_l):
        ai, xi = a[b:b + 1, :n].contiguous(), x[b:b + 1, :n].contiguous()
        ri, ti = _run(prec, C, enc_out, ai, xi, w1, b1, w2, b2, dil)
        assert torch.equal(raw[b, :n], ri[0]), f"item {b} (L = {n}): raw output differs from the item alone"
        assert torch.equal(act[b, :n], ti[0]), f"item {b} (L = {n}): activated output differs from the item alone"
        rest = raw[b, n:]
        assert torch.equal(rest, torch.full_like(rest, SENT) if prec == "tf32" else x[b, n:]), \
            f"item {b}: raw rows past its length were written"
        assert bool((act[b, n:] == SENT).all()), f"item {b}: activated rows past its length were written"
