"""Ragged batches: items of different lengths in one launch sequence (vfx_restore_ragged, Engine.restore(lens=...),
VoiceFixer.restore_batch(list)).

Every row of a ragged batch must be bit-identical to restoring that item alone, whatever the other items, the batch's
capacity or the contents of the padding and of the workspace.  The kernel tests check the per-item extents of each
kernel that reads along the time axis against the same kernel on the item alone and against float64."""
import ctypes
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
SENT = -1920.0
SR = 44100
PRECS = ["fp32", "tf32", "bf16", "fp16"]

# 1025 (the minimum, T = 3), T = 64 with L % 441 = 440, T = 65 with L % 441 = 0, an even T (114) and the capacity (3 s)
EDGE_LENS = [1025, 64 * 441 - 1, 64 * 441, 50000, 3 * SR]
EDGE_CAP = 3 * SR

_ENGINES = {}
_ALONE = {}


@pytest.fixture(autouse=True)
def _fp32_torch():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _engine(states, prec):
    if prec not in _ENGINES:
        from voicefixer_b200.engine import Engine
        _ENGINES[prec] = Engine(states[0], states[1], precision=prec)
    return _ENGINES[prec]


def _items(lens, seed):
    g = np.random.default_rng(seed)
    return [(0.3 * g.standard_normal(n)).astype(np.float32) for n in lens]


def _batch(items, L_cap, pad=0.0):
    x = torch.full((len(items), L_cap), pad, device=DEV)
    for i, a in enumerate(items):
        x[i, :a.shape[0]] = torch.from_numpy(a).to(DEV)
    lens = torch.tensor([a.shape[0] for a in items], dtype=torch.int32, device=DEV)
    return x, lens


def _alone(eng, a, ws=None):
    return eng.restore(torch.from_numpy(a)[None].to(DEV), ws=ws)[0]


def _alone_cached(eng, prec, items, seed):
    key = (prec, seed, tuple(a.shape[0] for a in items))
    if key not in _ALONE:
        _ALONE[key] = [_alone(eng, a).clone() for a in items]
    return _ALONE[key]


def _check_rows(y, items, alone):
    for i, a in enumerate(items):
        n = a.shape[0]
        assert torch.equal(y[i, :n], alone[i]), f"item {i} (L = {n}) differs from the same item restored alone"
        assert bool((y[i, n:] == 0).all()), f"item {i} (L = {n}): samples past its length are not zero"


# ============================================================================ 1. bit identity, every precision
@pytest.mark.parametrize("prec", PRECS)
def test_ragged_rows_equal_items_alone(states, prec):
    eng = _engine(states, prec)
    items = _items(EDGE_LENS, 1)
    x, lens = _batch(items, EDGE_CAP)
    y = eng.restore(x, lens=lens)
    torch.cuda.synchronize()
    _check_rows(y, items, _alone_cached(eng, prec, items, 1))


def test_ragged_restore_inmem_shape(states):
    """A full 30 s segment and a 2 s tail (what restore_inmem makes of a 32 s recording) in one ragged batch."""
    eng = _engine(states, "tf32")
    items = _items([30 * SR, 2 * SR + 123], 2)
    x, lens = _batch(items, 30 * SR)
    y = eng.restore(x, lens=lens)
    torch.cuda.synchronize()
    _check_rows(y, items, [_alone(eng, a) for a in items])


# ============================================================================ 2. poisoned padding and workspace
@pytest.mark.parametrize("prec", PRECS)
def test_ragged_ignores_padding_and_stale_workspace(states, prec):
    """NaN past every item's length in the input and 0xFF bytes (NaN as fp32) in the whole workspace: a kernel that
    reads beyond an item's extent, or a buffer location it never wrote, turns its row non-finite or different.  The
    references are computed on a poisoned workspace as well, which checks the equal-length path the same way."""
    eng = _engine(states, prec)
    items = _items(EDGE_LENS, 1)
    x, lens = _batch(items, EDGE_CAP, pad=float("nan"))
    B = len(items)
    ws = torch.full((eng.workspace_bytes(B, EDGE_CAP),), 0xFF, dtype=torch.uint8, device=DEV)
    y = eng.restore(x, lens=lens, ws=ws)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all())
    alone = _alone_cached(eng, prec, items, 1)
    _check_rows(y, items, alone)
    for i, a in enumerate(items):
        ws1 = torch.full((eng.workspace_bytes(1, a.shape[0]),), 0xFF, dtype=torch.uint8, device=DEV)
        assert torch.equal(_alone(eng, a, ws=ws1), alone[i]), f"equal-length path: item {i} depends on stale workspace"


# ============================================================================ 3. capacity invariance and graphs
def test_ragged_capacity_and_graph_replay(states):
    eng = _engine(states, "tf32")
    items = _items([1025, 44100, 70001, 2 * SR], 3)
    x1, lens = _batch(items, 2 * SR)
    y1 = eng.restore(x1, lens=lens).clone()
    x2, _ = _batch(items, 7 * SR)
    y2 = eng.restore(x2, lens=lens).clone()
    torch.cuda.synchronize()
    for i, a in enumerate(items):
        assert torch.equal(y1[i, :a.shape[0]], y2[i, :a.shape[0]]), f"item {i} depends on the batch capacity"
    # one graph of shape (4, 7 s), replayed with two sets of lengths
    out = torch.empty_like(x2)
    g = eng.make_graph(x2, out, lens=lens)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, y2)
    items2 = _items([7 * SR, 3000, 100000, 5 * SR + 7], 4)
    xb, lens_b = _batch(items2, 7 * SR)
    x2.copy_(xb)
    lens.copy_(lens_b)
    g.replay()
    torch.cuda.synchronize()
    direct = eng.restore(xb, lens=lens_b)
    torch.cuda.synchronize()
    assert torch.equal(out, direct)
    _check_rows(out, items2, [_alone(eng, a) for a in items2])


# ============================================================================ 4. kernels
def _desc(a, w, taps, out, seq_in, seq_out, seq_axis, prec):
    """vfx_conv_desc for a channels-last a (B, H, W, Cin), weights [tap][N][Cin], fp32 raw output out (B, H, W, N)."""
    from voicefixer_b200 import _lib
    B, H, W, Cin = a.shape
    N = w.shape[1]
    d = _lib.ConvDesc()
    d.a = a.data_ptr(); d.B, d.H, d.W, d.Cin = B, H, W, Cin
    d.a_sB, d.a_sH, d.a_sW = a.stride(0), a.stride(1), a.stride(2)
    d.w = w.data_ptr(); d.ntaps = len(taps)
    for i, (dh, dw) in enumerate(taps):
        d.dh[i], d.dw[i], d.w_off[i] = dh, dw, i * N * Cin
    d.Hq, d.Wq, d.N = H, W, N
    d.sh, d.sw, d.OH, d.OW = 1, 1, H, W
    d.out_raw = out.data_ptr(); d.o_sW, d.o_sH, d.o_sB = N, W * N, H * W * N
    d.seq_in = None if seq_in is None else seq_in.data_ptr()
    d.seq_out = None if seq_out is None else seq_out.data_ptr()
    d.seq_axis = seq_axis
    return d


def _run_conv(a, w, taps, prec, impl, ext=None, axis=0):
    from voicefixer_b200 import _lib
    B, H, W, _ = a.shape
    out = torch.full((B, H, W, w.shape[1]), SENT, device=DEV)
    d = _desc(a, w, taps, out, ext, ext, axis, prec)
    _lib.check(_lib.load().vfx_conv_gemm(_lib.PREC[prec], impl, ctypes.byref(d), None), "vfx_conv_gemm")
    torch.cuda.synchronize()
    return out


CONV_CASES = [
    # axis 0: the UNet's 3x3 over [B][T][F][C]; one item of a single row
    (0, (4, 20, 9, 32), [20, 7, 1, 13], [(dh, dw) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]),
    # axis 1: a dilated k3 over [B][1][L][C]; dilation 9 exceeds two items' extents; whole tiles lie past item 1's end
    (1, (4, 1, 300, 64), [300, 5, 8, 130], [(0, -9), (0, 0), (0, 9)]),
]


@pytest.mark.parametrize("impl,prec", [(1, "bf16"), (1, "tf32"), (1, "fp16"), (0, "fp32"), (0, "bf16")])
@pytest.mark.parametrize("case", range(len(CONV_CASES)))
def test_conv_gemm_seq_extents(case, impl, prec):
    from voicefixer_b200.weights import round_tf32
    axis, shape, ext_l, taps = CONV_CASES[case]
    B, H, W, C = shape
    g = torch.Generator().manual_seed(10 + case)
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(prec, torch.float32)
    q = (lambda t: round_tf32(t)) if prec == "tf32" else (lambda t: t.to(dt))
    a = q(torch.randn(B, H, W, C, generator=g).to(DEV))
    w = q((torch.randn(len(taps), 48, C, generator=g) / (len(taps) * C) ** 0.5).to(DEV))
    ext = torch.tensor(ext_l, dtype=torch.int32, device=DEV)
    out = _run_conv(a, w, taps, prec, impl, ext, axis)
    tol = 1e-6 if impl == 1 else 2.5e-6
    for b, e in enumerate(ext_l):
        item = a[b:b + 1, :e] if axis == 0 else a[b:b + 1, :, :e]
        alone = _run_conv(item.contiguous(), w, taps, prec, impl)
        got = out[b:b + 1, :e] if axis == 0 else out[b:b + 1, :, :e]
        assert torch.equal(got, alone), f"item {b}: rows inside the extent differ from the item alone"
        rest = out[b, e:] if axis == 0 else out[b, :, e:]
        assert bool((rest == SENT).all()), f"item {b}: an output past its extent was stored"
        # float64 reference of the item alone: taps as a convolution with zero padding at the item's own edges
        x64 = item.to(F64).permute(0, 3, 1, 2)
        w64 = w.to(F64)
        if axis == 0:
            ref = F.conv2d(x64, w64.reshape(3, 3, 48, C).permute(2, 3, 0, 1), padding=1)
        else:
            ref = F.conv1d(x64[:, :, 0], w64.permute(1, 2, 0), padding=9, dilation=9)[:, :, None]
        ref = ref.permute(0, 2, 3, 1)
        err = float((got.to(F64) - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
        assert err < tol, f"item {b}: relative RMS {err:.2e} against float64"


def _pair(prec, a, x, w1, b1, w2, b2, dil, lens=None, form="fused", x_out=None, enc=False):
    from voicefixer_b200 import _lib
    B, L, C = x.shape
    d = _lib.PairDesc()
    d.a, d.x = a.data_ptr(), x.data_ptr()
    d.w1, d.b1, d.dilation, d.w2, d.b2 = w1.data_ptr(), b1.data_ptr(), dil, w2.data_ptr(), b2.data_ptr()
    d.B, d.L, d.C, d.write_raw = B, L, C, 1
    d.precision, d.form = _lib.PREC[prec], _lib.PAIR_FORM[form]
    d.x_out = None if x_out is None else x_out.data_ptr()
    d.stream_enc, d.stream_enc_out = (1, 1) if enc else (0, 0)
    d.lens = None if lens is None else lens.data_ptr()
    rc = _lib.load().vfx_resstack_pair(ctypes.byref(d), None)
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("prec,C", [("bf16", 64), ("bf16", 128), ("fp16", 64), ("fp16", 128), ("tf32", 64)])
@pytest.mark.parametrize("dil", [1, 27, 243])
def test_fused_pair_lens_equal_items_alone(prec, C, dil):
    from voicefixer_b200.weights import round_tf32
    g = torch.Generator().manual_seed(20 + C + dil)
    lens_l = [400, 1, 127, 250, 5]
    B, L = len(lens_l), 400
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(prec, torch.float32)
    q = (lambda t: round_tf32(t)) if prec == "tf32" else (lambda t: t.to(dt))
    x = torch.randn(B, L, C, generator=g).to(DEV)
    w1 = q((torch.randn(3, C, C, generator=g) / (3 * C) ** 0.5).to(DEV))
    w2 = q((torch.randn(3, C, C, generator=g) * 0.3 / (3 * C) ** 0.5).to(DEV))
    b1 = (torch.randn(C, generator=g) * 0.1).to(DEV)
    b2 = (torch.randn(C, generator=g) * 0.1).to(DEV)
    lens = torch.tensor(lens_l, dtype=torch.int32, device=DEV)
    enc = prec == "tf32"
    if enc:      # the encoded stream S = bits(lrelu(x)) + 0x1000 is both operand and residual
        s = torch.where(x > 0, x, x * 0.01).contiguous().view(torch.int32).add(0x1000).view(torch.float32)
        a, xin = s, s
    else:
        a, xin = torch.where(x > 0, x, x * 0.01).to(dt), x.clone()
    before = xin.clone()
    out = torch.full_like(xin, SENT) if enc else xin
    assert _pair(prec, a, xin, w1, b1, w2, b2, dil, lens=lens, x_out=out if enc else None, enc=enc) == 0
    for b, n in enumerate(lens_l):
        ai = a[b:b + 1, :n].contiguous()
        xi = before[b:b + 1, :n].contiguous()
        oi = torch.full_like(xi, SENT) if enc else xi
        assert _pair(prec, ai if not enc else xi, xi, w1, b1, w2, b2, dil, x_out=oi if enc else None, enc=enc) == 0
        assert torch.equal(out[b, :n], oi[0]), f"item {b} (L = {n}) differs from the item alone"
        rest = out[b, n:]
        assert torch.equal(rest, torch.full_like(rest, SENT) if enc else before[b, n:]), \
            f"item {b}: rows past its length were written"
    # the blocked form refuses per-item lengths
    assert _pair(prec, a, xin, w1, b1, w2, b2, dil, lens=lens, form="blocked", x_out=out if enc else None, enc=enc) == -5


def _gru(gi, whh_t, bhh, lens=None):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    B, T = gi.shape[:2]
    out = torch.full((B, T, 512), SENT, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    if lens is None:
        _lib.check(lib.vfx_gru_layer(p(gi), p(whh_t), p(bhh), B, T, p(out), None), "vfx_gru_layer")
    else:
        _lib.check(lib.vfx_gru_layer_ragged(p(gi), p(whh_t), p(bhh), B, T, p(lens), p(out), None), "vfx_gru_layer_ragged")
    torch.cuda.synchronize()
    return out


def _torch_gru(gi, whh, bhh, dtype):
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


@pytest.mark.parametrize("B", [1, 17, 33])
def test_gru_ragged_fp64(B):
    """Each item against torch.nn.GRU in float64 on the item alone (the same bound as the equal-length test: within twice
    torch's own fp32 GRU error) and bit-identical to vfx_gru_layer on the item alone.  B = 1, 17 and 33 use the three
    cluster sizes."""
    T = 40
    g = torch.Generator().manual_seed(300 + B)
    gi = torch.randn(B, T, 2, 768, generator=g).to(DEV)
    whh = ((torch.rand(2, 768, 256, generator=g) * 2 - 1) / 16).to(DEV)
    bhh = ((torch.rand(2, 768, generator=g) * 2 - 1) / 16).to(DEV)
    whh_t = whh.transpose(1, 2).contiguous()
    lens_l = [T] + [int(v) for v in torch.randint(1, T + 1, (B - 1,), generator=g)]
    if B > 2:
        lens_l[1], lens_l[2] = 1, T - 1
    lens = torch.tensor(lens_l, dtype=torch.int32, device=DEV)
    out = _gru(gi, whh_t, bhh, lens)
    for b, n in enumerate(lens_l):
        item = gi[b:b + 1, :n].contiguous()
        alone = _gru(item, whh_t, bhh)
        assert torch.equal(out[b, :n], alone[0]), f"item {b} (T = {n}) differs from the item alone"
        with torch.backends.cudnn.flags(enabled=False):
            ref = _torch_gru(item.to(F64), whh.to(F64), bhh.to(F64), F64)[0]
            t32 = _torch_gru(item, whh, bhh, torch.float32)[0]
        err = float((out[b, :n].to(F64) - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
        err_t = float((t32.to(F64) - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
        assert err <= 2 * err_t + 1e-8, f"item {b}: {err:.2e} against float64, torch fp32 {err_t:.2e}"


# ============================================================================ 5. public API
def test_restore_batch_list(states):
    from voicefixer_b200.api import VoiceFixer
    eng = _engine(states, "tf32")
    vf = VoiceFixer.from_engine(eng)
    items = _items([1025, 30000, 2 * SR + 1], 5)
    calls = []
    real = eng.make_graph
    eng.make_graph = lambda *a, **k: (calls.append(k.get("lens") is not None), real(*a, **k))[1]
    try:
        got = vf.restore_batch(items)
        assert calls == [True]
        for i, a in enumerate(items):
            one = vf.restore_batch(a[None])[0]
            assert isinstance(got[i], np.ndarray) and got[i].shape == a.shape
            assert np.array_equal(got[i], one), f"item {i} differs from restore_batch(item[None])[0]"
        n_calls = len(calls)
        items2 = _items([5000, 3 * SR, 44100], 6)                           # same B, same cap (3 s): no new capture
        got2 = vf.restore_batch(items2)
        assert len(calls) == n_calls
        for i, a in enumerate(items2):
            assert np.array_equal(got2[i], vf.restore_batch(a[None])[0])
    finally:
        del eng.make_graph
    for bad in ([], [np.zeros((2, 5000), np.float32)], [np.zeros(1024, np.float32)],
                [np.zeros(30 * SR + 1, np.float32)]):
        with pytest.raises(ValueError):
            vf.restore_batch(bad)
