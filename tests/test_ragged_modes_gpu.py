"""Ragged batches in modes 1 and 2 (vfx_hf_cut_ragged, vfx_restore_ragged_mode, Engine.hf_cut(lens=...),
Engine.restore(lens=..., mode=2)) and VoiceFixer.restore_many.

Every row must be bit-identical to the same item run alone, whatever the other items, the capacity or the contents of
the padding and of the workspace.  The pre-filter's energy and the train-mode statistics are sums in double with
atomics; the identities rest on the float rounding of those sums not depending on their order."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100
PRECS = ["fp32", "tf32", "bf16", "fp16"]

# pre-filter: 3 frames (1536), the last length with 4 frames (2047), 5 frames (2048), L % 512 = 511, the capacity (3 s)
HF_LENS = [1536, 2047, 2048, 512 * 50 + 511, 3 * SR]
HF_CAP = 3 * SR
# mode 2: T = 65 (the first length the reference accepts), T = 128 / 129 (the Tp boundary 128 -> 192), an odd T
# (227) and the capacity (T = 301)
M2_LENS = [64 * 441, 128 * 441 - 1, 128 * 441, 100000, 3 * SR]
M2_CAP = 3 * SR

_ENGINES = {}


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


def _poison_ws(eng, nbytes):
    """Fills the engine's shared workspace (at least nbytes) with 0xFF bytes (NaN as fp32)."""
    ws = eng._workspace(nbytes)
    ws.fill_(0xFF)
    return ws


def _dev(a):
    return torch.from_numpy(a)[None].to(DEV)


def _check_rows(y, ns, alone, what):
    for i, n in enumerate(ns):
        assert torch.equal(y[i, :n], alone[i]), f"{what}: item {i} (L = {n}) differs from the same item run alone"
        assert bool((y[i, n:] == 0).all()), f"{what}: item {i} (L = {n}): samples past its length are not zero"


# ============================================================================ 1. the mode-1 pre-filter
@pytest.mark.parametrize("poison", [False, True])
def test_hf_cut_ragged_rows_equal_items_alone(states, poison):
    eng = _engine(states, "fp32")
    items = _items(HF_LENS, 11)
    alone = [eng.hf_cut(_dev(a)) for a in items]
    alone_out = [o[0].clone() for o, _ in alone]
    alone_cut = [int(c[0]) for _, c in alone]
    x, lens = _batch(items, HF_CAP, pad=float("nan") if poison else 0.0)
    if poison:
        _poison_ws(eng, eng.hf_cut_workspace_bytes(len(items), HF_CAP))
    out, cut, lens_out = eng.hf_cut(x, lens=lens)
    torch.cuda.synchronize()
    assert out.shape == (len(items), HF_CAP)
    assert lens_out.tolist() == [512 * (n // 512) for n in HF_LENS]
    assert cut.tolist() == alone_cut
    _check_rows(out, [512 * (n // 512) for n in HF_LENS], alone_out, "hf_cut")


@pytest.mark.parametrize("prec", PRECS)
def test_mode1_ragged_rows_equal_items_alone(states, prec):
    """hf_cut(lens=) then restore(lens=lens_out) on the device, without a host round trip."""
    eng = _engine(states, prec)
    items = _items(HF_LENS, 12)
    alone = []
    for a in items:
        f, _ = eng.hf_cut(_dev(a))
        alone.append(eng.restore(f)[0].clone())
    x, lens = _batch(items, HF_CAP)
    f, _, lens_out = eng.hf_cut(x, lens=lens)
    y = eng.restore(f, lens=lens_out)
    torch.cuda.synchronize()
    _check_rows(y, [512 * (n // 512) for n in HF_LENS], alone, "mode 1")


# ============================================================================ 2. mode 2 (train-mode statistics per item)
def _masks(B, T, seed):
    return torch.rand(2, B, T, 512, generator=torch.Generator().manual_seed(seed)) >= 0.5


def _mode2_alone(eng, items, masks):
    out = []
    for b, a in enumerate(items):
        T_b = 1 + a.shape[0] // 441
        m = None if masks is None else masks[:, b:b + 1, :T_b]
        out.append(eng.restore(_dev(a), mode=2, drop_masks=m)[0].clone())
    return out


@pytest.mark.parametrize("prec", PRECS)
def test_mode2_ragged_rows_equal_items_alone(states, prec):
    eng = _engine(states, prec)
    items = _items(M2_LENS, 21)
    B, T_cap = len(items), 1 + M2_CAP // 441
    masks = _masks(B, T_cap, 22)
    for m in (masks, None):
        alone = _mode2_alone(eng, items, m)
        x, lens = _batch(items, M2_CAP)
        y = eng.restore(x, mode=2, drop_masks=m, lens=lens)
        torch.cuda.synchronize()
        _check_rows(y, M2_LENS, alone, "mode 2" + (" with masks" if m is not None else ""))
        # NaN past every item's length and 0xFF bytes in the whole workspace: a statistic over rows past an item's
        # extent, or one BatchNorm left without extents, turns its row non-finite
        x, lens = _batch(items, M2_CAP, pad=float("nan"))
        ws = torch.full((eng.workspace_bytes(B, M2_CAP),), 0xFF, dtype=torch.uint8, device=DEV)
        y = eng.restore(x, mode=2, drop_masks=m, lens=lens, ws=ws)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(y).all())
        _check_rows(y, M2_LENS, alone, "mode 2 on NaN padding and a stale workspace")


def test_mode2_ragged_capacity_invariance(states):
    eng = _engine(states, "tf32")
    items = _items([64 * 441, 80000, 2 * SR], 23)
    masks = _masks(len(items), 1 + 4 * SR // 441, 24)
    ys = []
    for cap in (2 * SR, 4 * SR):
        x, lens = _batch(items, cap)
        ys.append(eng.restore(x, mode=2, drop_masks=masks[:, :, :1 + cap // 441], lens=lens).clone())
    torch.cuda.synchronize()
    for i, a in enumerate(items):
        n = a.shape[0]
        assert torch.equal(ys[0][i, :n], ys[1][i, :n]), f"item {i} depends on the batch capacity"


def test_mode2_ragged_rejects_mask_shape(states):
    eng = _engine(states, "tf32")
    x, lens = _batch(_items([70000, 80000], 25), 2 * SR)
    with pytest.raises(ValueError, match="drop_masks must have shape"):
        eng.restore(x, mode=2, drop_masks=_masks(2, 1 + 2 * SR // 441 - 1, 26), lens=lens)


def test_mode2_ragged_row_against_oracle(states):
    """One fp32 ragged mode-2 row against the CPU oracle of the reference's restore_inmem(mode=2), same masks."""
    from oracle import vf_oracle as O
    from conftest import rel_rms
    eng = _engine(states, "fp32")
    items = _items(M2_LENS, 27)
    B, T_cap = len(items), 1 + M2_CAP // 441
    masks = _masks(B, T_cap, 28)
    x, lens = _batch(items, M2_CAP)
    y = eng.restore(x, mode=2, drop_masks=masks, lens=lens)
    torch.cuda.synchronize()
    b = 2                                                           # T = 129: UNet padded to Tp = 192
    n = items[b].shape[0]
    T_b = 1 + n // 441
    ref = O.restore_inmem(items[b], states[0], states[1], mode=2, drop_masks_fn=lambda T: masks[:, b:b + 1, :T_b])
    err = rel_rms(y[b, :n].cpu().numpy()[None], ref)
    assert err < 2e-4, f"relative RMS {err:.2e} against the oracle"


# ============================================================================ 3. restore_many
MANY_LENS = [66150, 31 * SR, 65 * SR, 3 * SR]      # 1.5 s, a full segment plus a 1 s tail, two segments plus 5 s, 3 s


def test_restore_many_equals_restore_inmem(states):
    from voicefixer_b200.api import VoiceFixer
    eng = _engine(states, "tf32")
    vf = VoiceFixer.from_engine(eng)
    wavs = _items(MANY_LENS, 31)
    for mode, fn in ((0, None), (1, None), (2, False)):
        got = vf.restore_many(wavs, mode=mode, drop_masks_fn=fn)
        assert len(got) == len(wavs)
        for i, w in enumerate(wavs):
            want = vf.restore_inmem(w, cuda=True, mode=mode, drop_masks_fn=fn)
            assert got[i].shape == want.shape and got[i].dtype == want.dtype
            assert np.array_equal(got[i], want), f"mode {mode}: recording {i} differs from restore_inmem"
    torch.manual_seed(32)
    got = vf.restore_many(wavs, mode=2)                                # random dropout masks
    for g, w in zip(got, wavs):
        assert g.shape == (1, w.shape[0]) and np.isfinite(g).all()
    shapes = []
    got = vf.restore_many(wavs, mode=2, drop_masks_fn=lambda B, T: shapes.append((B, T)) or _masks(B, T, 33))
    assert shapes and all(np.isfinite(g).all() for g in got)
    with pytest.raises(ValueError, match="dropout masks must have shape"):
        vf.restore_many(wavs, mode=2, drop_masks_fn=lambda B, T: _masks(B, T - 1, 34))


@pytest.mark.parametrize("wavs,mode,match", [
    ([np.zeros(30 * SR + 1000, np.float32)], 0, "recording 0 has a segment"),
    ([np.zeros(5000, np.float32), np.zeros(30 * SR + 1500, np.float32)], 1, "recording 1 has a segment"),
    ([np.zeros(70000, np.float32), np.zeros(30 * SR + 64 * 441 - 1, np.float32)], 2, "recording 1, .*more than 1 value"),
    ([np.zeros((2, 5000), np.float32)], 0, "recording 0 has shape"),
    ([], 0, "non-empty list"),
])
def test_restore_many_rejects_before_launching(states, wavs, mode, match):
    from voicefixer_b200.api import VoiceFixer
    eng = _engine(states, "tf32")
    vf = VoiceFixer.from_engine(eng)
    n0 = eng.launch_count()
    with pytest.raises(ValueError, match=match):
        vf.restore_many(wavs, mode=mode)
    assert eng.launch_count() == n0
