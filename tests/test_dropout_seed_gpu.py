"""Mode 2's seeded dropout on the GPU: vfx_dropout_seeded against the host restatement (voicefixer_b200.philox) bit for
bit; Engine.restore / Engine.analysis with drop_keys against the explicit-mask path given the restated masks, in every
precision; restore_inmem and restore_many with dropout_seed against drop_masks_fn returning the restated masks; and
restore_many's batching invariance: each recording's output depends on its samples and seed only, whatever the other
recordings, their order, the batch plan, host or CUDA input, or sample_rate.  No host mask is drawn on the seeded path."""
import gc

import numpy as np
import pytest
import torch

from voicefixer_b200 import _lib, api, synthetic
from voicefixer_b200.api import SEG_LENGTH, VoiceFixer
from voicefixer_b200.engine import Engine, _ptr, _stream
from voicefixer_b200.philox import seeded_masks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100
TOP = (1 << 64) - 1

_ENGINES = {}


@pytest.fixture(scope="module")
def weights():
    return synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1)


@pytest.fixture(scope="module")
def eng_for(weights):
    def get(prec):
        if prec not in _ENGINES:
            _ENGINES[prec] = Engine(weights[0], weights[1], precision=prec)
        return _ENGINES[prec]
    yield get
    # the engines' weights and their workspaces, sized for 30 s batches, go back to the device, so that the tests
    # after this module find the memory they found before it (a VoiceFixer and its model shim form a cycle that
    # keeps an engine alive until the cycle collector runs)
    _ENGINES.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _wav(n, seed):
    return (0.3 * np.random.default_rng(seed).standard_normal(int(n))).astype(np.float32)


def _keys(pairs):
    """int64 (B, 2) CUDA tensor of (seed, stream) bit patterns."""
    return torch.from_numpy(np.array(pairs, dtype=np.uint64).reshape(-1, 2).view(np.int64)).to(DEV)


def _masks(pairs, T):
    """uint8 (2, B, T, 512): the restated masks of each item, stacked as the explicit-mask path takes them."""
    return torch.from_numpy(np.stack([seeded_masks(s, k, T) for s, k in pairs], 1))


def _bits(t):
    t = torch.as_tensor(t)
    return t.detach().cpu().contiguous().view(torch.int32)


def _same(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    return tuple(a.shape) == tuple(b.shape) and torch.equal(_bits(a), _bits(b))


# ============================================================================ 1. the kernel
@pytest.mark.parametrize("T", [1, 77, 301])
def test_dropout_seeded_kernel_equals_the_restated_masks(T):
    lib = _lib.load()
    pairs = [(0, 0), (1, 5), (1 << 63, 1), (TOP, TOP), (12345, 1 << 32)]
    B = len(pairs)
    x = torch.randn(B, T, 512, device=DEV)
    keys = _keys(pairs)
    m = _masks(pairs, T).to(DEV).bool()
    for layer in (0, 1):
        y = x.clone()
        _lib.check(lib.vfx_dropout_seeded(_ptr(y), B, T, _ptr(keys), layer, _stream()), "vfx_dropout_seeded")
        want = torch.where(m[layer], x * 2.0, torch.zeros_like(x))
        assert _same(y, want), f"T {T} layer {layer}"
    # one item alone, at its own pitch, gives its rows of the batch
    y1 = x[3:4].clone()
    _lib.check(lib.vfx_dropout_seeded(_ptr(y1), 1, T, _ptr(keys[3:4]), 1, _stream()), "vfx_dropout_seeded")
    assert _same(y1[0], torch.where(m[1, 3], x[3] * 2.0, torch.zeros_like(x[3])))


# ============================================================================ 2. the engine: keys against masks
PRECS = ["fp32", "tf32", "fp16", "bf16"]


@pytest.mark.parametrize("prec", PRECS)
def test_engine_restore_keys_equal_restated_masks(eng_for, prec):
    eng = eng_for(prec)
    pairs = [(7, 0), (TOP, 3), (1 << 63, 1)]
    # equal lengths: 2 s (T = 201)
    L = 2 * SR
    x = torch.from_numpy(np.stack([_wav(L, 30 + k) for k in range(3)])).to(DEV)
    got = eng.restore(x, mode=2, drop_keys=_keys(pairs))
    want = eng.restore(x, mode=2, drop_masks=_masks(pairs, 1 + L // 441))
    assert _same(got, want), prec
    # ragged: 3 s capacity, items of 3 s, 1.6 s and 2.2 s
    L_cap, ns = 3 * SR, [3 * SR, 70560, 97020]
    x = torch.zeros(3, L_cap, device=DEV)
    for k, n in enumerate(ns):
        x[k, :n] = torch.from_numpy(_wav(n, 40 + k)).to(DEV)
    lens = torch.tensor(ns, dtype=torch.int32, device=DEV)
    got = eng.restore(x, mode=2, drop_keys=_keys(pairs), lens=lens)
    want = eng.restore(x, mode=2, drop_masks=_masks(pairs, 1 + L_cap // 441), lens=lens)
    assert _same(got, want), prec
    # each ragged row is the item restored alone with its key
    for k, n in enumerate(ns):
        alone = eng.restore(x[k:k + 1, :n], mode=2, drop_keys=_keys(pairs[k:k + 1]))
        assert _same(got[k, :n], alone[0]), (prec, k)


@pytest.mark.parametrize("prec", PRECS)
def test_engine_analysis_keys_equal_restated_masks(eng_for, prec):
    eng = eng_for(prec)
    pairs = [(3, 2), (TOP - 1, 0)]
    mel = eng.frontend(torch.from_numpy(np.stack([_wav(2 * SR, 50 + k) for k in range(2)])).to(DEV))
    T = mel.shape[1]
    got = eng.analysis(mel, mode=2, drop_keys=_keys(pairs))
    want = eng.analysis(mel, mode=2, drop_masks=_masks(pairs, T))
    assert _same(got, want), prec


def test_engine_refuses_keys_with_masks_or_outside_mode_2(eng_for):
    eng = eng_for("tf32")
    x = torch.from_numpy(_wav(2 * SR, 1)[None]).to(DEV)
    keys = _keys([(1, 0)])
    with pytest.raises(ValueError, match="give one of them"):
        eng.restore(x, mode=2, drop_keys=keys, drop_masks=_masks([(1, 0)], 201))
    with pytest.raises(ValueError, match="mode 2"):
        eng.restore(x, mode=0, drop_keys=keys)
    for bad in (keys.cpu(), keys.to(torch.int32), _keys([(1, 0), (2, 0)]), keys.t().contiguous().t()[:, :1]):
        with pytest.raises(ValueError, match="drop_keys must be"):
            eng.restore(x, mode=2, drop_keys=bad)
    mel = eng.frontend(x)
    with pytest.raises(ValueError, match="give one of them"):
        eng.analysis(mel, mode=2, drop_keys=keys, drop_masks=_masks([(1, 0)], mel.shape[1]))


# ============================================================================ 3. the public API against explicit masks
def _mask_source(seed, plan):
    """drop_masks_fn that hands restore_inmem the restated masks of its groups in order: plan = [(segment indices, T)]."""
    calls = list(plan)

    def fn(B, T):
        idxs, T_want = calls.pop(0)
        assert (B, T) == (len(idxs), T_want)
        return _masks([(seed, k) for k in idxs], T)
    fn.calls = calls
    return fn


@pytest.mark.parametrize("hook", [False, True])
def test_restore_inmem_seed_equals_restated_masks(eng_for, hook):
    vf = VoiceFixer.from_engine(eng_for("tf32"))
    wav = _wav(65 * SR, 60)                                       # segments of 30, 30 and 5 s: two lengths
    seed = (1 << 63) + 12345
    kw = {"your_vocoder_func": lambda m: vf._vocoder(m, cuda=True)} if hook else {}
    fn = _mask_source(seed, [([0, 1], 1 + SEG_LENGTH // 441), ([2], 1 + 5 * SR // 441)])
    want = vf.restore_inmem(wav, cuda=True, mode=2, drop_masks_fn=fn, **kw)
    assert fn.calls == []
    got = vf.restore_inmem(wav, cuda=True, mode=2, dropout_seed=seed, **kw)
    assert got.shape == (1, wav.shape[0]) and _same(got, want)


# ============================================================================ 4. batching invariance
LENGTHS = [int(31.7 * SR), 2 * SR, int(4.2 * SR), int(1.5 * SR)]
SEEDS = [3, TOP, 3, 17]


def test_restore_many_each_recording_depends_on_its_samples_and_seed_only(eng_for, monkeypatch):
    vf = VoiceFixer.from_engine(eng_for("tf32"))
    wavs = [_wav(n, 70 + k) for k, n in enumerate(LENGTHS)]
    got = vf.restore_many(wavs, mode=2, dropout_seed=SEEDS)
    for i, w in enumerate(wavs):
        alone = vf.restore_many([w], mode=2, dropout_seed=SEEDS[i])[0]
        inmem = vf.restore_inmem(w, cuda=True, mode=2, dropout_seed=SEEDS[i])
        assert _same(got[i], alone) and _same(got[i], inmem), i
    rev = vf.restore_many(wavs[::-1], mode=2, dropout_seed=SEEDS[::-1])[::-1]
    assert all(_same(a, b) for a, b in zip(got, rev))
    monkeypatch.setattr(Engine, "max_batch", lambda self, L, **kw: 1)
    one = vf.restore_many(wavs, mode=2, dropout_seed=SEEDS)
    assert all(_same(a, b) for a, b in zip(got, one))


@pytest.mark.parametrize("rate", [SR, 16000])
def test_restore_many_host_and_cuda_inputs_are_equal(eng_for, rate):
    vf = VoiceFixer.from_engine(eng_for("tf32"))
    wavs = [_wav(n * rate // SR, 80 + k) for k, n in enumerate(LENGTHS)]
    host = vf.restore_many(wavs, mode=2, dropout_seed=SEEDS, sample_rate=rate)
    dev = vf.restore_many([torch.from_numpy(w).to(DEV) for w in wavs], mode=2, dropout_seed=SEEDS, sample_rate=rate)
    assert all(_same(d, h) for d, h in zip(dev, host))
    if rate != SR:                                                # one recording alone at its rate
        alone = vf.restore_many([wavs[1]], mode=2, dropout_seed=SEEDS[1], sample_rate=rate)[0]
        assert _same(host[1], alone)


def test_seeded_path_draws_no_host_mask_and_never_waits(eng_for, monkeypatch):
    vf = VoiceFixer.from_engine(eng_for("tf32"))

    def boom(*a, **k):
        raise AssertionError("the seeded path drew a host mask")
    monkeypatch.setattr(api, "_drop_masks", boom)
    wavs = [_wav(n, 90 + k) for k, n in enumerate(LENGTHS)]
    vf.restore_inmem(wavs[0], cuda=True, mode=2, dropout_seed=1)
    vf.restore_many(wavs, mode=2, dropout_seed=2)
    dwavs = [torch.from_numpy(w).to(DEV) for w in wavs]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = vf.restore_many(dwavs, mode=2, dropout_seed=SEEDS)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(o).all()) for o in outs)


def test_same_seed_gives_equal_output_and_different_seeds_differ(eng_for):
    vf = VoiceFixer.from_engine(eng_for("tf32"))
    wavs = [_wav(3 * SR, 95), _wav(3 * SR, 95)]                  # the same samples twice
    a = vf.restore_many(wavs, mode=2, dropout_seed=[5, 5])
    b = vf.restore_many(wavs, mode=2, dropout_seed=5)
    c = vf.restore_many(wavs, mode=2, dropout_seed=[5, 6])
    assert _same(a[0], a[1]) and _same(a[0], b[0]) and _same(c[0], a[0])
    assert not np.array_equal(c[1], a[1])
    nodrop = vf.restore_many(wavs[:1], mode=2, drop_masks_fn=False)[0]
    assert not np.array_equal(a[0], nodrop)


def test_bad_seeds_raise_before_anything_is_launched(eng_for):
    vf = VoiceFixer.from_engine(eng_for("tf32"))
    wavs = [_wav(2 * SR, 1), _wav(2 * SR, 2)]
    before = vf._engine.launch_count()
    for kw, match in (({"dropout_seed": [1, -1]}, "recording 1 has dropout_seed"),
                      ({"dropout_seed": [1]}, "1 entries for 2 recordings"),
                      ({"dropout_seed": 1, "mode": 0}, "mode 2's dropout"),
                      ({"dropout_seed": 1, "drop_masks_fn": False}, "not both")):
        with pytest.raises(ValueError, match=match):
            vf.restore_many(wavs, **dict({"mode": 2}, **kw))
    with pytest.raises(ValueError, match="restore_inmem has dropout_seed"):
        vf.restore_inmem(wavs[0], mode=2, dropout_seed=1 << 64)
    with pytest.raises(ValueError, match="mode 2's dropout"):
        vf.restore_inmem(wavs[0], mode=1, dropout_seed=1)
    assert vf._engine.launch_count() == before
