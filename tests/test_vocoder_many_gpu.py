"""Ragged batches through the stand-alone vocoder (vfx_vocoder_ragged, Engine.vocoder(lens=...), Vocoder.forward_many)
and Vocoder.oracle's front end on the device (vfx_oracle_cond, vfx_oracle, Vocoder.oracle_many).

Every row of a ragged batch must be bit-identical to the same item run alone, whatever the other items, the capacity
or the contents of the padding and of the workspace.  The device front end is checked against the host's
oracle_conditions, and the whole device oracle against the CPU oracle at DESIGN.md §2's tolerances."""
import numpy as np
import pytest
import torch
from conftest import rel_rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -1920.0
SR = 44100
PRECS = ["fp32", "tf32", "bf16", "fp16"]
FRAMES = [1, 2, 3, 63, 64, 65, 1001]
T_CAP = 1100
ORACLE_LENS = [1, 440, 441, 442, 2048, 3 * SR]
L_CAP = 3 * SR + 1000

_VOC = {}


def _voc_engine(states, prec):
    """A vocoder-only engine: the reference's stand-alone Vocoder loads nothing but the synthesis checkpoint."""
    if prec not in _VOC:
        from voicefixer_b200.engine import Engine
        from voicefixer_b200.weights import pack_vocoder
        _VOC[prec] = Engine(packed=pack_vocoder(states[1], prec), precision=prec)
    return _VOC[prec]


def _mels(frames, seed):
    g = np.random.default_rng(seed)
    return [np.exp(g.normal(-3.0, 2.0, size=(T, 128))).astype(np.float32) for T in frames]


def _mel_batch(mels, T_cap):
    x = torch.full((len(mels), T_cap, 128), SENT, device=DEV)
    for i, m in enumerate(mels):
        x[i, :m.shape[0]] = torch.from_numpy(m).to(DEV)
    return x, torch.tensor([m.shape[0] for m in mels], dtype=torch.int32, device=DEV)


def _S(T):
    return (T + T % 2 + 4) * 441


def _garbage_ws(nbytes):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)


def _check_rows(y, alone, lengths):
    for i, (a, n) in enumerate(zip(alone, lengths)):
        assert torch.equal(y[i, :n], a), f"item {i} ({n} samples) differs from the same item run alone"
        assert bool((y[i, n:] == 0).all()), f"item {i}: samples past its length are not zero"


def _recordings(lens, seed):
    """Harmonic-plus-noise utterances (every one has a non-zero peak)."""
    g = np.random.default_rng(seed)
    out = []
    for n in lens:
        t = np.arange(n) / SR
        f0 = g.uniform(90, 250)
        x = sum(np.sin(2 * np.pi * f0 * k * t + g.uniform(0, 6.28)) / k for k in range(1, 12))
        x = 0.3 * x * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + 0.02 * g.standard_normal(n)
        out.append(x.astype(np.float32))
    return out


def _wav_batch(items, L_cap, pad=SENT):
    x = torch.full((len(items), L_cap), pad, device=DEV)
    for i, a in enumerate(items):
        x[i, :a.shape[0]] = torch.from_numpy(a).to(DEV)
    return x, torch.tensor([a.shape[0] for a in items], dtype=torch.int32, device=DEV)


# ============================================================================ 1. vfx_vocoder_ragged
@pytest.mark.parametrize("prec", PRECS)
def test_vocoder_ragged_rows_equal_items_alone(states, prec):
    eng = _voc_engine(states, prec)
    mels = _mels(FRAMES + [T_CAP], 1)
    x, lens = _mel_batch(mels, T_CAP)
    y = eng.vocoder(x, lens=lens, ws=_garbage_ws(eng.workspace_bytes_frames(len(mels), T_CAP)))
    assert tuple(y.shape) == (len(mels), _S(T_CAP))
    alone = []
    for m in mels:
        ws1 = _garbage_ws(eng.workspace_bytes_frames(1, m.shape[0]))
        alone.append(eng.vocoder(torch.from_numpy(m)[None].to(DEV), ws=ws1)[0].clone())
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all())
    _check_rows(y, alone, [_S(m.shape[0]) for m in mels])


# ============================================================================ 2. vfx_oracle, bit identity
@pytest.mark.parametrize("prec", PRECS)
def test_oracle_rows_equal_items_alone(states, prec):
    eng = _voc_engine(states, prec)
    items = _recordings(ORACLE_LENS, 2)
    x, lens = _wav_batch(items, L_CAP)
    B = len(items)
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import _ptr, _stream
    ws = _garbage_ws(eng.oracle_workspace_bytes(B, L_CAP))
    T_cap = 1 + L_CAP // 441
    y = torch.empty(B, _S(T_cap), device=DEV)
    _lib.check(eng.lib.vfx_oracle(eng.h, _ptr(x), B, L_CAP, _ptr(lens), 1.0, _ptr(y), _ptr(ws), ws.numel(), _stream()),
               "vfx_oracle")
    alone = []
    for a in items:
        ws1 = _garbage_ws(eng.oracle_workspace_bytes(1, a.shape[0]))
        o = torch.empty(1, _S(1 + a.shape[0] // 441), device=DEV)
        xa = torch.from_numpy(a)[None].to(DEV)
        _lib.check(eng.lib.vfx_oracle(eng.h, _ptr(xa), 1, a.shape[0], None, 1.0, _ptr(o), _ptr(ws1), ws1.numel(),
                                      _stream()), "vfx_oracle")
        alone.append(o[0])
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all())
    _check_rows(y, alone, [_S(1 + a.shape[0] // 441) for a in items])


# ============================================================================ 3. vfx_oracle_cond vs the host front end
def _fe_cases():
    g = np.random.default_rng(7)
    t = np.arange(2 * SR) / SR
    tone = (0.8 * np.sin(2 * np.pi * 440.0 * t)).astype(np.float32)
    quiet = np.concatenate([_recordings([SR], 8)[0], np.zeros(SR // 2, np.float32),
                            (1e-4 * g.standard_normal(SR)).astype(np.float32)])
    return _recordings([3 * SR, 96076, 20000], 3) + [tone, quiet]


def test_oracle_cond_matches_host_front_end(states):
    from voicefixer_b200.api import oracle_conditions
    eng = _voc_engine(states, "tf32")
    items = _fe_cases()
    L_cap = max(a.shape[0] for a in items) + 500
    x, lens = _wav_batch(items, L_cap)
    cond = eng.oracle(x, lens=lens, return_cond=True).cpu().numpy()
    T_cap = 1 + L_cap // 441
    assert cond.shape == (len(items), T_cap + T_cap % 2 + 4, 128)
    worst = 0.0
    for i, a in enumerate(items):
        ref = oracle_conditions(a)[0]
        T = 1 + a.shape[0] // 441
        Tc = T + T % 2 + 4
        assert ref.shape[0] == Tc
        err = float(np.max(np.abs(cond[i, :Tc] - ref)))
        worst = max(worst, err)
        assert err <= 1e-4, f"item {i}: max-abs {err:.3e} against oracle_conditions"
        assert bool((cond[i, T:Tc] == -4.0).all()), f"item {i}: the tail pad rows are not -4"
        assert bool((cond[i, Tc:] == 0.0).all()), f"item {i}: rows after Tc_b are not zero"
    print(f"vfx_oracle_cond vs oracle_conditions: max-abs {worst:.3e}")
    # lens = NULL: every row is L_cap long
    a = items[0]
    c1 = eng.oracle(torch.from_numpy(a)[None].to(DEV), return_cond=True).cpu().numpy()[0]
    assert np.array_equal(c1, cond[0, :c1.shape[0]])


# ============================================================================ 4. parity with the CPU oracle
TOLS = {"fp32": (2e-4, None), "tf32": (2e-3, 1e-3), "fp16": (2e-3, 1e-3), "bf16": (3e-2, 5e-3)}
# fp32: the device front end against the host's, through the same fp32 generator.  Measured on an H100 at 400 W: see
# DESIGN.md §6 (the front ends differ by the order of the mel sums and the float64 FFT's rounding).
HOST_PATH_TOL = 1e-5


@pytest.fixture(scope="module")
def oracle_ref(states):
    from oracle import vf_oracle as O
    wav = _recordings([int(1.5 * SR) + 123], 11)[0]
    return wav, O.oracle_wave(wav, states[1])[0, 0] / 2 ** 15


@pytest.mark.parametrize("prec", PRECS)
def test_oracle_vs_cpu_oracle(states, oracle_ref, prec):
    wav, ref = oracle_ref
    eng = _voc_engine(states, prec)
    y = eng.oracle(torch.from_numpy(wav)[None]).cpu().numpy()[0]
    assert y.shape == ref.shape
    rr, ma = TOLS[prec]
    err = rel_rms(y, ref)
    mean_abs = float(np.mean(np.abs(y - ref)))
    assert err <= rr, f"{prec}: rel-RMS {err:.3e}"
    if ma is not None:
        assert mean_abs <= ma, f"{prec}: mean-abs {mean_abs:.3e}"


def test_oracle_many_vs_host_front_end_path(states):
    from voicefixer_b200 import api
    from voicefixer_b200.api import oracle_conditions
    eng = _voc_engine(states, "fp32")
    voc = api.Vocoder(44100, _engine=eng)
    items = _recordings([int(1.5 * SR) + 123, 20000, 3 * SR], 12)
    got = voc.oracle_many(items)
    worst = 0.0
    for a, y in zip(items, got):
        host = eng.vocoder_cond(torch.from_numpy(oracle_conditions(a))).cpu().numpy()
        assert y.shape == host.shape
        worst = max(worst, rel_rms(y, host))
    print(f"oracle_many vs oracle_conditions -> vocoder_cond (fp32): rel-RMS {worst:.3e}")
    assert worst <= HOST_PATH_TOL


# ============================================================================ 5. API
def _check_forward_many(voc, mels, cuda):
    got = voc.forward_many(mels, cuda=cuda)
    assert len(got) == len(mels)
    for i, m in enumerate(mels):
        want = voc.forward(m, cuda=cuda)
        assert got[i].device == want.device
        assert torch.equal(got[i], want), f"forward_many[{i}] differs from forward"


def test_forward_many_standalone_vocoder_and_voicefixer(tmp_path, monkeypatch):
    from voicefixer_b200 import api, synthetic
    monkeypatch.setenv("HOME", str(tmp_path))
    synthetic.write_checkpoints(str(tmp_path), seed=0)
    mels = [torch.from_numpy(m)[None, None] for m in _mels([5, 120, 1, 64, 120, 301], 4)]
    voc = api.Vocoder(44100, precision="tf32")
    _check_forward_many(voc, mels, cuda=False)
    _check_forward_many(voc, mels, cuda=True)
    # a small per-batch limit: several batches, the order restored
    monkeypatch.setattr(voc._engine, "max_batch_frames", lambda T, **k: 2)
    _check_forward_many(voc, mels, cuda=False)
    vf = api.VoiceFixer(precision="bf16")
    _check_forward_many(vf._model.vocoder, mels, cuda=True)


def test_oracle_many_lengths_and_order(states, monkeypatch):
    from voicefixer_b200 import api
    eng = _voc_engine(states, "tf32")
    voc = api.Vocoder(44100, _engine=eng)
    lens = [96076, 1, 441, 20000, 96076]
    items = _recordings(lens, 5)
    got = voc.oracle_many(items)
    for n, y in zip(lens, got):
        T = 1 + n // 441
        assert y.dtype == np.float32 and y.shape == (1, (T + T % 2 + 4) * 441)
    assert got[0].shape[1] == 97902                # the reference's oracle.flac fixture: 96076 -> 97902 samples
    monkeypatch.setattr(eng, "_fit", lambda *a: 2)
    again = voc.oracle_many(items)
    for a, b in zip(got, again):
        assert np.array_equal(a, b)
    with pytest.raises(ValueError, match="item 1 is all zeros"):
        voc.oracle_many([items[0], np.zeros(500, np.float32)])


# ============================================================================ 6. graph capture
def test_vocoder_ragged_graph_replays_with_new_lengths(states):
    eng = _voc_engine(states, "tf32")
    B, T_cap = 4, 400
    x, lens = _mel_batch(_mels([400, 3, 121, 250], 6), T_cap)
    ws = torch.empty(eng.workspace_bytes_frames(B, T_cap), dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eng.vocoder(x, lens=lens, ws=ws)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = eng.vocoder(x, lens=lens, ws=ws)
    for frames, seed in (([400, 3, 121, 250], 6), ([7, 400, 1, 333], 7)):
        mels = _mels(frames, seed)
        xb, lb = _mel_batch(mels, T_cap)
        x.copy_(xb)
        lens.copy_(lb)
        g.replay()
        torch.cuda.synchronize()
        alone = [eng.vocoder(torch.from_numpy(m)[None].to(DEV))[0] for m in mels]
        torch.cuda.synchronize()
        _check_rows(out, alone, [_S(T) for T in frames])


# ============================================================================ 7. preflight
def test_too_small_workspace_is_refused_before_any_launch(states):
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import _ptr, _stream
    eng = _voc_engine(states, "tf32")
    lib = eng.lib
    x, lens = _mel_batch(_mels([10, 20], 9), 20)
    w, wl = _wav_batch(_recordings([5000, 9000], 9), 9000)
    out = torch.empty(2, _S(1 + 9000 // 441) * 128, device=DEV)
    need_v = eng.workspace_bytes_frames(2, 20)
    need_o = eng.oracle_workspace_bytes(2, 9000)
    ws = torch.empty(max(need_v, need_o), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    calls = [
        lambda: lib.vfx_vocoder_ragged(eng.h, _ptr(x), 2, 20, _ptr(lens), 0, _ptr(out), 1.0, _ptr(ws), 4096, _stream()),
        lambda: lib.vfx_oracle(eng.h, _ptr(w), 2, 9000, _ptr(wl), 1.0, _ptr(out), _ptr(ws), 4096, _stream()),
        lambda: lib.vfx_oracle_cond(eng.h, _ptr(w), 2, 9000, _ptr(wl), _ptr(out), _ptr(ws), 4, _stream()),
    ]
    for call in calls:
        assert call() == -3
        assert b"workspace too small" in lib.vfx_last_error()
    assert eng.launch_count() == n0
    # the sizes the planners give are enough
    assert lib.vfx_vocoder_ragged(eng.h, _ptr(x), 2, 20, _ptr(lens), 0, _ptr(out), 1.0, _ptr(ws), need_v, _stream()) == 0
    assert lib.vfx_oracle(eng.h, _ptr(w), 2, 9000, _ptr(wl), 1.0, _ptr(out), _ptr(ws), need_o, _stream()) == 0
    torch.cuda.synchronize()
