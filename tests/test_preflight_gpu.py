"""Every C-ABI entry point that takes a workspace refuses one below the call's need before its first launch: it returns
VFX_ERR_WORKSPACE with "workspace too small", launches nothing and leaves its output untouched.  The size the matching
planner reports is accepted."""
import pytest
import torch

from voicefixer_b200.engine import _ptr, _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = -1920.0
B, T, L = 2, 20, 9000
TC = T + T % 2 + 4                                   # the vocoder's conditioning frames for T mel frames
TC_L = (1 + L // 441) + (1 + L // 441) % 2 + 4       # ... for L samples

_ENGINE = {}


def _engine(states):
    if not _ENGINE:
        from voicefixer_b200.engine import Engine
        _ENGINE[0] = Engine(states[0], states[1], precision="tf32")
    return _ENGINE[0]


def _out(*shape):
    return torch.full(shape, SENT, device=DEV)


def _case(eng, name):
    """(call(ws, nbytes) -> status, output, the planner's size) for one entry point on a small batch."""
    lib, h = eng.lib, eng.h
    g = torch.Generator().manual_seed(0)
    mel = (torch.rand(B, T, 128, generator=g) + 0.01).to(DEV)
    wav = (0.3 * torch.randn(B, L, generator=g)).to(DEV)
    frames = torch.tensor([T // 2, T], dtype=torch.int32, device=DEV)
    lens = torch.tensor([L // 3, L], dtype=torch.int32, device=DEV)
    if name == "vfx_analysis":
        out = _out(B, T, 128)
        return (lambda ws, n: lib.vfx_analysis(h, _ptr(mel), B, T, 0, None, _ptr(out), _ptr(ws), n, _stream()),
                out, eng.workspace_bytes_frames(B, T))
    if name == "vfx_vocoder":
        out = _out(B, TC * 441)
        return (lambda ws, n: lib.vfx_vocoder(h, _ptr(mel), B, T, 0, _ptr(out), -1, 1.0, _ptr(ws), n, _stream()),
                out, eng.workspace_bytes_frames(B, T))
    if name == "vfx_vocoder_cond":
        out = _out(B, T * 441)                     # the mels stand in for T rows of normalised conditions
        return (lambda ws, n: lib.vfx_vocoder_cond(h, _ptr(mel), B, T, _ptr(out), -1, 1.0, _ptr(ws), n, _stream()),
                out, eng.workspace_bytes_frames(B, T))
    if name == "vfx_vocoder_ragged":
        out = _out(B, TC * 441)
        return (lambda ws, n: lib.vfx_vocoder_ragged(h, _ptr(mel), B, T, _ptr(frames), 0, _ptr(out), 1.0, _ptr(ws), n,
                                                     _stream()),
                out, eng.workspace_bytes_frames(B, T))
    if name == "vfx_oracle_cond":
        out = _out(B, TC_L, 128)
        return (lambda ws, n: lib.vfx_oracle_cond(h, _ptr(wav), B, L, _ptr(lens), _ptr(out), _ptr(ws), n, _stream()),
                out, 4 * B)
    if name == "vfx_oracle":
        out = _out(B, TC_L * 441)
        return (lambda ws, n: lib.vfx_oracle(h, _ptr(wav), B, L, _ptr(lens), 1.0, _ptr(out), _ptr(ws), n, _stream()),
                out, eng.oracle_workspace_bytes(B, L))
    if name == "vfx_restore":
        out = _out(B, L)
        return (lambda ws, n: lib.vfx_restore(h, _ptr(wav), B, L, 0, None, _ptr(out), _ptr(ws), n, _stream()),
                out, eng.workspace_bytes(B, L))
    if name == "vfx_restore_ragged_mode":
        out = _out(B, L)
        return (lambda ws, n: lib.vfx_restore_ragged_mode(h, _ptr(wav), B, L, _ptr(lens), 0, None, _ptr(out), _ptr(ws), n,
                                                          _stream()),
                out, eng.workspace_bytes(B, L))
    assert name == "vfx_hf_cut"
    out = _out(B, 512 * (L // 512))
    cut = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    return (lambda ws, n: lib.vfx_hf_cut(h, _ptr(wav), B, L, 0.95, _ptr(out), _ptr(cut), _ptr(ws), n, _stream()),
            out, eng.hf_cut_workspace_bytes(B, L))


@pytest.mark.parametrize("name", ["vfx_analysis", "vfx_vocoder", "vfx_vocoder_cond", "vfx_vocoder_ragged",
                                  "vfx_oracle_cond", "vfx_oracle", "vfx_restore", "vfx_restore_ragged_mode",
                                  "vfx_hf_cut"])
def test_too_small_workspace_is_refused_before_any_launch(states, name):
    eng = _engine(states)
    call, out, need = _case(eng, name)
    small = 4 if name == "vfx_oracle_cond" else 4096
    assert need > small
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    assert call(ws, small) == -3
    assert b"workspace too small" in eng.lib.vfx_last_error()
    torch.cuda.synchronize()
    assert eng.launch_count() == n0
    assert bool((out == SENT).all()), "a refused call wrote its output"
    assert call(ws, need) == 0, eng.lib.vfx_last_error()
    torch.cuda.synchronize()
    assert eng.launch_count() > n0
