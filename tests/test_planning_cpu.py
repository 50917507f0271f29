"""Workspace planners on planning-only engines (no GPU): every size the library reports for a restore, frames or oracle
call, and the mode-1 pre-filter's workspace.

The expected sizes are literals from the build before the planners and the launching calls came to share one dry pass,
so a change in what the dry pass allocates shows here as a changed number."""
import pytest

SR = 44100
BS = [1, 2, 7, 64, 68, 69, 70]                  # the extent table fits the 4 KB slack up to 68 items
LS = [1025, SR, 10 * SR, 30 * SR]
FRAMES = [(1, 1), (1, 64), (2, 101), (7, 3001), (70, 500)]
ORACLE = [(1, 1), (2, 9000), (7, 10 * SR), (70, SR)]

# vfx_workspace_bytes(B, L): rows BS, columns LS.  TF32 keeps fp32 storage, so its sizes are fp32's.
RESTORE_FP32 = [
    [14363904, 48488448, 459982848, 1374414848],
    [28714240, 96972800, 919961600, 2748825600],
    [100492032, 339394560, 3219855360, 9620879360],
    [918707200, 3103002624, 29438644224, 87962292224],
    [976126720, 3296940032, 31278559232, 93459935232],
    [990486016, 3345424640, 31738538240, 94834346240],
    [1004836352, 3393908992, 32198516992, 96208756992],
]
RESTORE_BF16 = [
    [11762944, 30281472, 287292672, 858428672],
    [23512320, 60558848, 574581248, 1716853248],
    [82285312, 211945728, 2011024128, 6008976128],
    [752245760, 1937756160, 18386472960, 54939176960],
    [799261440, 2058865664, 19535627264, 58372875264],
    [811019776, 2089143296, 19822916096, 59231300096],
    [822769152, 2119420672, 20110204672, 60089724672],
]
RESTORE = {"fp32": RESTORE_FP32, "tf32": RESTORE_FP32, "bf16": RESTORE_BF16}
# vfx_workspace_bytes_frames on FRAMES: (full weight set, vocoder-only weight set)
FRAMES_FP32 = ([14359296, 31082496, 96869376, 9610123776, 16114098432],
               [2766336, 31082496, 96869376, 9610123776, 16114098432])
FRAMES_BF16 = ([11758336, 19398144, 60455424, 5998220544, 10057496832],
               [1724160, 19398144, 60455424, 5998220544, 10057496832])
FRAMES_BYTES = {"fp32": FRAMES_FP32, "tf32": FRAMES_FP32, "bf16": FRAMES_BF16}
# vfx_oracle_workspace_bytes on ORACLE (the same for both weight sets)
ORACLE_BYTES = {"fp32": [2762496, 23771904, 3212677120, 3386670336],
                "tf32": [2762496, 23771904, 3212677120, 3386670336],
                "bf16": [1720320, 14821632, 2003845888, 2112182016]}

_PLANNERS = {}


def _planners(states, prec):
    """(full, vocoder-only) planning-only engines."""
    if prec not in _PLANNERS:
        from voicefixer_b200.engine import Planner
        from voicefixer_b200.weights import pack_analysis, pack_vocoder
        voc = pack_vocoder(states[1], prec)
        _PLANNERS[prec] = Planner(dict(pack_analysis(states[0], prec), **voc), prec), Planner(voc, prec)
    return _PLANNERS[prec]


@pytest.mark.parametrize("prec", ["fp32", "bf16", "tf32"])
def test_restore_workspace_is_unchanged(states, prec):
    full, voc = _planners(states, prec)
    got = [[full.workspace_bytes(B, L) for L in LS] for B in BS]
    assert got == RESTORE[prec]
    assert voc.workspace_bytes(1, SR) == 0 and voc.workspace_bytes(2, 10 * SR) == 0    # restore() needs the analysis module


@pytest.mark.parametrize("prec", ["fp32", "bf16", "tf32"])
def test_frames_and_oracle_workspace_are_unchanged(states, prec):
    full, voc = _planners(states, prec)
    assert [full.workspace_bytes_frames(B, T) for B, T in FRAMES] == FRAMES_BYTES[prec][0]
    assert [voc.workspace_bytes_frames(B, T) for B, T in FRAMES] == FRAMES_BYTES[prec][1]
    for p in (full, voc):
        assert [p.oracle_workspace_bytes(B, L) for B, L in ORACLE] == ORACLE_BYTES[prec]


def test_hf_cut_workspace_is_the_librarys():
    """vfx_hf_cut_workspace_bytes is hf_cut.cu's buffer plan: the spectra, the frames, the energies, the cut bins and
    4 KB of slack that covers each buffer's 256-byte alignment.  Engine.hf_cut_workspace_bytes returns the same without
    an engine."""
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import Engine
    lib = _lib.load()
    for B in [1, 2, 7, 64, 15359, 15360, 15361]:
        for L in [0, 511, 512, 1536, SR, 30 * SR]:
            nfr = 1 + L // 512
            want = B * nfr * 1025 * 8 + B * nfr * 2048 * 4 + B * 1025 * 8 + 4 * B + 4096
            assert lib.vfx_hf_cut_workspace_bytes(B, L) == want, (B, L)
            assert Engine.hf_cut_workspace_bytes(B, L) == want, (B, L)
    assert lib.vfx_hf_cut_workspace_bytes(-1, SR) == 0 and lib.vfx_hf_cut_workspace_bytes(1, -1) == 0
