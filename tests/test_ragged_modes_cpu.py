"""restore_many without a GPU: the segmenting and packing plan, its validation, and the bindings of the ragged mode-1 /
mode-2 entry points."""
import os
import re
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 44100
SEG = 30 * SR


def _inmem_segments(n):
    """restore_inmem's loop (voicefixer/base.py:117-119) on an index array: the sample indices of each segment."""
    idx = np.arange(n)
    segs, bp = [], SEG
    while bp < n + SEG:
        segs.append(idx[bp - SEG: bp])
        bp += SEG
    return segs


LENGTHS = [66150, SEG, SEG + SR, 65 * SR, 3 * SR, 2 * SEG, 1025 + 512, 90 * SR + 44100]


@pytest.mark.parametrize("n", LENGTHS)
def test_segments_match_restore_inmem(n):
    from voicefixer_b200.api import segment_bounds
    got = segment_bounds(n)
    want = _inmem_segments(n)
    assert [(int(s[0]), int(s[-1]) + 1) for s in want] == got


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("cap", [1, 2, 3, 64])
def test_plan_covers_every_sample_once_and_respects_max_items(mode, cap):
    from voicefixer_b200.api import plan_many
    asked = []

    def max_items(L_cap):
        asked.append(L_cap)
        return cap

    lengths = [n for n in LENGTHS if mode != 2 or n > 64 * 441]   # mode 2 refuses segments of 64 frames or fewer
    plan = plan_many(lengths, mode, max_items)
    assert asked == [L_cap for L_cap, _ in plan]
    seen = {i: [] for i in range(len(lengths))}
    prev_cap = None
    for L_cap, segs in plan:
        assert 1 <= len(segs) <= cap
        lens = [b - a for _, a, b in segs]
        assert L_cap == max(lens) == lens[0]                       # capacity = the batch's longest segment
        assert lens == sorted(lens, reverse=True)
        assert prev_cap is None or L_cap <= prev_cap               # batches ordered by length
        prev_cap = L_cap
        for i, a, b in segs:
            seen[i].append((a, b))
    for i, n in enumerate(lengths):
        spans = sorted(seen[i])
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(spans[k][1] == spans[k + 1][0] for k in range(len(spans) - 1))   # once each, in order, no gaps
        assert spans == [(int(s[0]), int(s[-1]) + 1) for s in _inmem_segments(n)]


def test_plan_packs_all_recordings_together():
    from voicefixer_b200.api import plan_many
    plan = plan_many([2 * SR, 5 * SR, 3 * SR], 0, lambda L: 64)
    assert len(plan) == 1 and plan[0][0] == 5 * SR
    assert [s[0] for s in plan[0][1]] == [1, 2, 0]


@pytest.mark.parametrize("lengths,mode,match", [
    ([], 0, "non-empty list"),
    ([5000, 0], 0, "recording 1 is empty"),
    ([5000, 1024], 0, "recording 1 has a segment .* of 1024 samples"),
    ([SEG + 1024, 5000], 0, r"recording 0 has a segment \(samples 1323000\.\.1324024\)"),
    ([5000, 1535], 1, "recording 1 has a segment .* 1024 after the mode-1 pre-filter"),
    ([SEG + 1500], 1, "recording 0 has a segment"),
    ([64 * 441 - 1], 2, "recording 0, .*Expected more than 1 value per channel when training"),
    ([60000, SEG + 64 * 441 - 1], 2, r"recording 1, samples 1323000\.\.1351223: Expected more than 1 value"),
    ([5000], 3, "mode must be 0, 1 or 2"),
])
def test_plan_validation_messages(lengths, mode, match):
    from voicefixer_b200.api import plan_many
    calls = []
    with pytest.raises(ValueError, match=match):
        plan_many(lengths, mode, lambda L: calls.append(L) or 8)
    assert calls == []                                             # nothing is sized (or launched) before validation


def test_plan_accepts_the_smallest_segments():
    from voicefixer_b200.api import plan_many
    assert plan_many([1025], 0, lambda L: 1)[0][0] == 1025
    assert plan_many([1536], 1, lambda L: 1)[0][0] == 1536
    assert plan_many([64 * 441], 2, lambda L: 1)[0][0] == 64 * 441


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "vfx_b200.h")).read()
    m = re.search(r"\b" + name + r"\((.*?)\);", hdr, flags=re.S)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["vfx_restore_ragged_mode", "vfx_hf_cut_ragged"])
def test_new_entry_points_bound_like_the_header(name):
    from voicefixer_b200 import _lib
    assert name in _lib.SIGNATURES
    lib = _lib.load()
    assert hasattr(lib, name)
    args = _header_args(name)
    assert len(_lib.SIGNATURES[name][1]) == len(args)
    floats = [i for i, a in enumerate(args) if a.startswith("float ")]
    assert [i for i, t in enumerate(_lib.SIGNATURES[name][1]) if t is _lib._f] == floats
