"""Ragged batches without a GPU: the list form's validation and capacity rounding, and the C / ctypes descriptors."""
import os
import re
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 44100


def test_ragged_plan_rounds_capacity_to_whole_seconds():
    from voicefixer_b200.api import ragged_plan
    items, lens, cap = ragged_plan([np.zeros(1025), np.ones(SR, np.float64), [0.5] * 2000])
    assert lens == [1025, SR, 2000] and cap == SR
    assert all(a.dtype == np.float32 and a.flags.c_contiguous for a in items)
    assert ragged_plan([np.zeros(SR + 1, np.float32)])[2] == 2 * SR
    assert ragged_plan([np.zeros(30 * SR, np.float32), np.zeros(5000, np.float32)])[2] == 30 * SR


@pytest.mark.parametrize("bad,match", [
    ([], "non-empty list"),
    ([np.zeros(5000, np.float32), np.zeros((2, 5000), np.float32)], "item 1 has shape"),
    ([np.zeros(1024, np.float32)], "at least 1025"),
    ([np.zeros(30 * SR + 1, np.float32)], "more than 30 s"),
])
def test_ragged_plan_rejects_bad_items(bad, match):
    from voicefixer_b200.api import ragged_plan
    with pytest.raises(ValueError, match=match):
        ragged_plan(bad)


def test_pair_desc_layout_matches_header():
    """ctypes mirror of struct vfx_pair_desc has the same field order as the header (lens is the last field)."""
    from voicefixer_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "vfx_b200.h")).read()
    body = re.search(r"typedef struct vfx_pair_desc \{(.*?)\} vfx_pair_desc;", hdr, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for stmt in body.split(";"):
        stmt = stmt.strip()
        if not stmt:
            continue
        for part in re.split(r"[;,]", stmt):
            part = re.sub(r"^(const\s+)?(void|float|int|size_t)\s*\*?", "", part.strip())
            names.append(part.replace("*", "").strip())
    assert names == [f[0] for f in _lib.PairDesc._fields_]
    assert names[-1] == "lens"


def test_conv_desc_extent_fields_are_last():
    """Zero-initialised descriptors (memset / ctypes) keep their meaning: the extent fields trail the struct."""
    from voicefixer_b200 import _lib
    assert [f[0] for f in _lib.ConvDesc._fields_][-3:] == ["seq_in", "seq_out", "seq_axis"]
    d = _lib.ConvDesc()
    assert d.seq_in is None and d.seq_out is None and d.seq_axis == 0


def test_ragged_entry_points_are_bound():
    from voicefixer_b200 import _lib
    lib = _lib.load()
    for name in ("vfx_restore_ragged", "vfx_gru_layer_ragged"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)


def test_planner_workspace_holds_the_extent_table(states):
    """The ragged path takes its extent table (15 int32 per item) from the planner's slack: one workspace size
    serves vfx_restore and vfx_restore_ragged.  The planner's numbers for up to 68 items are what they were before."""
    from voicefixer_b200 import weights
    from voicefixer_b200.engine import Planner
    packed = dict(weights.pack_analysis(states[0], "fp32"))
    packed.update(weights.pack_vocoder(states[1], "fp32"))
    p = Planner(packed, "fp32")
    for B in (1, 64, 100):
        assert p.workspace_bytes(B, 3 * SR) > 0
    extra = p.workspace_bytes(100, 3 * SR) - p.workspace_bytes(99, 3 * SR)
    per_item = p.workspace_bytes(65, 3 * SR) - p.workspace_bytes(64, 3 * SR)
    assert extra >= per_item
