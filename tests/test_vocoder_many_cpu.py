"""Vocoder.forward_many / oracle_many without a GPU: the packing plan, its validation, the oracle's workspace planner on a
planning-only engine, and the bindings of the new entry points."""
import os
import re
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mels(frames):
    return [np.zeros((1, 1, T, 128), np.float32) for T in frames]


def _check_plan(plan, lengths, cap, asked):
    assert asked == [c for c, _ in plan]
    order = [i for _, idx in plan for i in idx]
    assert sorted(order) == list(range(len(lengths)))                      # every item exactly once
    want = sorted(range(len(lengths)), key=lambda i: -lengths[i])         # longest first, stable on ties
    assert order == want
    for c, idx in plan:
        assert 1 <= len(idx) <= cap
        assert c == lengths[idx[0]] == max(lengths[i] for i in idx)


@pytest.mark.parametrize("cap", [1, 2, 3, 64])
def test_mel_plan_orders_longest_first_stable_and_chunks(cap):
    from voicefixer_b200.api import plan_vocoder_many
    frames = [5, 1001, 5, 64, 1, 1001, 65, 5, 300]
    asked = []
    plan = plan_vocoder_many(_mels(frames), "mel", lambda T: asked.append(T) or cap)
    _check_plan(plan, frames, cap, asked)
    if cap == 64:
        assert plan == [(1001, [1, 5, 8, 6, 3, 0, 2, 7, 4])]


@pytest.mark.parametrize("cap", [1, 3])
def test_wav_plan_orders_longest_first_stable_and_chunks(cap):
    from voicefixer_b200.api import plan_vocoder_many
    lens = [441, 96076, 441, 1, 5 * 44100, 96076]
    wavs = [np.ones(n, np.float32) for n in lens]
    asked = []
    plan = plan_vocoder_many(wavs, "wav", lambda L: asked.append(L) or cap)
    _check_plan(plan, lens, cap, asked)


def test_plan_never_asks_for_zero_items():
    from voicefixer_b200.api import plan_vocoder_many
    plan = plan_vocoder_many(_mels([3, 2, 1]), "mel", lambda T: 0)            # a single item that does not fit runs alone
    assert plan == [(3, [0]), (2, [1]), (1, [2])]


@pytest.mark.parametrize("kind,items,exc,match", [
    ("mel", [], ValueError, "forward_many takes a non-empty list"),
    ("wav", [], ValueError, "oracle_many takes a non-empty list"),
    ("mel", [np.zeros((1, 1, 4, 128)), np.zeros((1, 1, 4, 127))], AssertionError, "item 1 .*128 bins"),
    ("mel", [np.zeros((1, 4, 128))], ValueError, r"item 0 has shape \(1, 4, 128\)"),
    ("mel", [np.zeros((1, 1, 4, 128)), np.zeros((2, 1, 4, 128))], ValueError, "item 1 .*must be \\[1, 1, T >= 1, 128\\]"),
    ("mel", [np.zeros((1, 2, 4, 128))], ValueError, "item 0"),
    ("mel", [np.zeros((1, 1, 0, 128))], ValueError, "item 0"),
    ("wav", [np.ones(10, np.float32), np.zeros(0, np.float32)], ValueError, "item 1 is empty"),
    ("wav", [np.ones((2, 10), np.float32)], ValueError, "item 0 .*1-D"),
    ("wav", [np.ones(10, np.float32), np.ones(3, np.float32), np.zeros(500, np.float32)], ValueError,
     "item 2 is all zeros"),
])
def test_plan_validation_messages(kind, items, exc, match):
    from voicefixer_b200.api import plan_vocoder_many
    calls = []
    with pytest.raises(exc, match=match):
        plan_vocoder_many(items, kind, lambda n: calls.append(n) or 8)
    assert calls == []                                                     # nothing is sized (or launched) first


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_oracle_workspace_on_planning_only_vocoder_engine(states, precision):
    from voicefixer_b200.engine import Planner
    from voicefixer_b200.weights import pack_vocoder
    pv = Planner(pack_vocoder(states[1], precision), precision)
    one, two, eight = (pv.oracle_workspace_bytes(B, 44100) for B in (1, 2, 8))
    assert 0 < one < two < eight
    assert pv.oracle_workspace_bytes(8, 44100) == eight                   # deterministic
    assert 0 < pv.oracle_workspace_bytes(1, 1) < one                       # one sample is a whole (6-row) item
    assert pv.oracle_workspace_bytes(1, 10 * 44100) > one
    for B, L in ((0, 44100), (-1, 44100), (1, 0), (1, -5), (1, 2 ** 31 - 1)):
        assert pv.oracle_workspace_bytes(B, L) == 0


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "vfx_b200.h")).read()
    m = re.search(r"^(?:int|size_t) " + name + r"\((.*?)\);", hdr, flags=re.S | re.M)   # the declaration, not a comment
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["vfx_vocoder_ragged", "vfx_oracle_cond", "vfx_oracle", "vfx_oracle_workspace_bytes"])
def test_new_entry_points_bound_like_the_header(name):
    from voicefixer_b200 import _lib
    assert name in _lib.SIGNATURES
    lib = _lib.load()
    assert hasattr(lib, name)
    args = _header_args(name)
    sig = _lib.SIGNATURES[name][1]
    assert len(sig) == len(args)
    floats = [i for i, a in enumerate(args) if a.startswith("float ")]
    assert [i for i, t in enumerate(sig) if t is _lib._f] == floats
    ints = [i for i, a in enumerate(args) if a.startswith("int ")]
    assert [i for i, t in enumerate(sig) if t is _lib._i] == ints
