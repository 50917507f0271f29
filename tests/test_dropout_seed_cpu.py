"""CPU tests of mode 2's seeded dropout: the host Philox restatement against the published known answers, the masks'
statistics, the seed and key helpers of the public API, and the new C entry points (planning-only engine)."""
import ctypes

import numpy as np
import pytest

from voicefixer_b200 import api
from voicefixer_b200.philox import philox4x32_10, seeded_masks

# Random123's kat_vectors for philox4x32_10: (counter, key, output)
KAT = [
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
     [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
]


@pytest.mark.parametrize("ctr,key,out", KAT)
def test_philox_known_answers(ctr, key, out):
    assert philox4x32_10(np.array(ctr), np.array(key)).tolist() == out


def test_philox_is_vectorised_over_counters():
    ctr = np.array([k[0] for k in KAT])
    key = np.array([k[1] for k in KAT])
    assert philox4x32_10(ctr, key).tolist() == [k[2] for k in KAT]


def test_mask_layout_is_the_documented_bit_order():
    seed, stream, T = (1 << 64) - 3, (1 << 40) + 7, 5
    m = seeded_masks(seed, stream, T)
    assert m.shape == (2, T, 512) and m.dtype == np.uint8
    for l in (0, 1):
        for t in (0, T - 1):
            for j in (0, 31, 32, 127, 128, 300, 511):
                w = philox4x32_10(np.array([t, 4 * l + j // 128, stream & 0xFFFFFFFF, stream >> 32]),
                                  np.array([seed & 0xFFFFFFFF, seed >> 32]))
                assert m[l, t, j] == (int(w[(j % 128) // 32]) >> (j % 32)) & 1


def test_masks_are_deterministic_and_differ_across_seed_stream_and_layer():
    a = seeded_masks(7, 0, 200)
    assert np.array_equal(a, seeded_masks(7, 0, 200))
    assert np.array_equal(a[:, :50], seeded_masks(7, 0, 50))                 # a frame's bits do not depend on T
    for other in (seeded_masks(8, 0, 200), seeded_masks(7, 1, 200), seeded_masks(7, 1 << 32, 200),
                  seeded_masks(7 + (1 << 32), 0, 200)):
        assert not np.array_equal(a, other)
    assert not np.array_equal(a[0], a[1])


def test_keep_fraction_is_one_half_per_layer_and_unit():
    T = 3001
    m = seeded_masks(12345, 3, T).astype(np.float64)
    for l in (0, 1):                                                         # per layer: T * 512 bits
        n = T * 512
        assert abs(m[l].mean() - 0.5) < 6 * 0.5 / np.sqrt(n)
    per_unit = m.mean(axis=1)                                                # (2, 512), T bits each
    assert np.all(np.abs(per_unit - 0.5) < 6 * 0.5 / np.sqrt(T))


def test_bits_of_different_streams_agree_half_the_time():
    T = 3001
    a, b = seeded_masks(99, 0, T), seeded_masks(99, 1, T)
    n = a.size
    assert abs(np.mean(a == b) - 0.5) < 6 * 0.5 / np.sqrt(n)
    c = seeded_masks(100, 0, T)
    assert abs(np.mean(a == c) - 0.5) < 6 * 0.5 / np.sqrt(n)


def test_seeded_masks_refuse_out_of_range_keys():
    for seed, stream in ((-1, 0), (1 << 64, 0), (0, -1), (0, 1 << 64)):
        with pytest.raises(ValueError):
            seeded_masks(seed, stream, 3)


# ------------------------------------------------------------------ seed and key helpers of the API
@pytest.mark.parametrize("bad", [True, np.bool_(False), 1.0, 2.5, "3", None, -1, 1 << 64, np.int64(-5)])
def test_bad_seed_is_refused_naming_the_recording(bad):
    with pytest.raises(ValueError, match=r"restore_many: recording 1 has dropout_seed"):
        api.dropout_seeds([0, bad, 2], 2, None, 3, "restore_many")
    if bad is not None:
        with pytest.raises(ValueError, match=r"restore_inmem has dropout_seed"):
            api.check_dropout_seed(bad, "restore_inmem")


def test_good_seeds_one_or_one_per_recording():
    top = (1 << 64) - 1
    assert api.dropout_seeds(5, 2, None, 3, "restore_many") == [5, 5, 5]
    assert api.dropout_seeds([0, top, np.uint64(top)], 2, None, 3, "restore_many") == [0, top, top]
    assert api.dropout_seeds(np.array([1, 2], dtype=np.uint64), 2, None, 2, "restore_many") == [1, 2]
    assert api.dropout_seeds((np.int64(3),), 2, None, 1, "restore_many") == [3]
    assert api.dropout_seeds(None, 0, lambda B, T: None, 3, "restore_many") is None     # no seed: nothing checked


def test_wrong_seed_count_mode_or_mask_source_is_refused():
    with pytest.raises(ValueError, match="dropout_seed has 2 entries for 3 recordings"):
        api.dropout_seeds([1, 2], 2, None, 3, "restore_many")
    for mode in (0, 1):
        with pytest.raises(ValueError, match="dropout_seed is mode 2's dropout"):
            api.dropout_seeds(1, mode, None, 1, "restore_many")
    for fn in (False, lambda B, T: None):
        with pytest.raises(ValueError, match="dropout_seed or drop_masks_fn, not both"):
            api.dropout_seeds(1, 2, fn, 1, "restore_many")


def test_key_rows_follow_the_segments_of_a_multi_segment_plan():
    S = api.SEG_LENGTH
    lengths = [S + 44100 * 5, 44100 * 3, 2 * S + 44100 * 2]
    seeds = [11, (1 << 64) - 1, 7]
    plan = api.plan_many(lengths, 2, lambda L: 2)
    assert sum(len(segs) for _, segs in plan) == 6 and len(plan) > 1
    for _, segs in plan:
        rows = api.drop_key_rows(segs, seeds)
        assert rows.dtype == np.uint64 and rows.shape == (len(segs), 2)
        assert rows.tolist() == [[seeds[i], a // S] for i, a, _ in segs]
    keys = sorted(tuple(r) for _, segs in plan for r in api.drop_key_rows(segs, seeds).tolist())
    assert keys == sorted([(11, 0), (11, 1), (seeds[1], 0), (7, 0), (7, 1), (7, 2)])
    # the bit pattern the engine reads: int64 view, two's complement above 2^63
    assert api.drop_key_rows([(1, 0, 100)], seeds).view(np.int64).tolist() == [[-1, 0]]


# ------------------------------------------------------------------ the C entry points
def test_seeded_entry_points_are_declared_exported_and_refuse_bad_calls(states):
    from voicefixer_b200 import _lib
    from voicefixer_b200.engine import Planner
    from voicefixer_b200.weights import pack_analysis, pack_vocoder
    lib = _lib.load()
    for name in ("vfx_restore_seeded", "vfx_analysis_seeded", "vfx_dropout_seeded"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    pl = Planner(dict(pack_analysis(states[0], "tf32"), **pack_vocoder(states[1], "tf32")), "tf32")
    one, keys = ctypes.c_void_p(4096), ctypes.c_void_p(8192)
    # a planning-only engine never launches; missing or misaligned keys are refused first
    assert lib.vfx_restore_seeded(pl.h, one, 1, 44100, None, keys, one, one, 1 << 30, None) == -1
    assert b"planning-only" in lib.vfx_last_error()
    assert lib.vfx_analysis_seeded(pl.h, one, 1, 101, keys, one, one, 1 << 30, None) == -1
    assert b"planning-only" in lib.vfx_last_error()
    for bad in (None, ctypes.c_void_p(8196)):
        assert lib.vfx_restore_seeded(pl.h, one, 1, 44100, None, bad, one, one, 1 << 30, None) == -1
        assert b"keys" in lib.vfx_last_error()
        assert lib.vfx_analysis_seeded(pl.h, one, 1, 101, bad, one, one, 1 << 30, None) == -1
        assert b"keys" in lib.vfx_last_error()
    assert lib.vfx_restore_seeded(pl.h, one, 65536, 44100, None, keys, one, one, 1 << 30, None) == -1
    assert b"65535" in lib.vfx_last_error()
    # the kernel's entry point: every argument error before any launch (no CUDA call is made)
    x = ctypes.c_void_p(4096)
    for args, what in (((None, 1, 8, keys, 0), b"bad arguments"), ((x, 1, 8, None, 0), b"bad arguments"),
                       ((x, 1, 8, keys, 2), b"layer"), ((x, 1, 8, keys, -1), b"layer"),
                       ((x, 65536, 8, keys, 0), b"65535"), ((x, 0, 8, keys, 0), b"bad arguments"),
                       ((x, 1, 0, keys, 0), b"bad arguments"), ((ctypes.c_void_p(4100), 1, 8, keys, 0), b"aligned"),
                       ((x, 1, 8, ctypes.c_void_p(8196), 1), b"aligned")):
        assert lib.vfx_dropout_seeded(*args, None) == -1, args
        assert what in lib.vfx_last_error(), (args, lib.vfx_last_error())


def test_workspace_sizes_are_unchanged(states):
    """The keys are caller-owned device memory, so the seeded entry points share vfx_workspace_bytes: the 20 x 30 s
    bf16 restore workspace is still the figure a GPU run of that batch allocates."""
    from voicefixer_b200.engine import Planner
    from voicefixer_b200.weights import pack_analysis, pack_vocoder
    pl = Planner(dict(pack_analysis(states[0], "bf16"), **pack_vocoder(states[1], "bf16")), "bf16")
    assert pl.workspace_bytes(20, 44100 * 30) == 17168495616
