"""The pure half of device-resident restore_many / oracle_many (voicefixer_b200.api), without a GPU: the rows each
batch reads (vfx_resample_src items) and writes (vfx_scatter_rows items) for recordings around the 30 s boundary in
every mode, that the written ranges tile every output exactly once, and the ValueErrors for lists that cannot run on the
device (fake tensor-like items stand in for CUDA tensors)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from voicefixer_b200 import api, resample
from voicefixer_b200.api import SEG_LENGTH, _gen_len, _net_len, plan_many, plan_vocoder_many, segment_bounds

SR = 44100
LENGTHS = [SEG_LENGTH, 95 * SR, SEG_LENGTH + 2 * SR, 2 * SEG_LENGTH, 3 * SR + 17]   # every segment > 64 frames


def _tiles(lengths, mode, max_items):
    """{recording: [(dst_off, len), ...]} of every row restore_many writes, over all batches, and the batches."""
    written = {i: [] for i in range(len(lengths))}
    batches = plan_many(lengths, mode, max_items)
    for _, segs in batches:
        for (i, a, b), (j, off, n) in zip(segs, api.restore_rows(segs, mode)):
            assert j == i and n == _net_len(b - a, mode)
            written[i].append((off, n))
    return written, batches


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("per_batch", [1, 2, 64])
def test_restore_rows_tile_each_output_once(mode, per_batch):
    written, batches = _tiles(LENGTHS, mode, lambda L: per_batch)
    for i, n in enumerate(LENGTHS):
        total = api.restore_out_len(n, mode)
        assert total == sum(_net_len(b - a, mode) for a, b in segment_bounds(n))
        cover = np.zeros(total, np.int32)
        for off, k in written[i]:
            assert 0 <= off and off + k <= total
            cover[off:off + k] += 1
        assert (cover == 1).all(), f"mode {mode}: recording {i} ({n} samples)"
    # segments of one recording fall into different batches when batches are small; every batch writes only its own
    if per_batch == 1:
        assert len({i for _, segs in batches for i, _, _ in segs}) == len(LENGTHS)
        assert len(batches) == sum(len(segment_bounds(n)) for n in LENGTHS)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_restore_rows_around_the_30s_boundary(mode):
    seg = _net_len(SEG_LENGTH, mode)
    segs = [(0, 0, SEG_LENGTH), (1, SEG_LENGTH, SEG_LENGTH + 1025), (2, 2 * SEG_LENGTH, 95 * SR), (2, 0, SEG_LENGTH)]
    assert api.restore_rows(segs, mode) == [
        (0, 0, seg), (1, seg, _net_len(1025, mode)), (2, 2 * seg, _net_len(95 * SR - 2 * SEG_LENGTH, mode)), (2, 0, seg)]
    assert api.restore_out_len(SEG_LENGTH, mode) == seg
    assert api.restore_out_len(SEG_LENGTH + 1, mode) == seg + _net_len(1, mode)
    assert api.restore_out_len(95 * SR, mode) == 3 * seg + _net_len(95 * SR - 3 * SEG_LENGTH, mode)
    if mode == 1:
        assert seg == 512 * (SEG_LENGTH // 512) < SEG_LENGTH


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_thirty_seconds_and_one_sample_is_refused_by_the_plan(mode):
    """30 s + 1 leaves a 1-sample segment, which restore_inmem cannot restore either: the plan refuses it, naming it,
    on the host and the device path alike (oracle_many takes it whole: test_oracle_rows_one_whole_output_per_item)."""
    with pytest.raises(ValueError, match=r"recording 1.*samples 1323000\.\.1323001"):
        plan_many([SEG_LENGTH, SEG_LENGTH + 1], mode, lambda L: 64)


@pytest.mark.parametrize("rates", [[SR] * 3, [16000, SR, 48000], [8000, 22050, 96000]])
def test_resample_rows_read_each_segment_of_its_stream(rates):
    n_in = [SEG_LENGTH, 95 * 16000, 31 * 48000]
    lengths = [resample.out_len(n, r) for n, r in zip(n_in, rates)]
    for _, segs in plan_many(lengths, 0, lambda L: 3):
        rows = api.resample_rows(segs, rates)
        assert rows == [(i, rates[i], a, b - a) for i, a, b in segs]
        for i, rate, y_first, y_len in rows:                            # inside the stream vfx_resample_src validates
            assert 0 <= y_first and y_first + y_len <= resample.out_len(n_in[i], rate) and y_len <= SEG_LENGTH


def test_oracle_rows_one_whole_output_per_item():
    lengths = [1025, SEG_LENGTH, SEG_LENGTH + 1, 95 * SR]
    items = [np.ones(n, np.float32) for n in lengths]
    seen = []
    for _, idx in plan_vocoder_many(items, "wav", lambda L: 2):
        for i, off, n in api.oracle_rows(idx, lengths):
            assert off == 0 and n == _gen_len(1 + lengths[i] // 441)
            seen.append(i)
    assert sorted(seen) == list(range(len(lengths)))


def _fake(shape=(4410,), dtype=torch.float32, device="cuda:0", stride=1):
    """Stands in for a CUDA tensor: check_device_items reads only is_cuda, device, dtype, shape and stride."""
    return SimpleNamespace(is_cuda=True, device=torch.device(device), dtype=dtype, shape=shape, stride=lambda d: stride)


def test_host_lists_stay_on_the_host_path():
    assert api.check_device_items([np.zeros(3), torch.zeros(3), [0.0, 1.0]], torch.device("cuda:0"), "x") is False
    assert api.check_device_items([], torch.device("cuda:0"), "x") is False
    assert api.check_device_items([_fake(), _fake((7,), stride=3)], torch.device("cuda:0"), "x") is True


@pytest.mark.parametrize("items,match", [
    ([_fake(), np.zeros(4410, np.float32)], "restore_many: recording 1 is not a CUDA tensor but recording 0 is"),
    ([torch.zeros(4410), _fake()], "restore_many: recording 0 is not a CUDA tensor but recording 1 is"),
    ([_fake(), _fake(dtype=torch.float64)], "restore_many: recording 1 has dtype torch.float64"),
    ([_fake(dtype=torch.float16)], "restore_many: recording 0 has dtype torch.float16"),
    ([_fake(), _fake((4410, 2))], r"restore_many: recording 1 has shape \(4410, 2\); each recording must be 1-D"),
    ([_fake(())], r"restore_many: recording 0 has shape \(\)"),
    ([_fake(), _fake(device="cuda:1")], "restore_many: recording 1 is on cuda:1; this engine runs on cuda:0"),
    ([_fake(), _fake(stride=0)], r"restore_many: recording 1 has element stride 0 \(an expanded tensor\)"),
])
def test_refusals_name_the_recording(items, match):
    with pytest.raises(ValueError, match=match):
        api.check_device_items(items, torch.device("cuda:0"), "restore_many")


# ============================================================================ the two library entries, without a GPU
def _header_args(name):
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vfx_b200.h")).read()
    m = re.search(r"\b" + name + r"\((.*?)\);", hdr, flags=re.S)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["vfx_resample_src", "vfx_scatter_rows"])
def test_entries_bound_like_the_header(name):
    from voicefixer_b200 import _lib
    args, types = _header_args(name), _lib.SIGNATURES[name][1]
    assert hasattr(_lib.load(), name) and len(types) == len(args) and args[-1] == "void* stream"
    for t, kind in ((_lib._ll, "long long "), (_lib._i, "int ")):
        assert [i for i, a in enumerate(args) if a.startswith(kind)] == [i for i, u in enumerate(types) if u is t]


def test_table_layouts_and_workspaces():
    import ctypes
    from voicefixer_b200 import _lib
    assert ctypes.sizeof(_lib.ResampleSrcItem) == 64 and ctypes.sizeof(_lib.ScatterItem) == 32
    lib = _lib.load()
    for query, item in ((lib.vfx_resample_src_workspace_bytes, 64), (lib.vfx_scatter_rows_workspace_bytes, 32)):
        assert query(0) == 0 and query(-1) == 0
        assert all(query(B) >= item * B for B in (1, 7, 64, 65535))


# Device pointers are never dereferenced by a refused call: fake addresses stand in for them.
@pytest.mark.parametrize("case,match", [
    ("null", "item 1: dst is null"),
    ("long", "item 1: len 5000 is not in [0, ldx = 4096]"),
    ("negative", "item 0: len -1"),
    ("outside", "item 1: destination [9000, 10100) is not inside its 10000 elements"),
    ("overlap", "item 1: its destination overlaps item 0's"),
])
def test_scatter_rows_refuses_a_bad_table_before_any_cuda_call(case, match):
    from voicefixer_b200 import _lib
    lib = _lib.load()
    table = (_lib.ScatterItem * 2)()
    for b, (dst, off, n) in enumerate([(0x100000, 4000, 1000), (0x100000, 5000, 1100)]):
        table[b].dst, table[b].dst_elems, table[b].dst_off, table[b].len = dst, 10000, off, n
    if case == "null":
        table[1].dst = None
    elif case == "long":
        table[1].len = 5000
    elif case == "negative":
        table[0].len = -1
    elif case == "outside":
        table[1].dst_off = 9000
    else:
        table[0].dst_off = 4100                  # [4100, 5100) runs into item 1's [5000, 6100)
    rc = lib.vfx_scatter_rows(0x1000, 2, 4096, table, 0x2000, 4096, None)
    assert rc == -1 and match.encode() in lib.vfx_last_error(), lib.vfx_last_error()
