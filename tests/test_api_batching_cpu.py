"""The batch steps that restore_many, Vocoder.forward_many and Vocoder.oracle_many share, without a GPU: the packer of
plan_many / plan_vocoder_many, the mode-2 dropout-mask source and the batch stager."""
import numpy as np
import pytest
import torch

from voicefixer_b200 import api, resample

CAPS = [1, 2, 3, 64, 0]                  # 0: a max_items that never fits a second item


def _plan_many_packer(segs, max_items):
    """plan_many's packing, written out on its own: segments (recording, start, stop) sorted longest first, stable."""
    segs = sorted(segs, key=lambda s: s[1] - s[2])
    batches, k = [], 0
    while k < len(segs):
        L_cap = segs[k][2] - segs[k][1]
        n = max(1, int(max_items(L_cap)))
        batches.append((L_cap, segs[k:k + n]))
        k += n
    return batches


def _vocoder_packer(lengths, max_items):
    """plan_vocoder_many's packing, written out on its own: item indices sorted longest first, stable."""
    order = sorted(range(len(lengths)), key=lambda i: -lengths[i])
    batches, k = [], 0
    while k < len(order):
        cap = lengths[order[k]]
        n = max(1, int(max_items(cap)))
        batches.append((cap, order[k:k + n]))
        k += n
    return batches


def _recorder(cap):
    asked = []
    return asked, lambda L: asked.append(L) or cap


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("seed", range(6))
def test_pack_equals_both_packers(seed, cap):
    rng = np.random.default_rng(seed)
    lengths = [int(n) for n in rng.integers(1, 12, size=int(rng.integers(1, 40)))]   # a narrow range: many ties
    asked, max_items = _recorder(cap)
    got = api._pack(lengths, max_items)
    want_asked, want_max = _recorder(cap)
    assert got == _vocoder_packer(lengths, want_max)
    assert asked == want_asked                              # once per batch, in batch order

    segs = [(int(rng.integers(0, 5)), a, a + n) for a, n in zip(np.cumsum([0] + lengths[:-1]).tolist(), lengths)]
    asked, max_items = _recorder(cap)
    got = [(L_cap, [segs[j] for j in idx]) for L_cap, idx in api._pack([b - a for _, a, b in segs], max_items)]
    want_asked, want_max = _recorder(cap)
    assert got == _plan_many_packer(segs, want_max)
    assert asked == want_asked


def test_pack_with_a_max_items_that_varies_by_capacity():
    lengths = [5, 9, 9, 2, 7, 9, 5, 1]
    fn = lambda c: c % 3                                    # noqa: E731  0, 1 or 2 items by capacity
    assert api._pack(lengths, fn) == _vocoder_packer(lengths, fn)
    assert api._pack(lengths, fn) == [(9, [1]), (9, [2]), (9, [5]), (7, [4]), (5, [0, 6]), (2, [3, 7])]


@pytest.mark.parametrize("seed", [0, 7])
def test_default_masks_are_the_seeded_draw(seed):
    B, T = 3, 70
    torch.manual_seed(seed)
    got = api._drop_masks(None, B, T)
    after = torch.rand(4)
    torch.manual_seed(seed)
    want = torch.rand(2, B, T, 512) >= 0.5
    assert got.dtype == torch.uint8 and torch.equal(got, want.to(torch.uint8))
    assert torch.equal(after, torch.rand(4))                # exactly one draw: the generator is where it would be


def test_supplied_masks_pass_through_as_uint8():
    seen = []

    def fn(B, T):
        seen.append((B, T))
        return np.random.default_rng(1).random((2, B, T, 512)) >= 0.5

    got = api._drop_masks(fn, 2, 66)
    assert seen == [(2, 66)]
    assert got.dtype == torch.uint8 and torch.equal(got, torch.as_tensor(fn(2, 66)).to(torch.uint8))


def test_no_dropout_gives_none_and_draws_nothing():
    torch.manual_seed(3)
    assert api._drop_masks(False, 2, 66) is None
    after = torch.rand(4)
    torch.manual_seed(3)
    assert torch.equal(after, torch.rand(4))


def test_masks_of_the_wrong_shape_are_refused():
    with pytest.raises(ValueError, match=r"dropout masks must have shape \(2, 3, 70, 512\), got \(2, 3, 69, 512\)"):
        api._drop_masks(lambda B, T: torch.ones(2, B, T - 1, 512), 3, 70)


class _NoResampler:
    def resample(self, *args):
        raise AssertionError("the resampler ran")


class _RecordingResampler:
    def resample(self, x, table, cap):
        self.call = (x, table, cap)
        return "batch"


def _items():
    rng = np.random.default_rng(5)
    return [rng.standard_normal(n).astype(np.float32) for n in (9000, 20000, 1500)]


def test_batch_input_at_44100_copies_the_ranges():
    items = _items()
    ranges = [(1, 3000, 19000), (0, 0, 9000), (2, 0, 1500), (1, 0, 10)]
    cap = 16003
    x, lens = api._batch_input(_NoResampler(), items, [44100] * 3, ranges, cap, "cpu")
    assert x.shape == (len(ranges), cap) and x.dtype == torch.float32
    assert lens.dtype == torch.int32 and lens.tolist() == [b - a for _, a, b in ranges]
    for k, (i, a, b) in enumerate(ranges):
        assert np.array_equal(x[k, :b - a].numpy().view(np.uint32), items[i][a:b].view(np.uint32))
        assert bool((x[k, b - a:] == 0).all())


def test_batch_input_resamples_when_a_rate_differs():
    items = _items()
    rates = [44100, 16000, 44100]
    n = [resample.out_len(a.shape[0], r) for a, r in zip(items, rates)]
    ranges = [(1, 0, n[1]), (0, 100, n[0]), (2, 0, n[2])]
    eng = _RecordingResampler()
    assert api._batch_input(eng, items, rates, ranges, n[1], "cpu") == "batch"
    x, table, cap = eng.call
    want_x, want_table = api._stage(items, rates, ranges, "cpu")
    assert torch.equal(x, want_x) and table == want_table and cap == n[1]


def test_pad_rows_keeps_trailing_dimensions():
    rows = [torch.ones(3, 128, dtype=torch.float64), torch.full((5, 128), 2.0)]
    x, lens = api._pad_rows(rows, 6, "cpu")
    assert x.shape == (2, 6, 128) and x.dtype == torch.float32 and lens.tolist() == [3, 5]
    assert bool((x[0, :3] == 1).all() and (x[0, 3:] == 0).all() and (x[1, :5] == 2).all() and (x[1, 5:] == 0).all())
