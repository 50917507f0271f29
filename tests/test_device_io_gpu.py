"""Device-resident restore_many / oracle_many: CUDA tensors in, CUDA tensors out.  Each output is bit-identical to the
host call on the items' host copies (modes 0, 1 and 2 without dropout, two precisions, three rate settings), strided
input is read in place and left unchanged, nothing waits on the host (torch's sync debug mode), each batch launches
exactly the two new kernels' share, side streams work (also two streams on one engine, and shared buffers the engine
replaces while a side stream still needs them), one-shot iterables are taken like lists, and the two new library
entries refuse a bad table entry before writing anything and match torch indexing on random tables."""
import numpy as np
import pytest
import torch

from voicefixer_b200 import _lib, resample, synthetic
from voicefixer_b200.api import SEG_LENGTH, VoiceFixer, _pack, _stage, plan_many, restore_out_len
from voicefixer_b200.engine import Engine, _ptr, _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100

_ENGINES = {}


@pytest.fixture(scope="module")
def weights():
    """Seeded synthetic checkpoints."""
    return synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1)


@pytest.fixture(scope="module")
def vf_for(weights):
    def get(prec):
        if prec not in _ENGINES:
            _ENGINES[prec] = Engine(weights[0], weights[1], precision=prec)
        return VoiceFixer.from_engine(_ENGINES[prec])
    yield get
    _ENGINES.clear()


def _wav(n, seed):
    return torch.from_numpy((0.3 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32))


def _same_bits(dev_out, host_out):
    """A device output against the host call's array: float32 CUDA tensor of the same shape and the same bits."""
    assert dev_out.is_cuda and dev_out.device == torch.device(DEV) and dev_out.dtype == torch.float32
    h = torch.from_numpy(np.ascontiguousarray(host_out))
    return tuple(dev_out.shape) == tuple(h.shape) and torch.equal(dev_out.cpu().view(torch.int32), h.view(torch.int32))


# the rate settings: 44.1 kHz only (the default), one int for every recording, one rate per recording (a mix)
RATE_SETTINGS = {"44k": None, "16k": 16000, "mixed": [16000, SR, 48000, 16000]}


def _rates(setting, n):
    r = RATE_SETTINGS[setting]
    return [SR] * n if r is None else (r if isinstance(r, list) else [r] * n)


def _kw(setting):
    r = RATE_SETTINGS[setting]
    return {} if r is None else {"sample_rate": r}


def _recordings(setting, seconds, seed):
    """CUDA recordings of the given lengths (seconds, or ("n", samples)) at the setting's rates."""
    rates = _rates(setting, len(seconds))
    out = []
    for k, (s, r) in enumerate(zip(seconds, rates)):
        n = s[1] if isinstance(s, tuple) else int(round(s * r))
        out.append(_wav(n, seed + k).to(DEV))
    return out


# ============================================================================ 1 + 3. bit-identical to the host call
RESTORE_LENGTHS = {0: [("n", 1025), 30, 95.3, 4.2], 1: [30, 95.3, 4.2, 31.7], 2: [30, 95.3, 4.2, 31.7]}


@pytest.mark.parametrize("setting", list(RATE_SETTINGS))
@pytest.mark.parametrize("prec", ["tf32", "bf16"])
def test_restore_many_on_cuda_tensors_equals_the_host_call(vf_for, prec, setting):
    vf = vf_for(prec)
    for mode in (0, 1, 2):
        wavs = _recordings(setting, RESTORE_LENGTHS[mode], 10 * mode)
        got = vf.restore_many(wavs, mode=mode, drop_masks_fn=False, **_kw(setting))
        want = vf.restore_many([w.cpu().numpy() for w in wavs], mode=mode, drop_masks_fn=False, **_kw(setting))
        assert isinstance(got, list) and len(got) == len(wavs)
        for i in range(len(wavs)):
            assert _same_bits(got[i], want[i]), f"{prec} {setting} mode {mode}: recording {i}"
            n44 = resample.out_len(wavs[i].shape[0], _rates(setting, len(wavs))[i])
            assert tuple(got[i].shape) == (1, restore_out_len(n44, mode))


def test_thirty_seconds_and_one_sample_is_refused_on_both_paths(vf_for):
    """At 44.1 kHz the tail segment has 1 sample; restore_inmem cannot restore it and both paths refuse it alike."""
    vf = vf_for("tf32")
    wavs = [_wav(SEG_LENGTH + 1, 3).to(DEV)]
    with pytest.raises(ValueError) as dev_err:
        vf.restore_many(wavs)
    with pytest.raises(ValueError) as host_err:
        vf.restore_many([wavs[0].cpu().numpy()])
    assert str(dev_err.value) == str(host_err.value)


ORACLE_LENGTHS = [("n", 1025), 30, ("n", SEG_LENGTH + 1), 95.3]


@pytest.mark.parametrize("setting", list(RATE_SETTINGS))
@pytest.mark.parametrize("prec", ["tf32", "bf16"])
def test_oracle_many_on_cuda_tensors_equals_the_host_call(vf_for, prec, setting):
    vf = vf_for(prec)
    wavs = _recordings(setting, ORACLE_LENGTHS, 40)
    got = vf._vocoder.oracle_many(wavs, **_kw(setting))
    want = vf._vocoder.oracle_many([w.cpu().numpy() for w in wavs], **_kw(setting))
    for i in range(len(wavs)):
        assert _same_bits(got[i], want[i]), f"{prec} {setting}: recording {i}"
        n44 = resample.out_len(wavs[i].shape[0], _rates(setting, len(wavs))[i])
        T = 1 + n44 // 441
        assert tuple(got[i].shape) == (1, (T + T % 2 + 4) * 441)


def test_all_zero_cuda_recording_gives_what_the_device_front_end_makes(vf_for):
    """oracle_many reads no device sample on the host, so an all-zero CUDA recording is not refused: its output is
    exactly Engine.oracle's on that row (the front end's zero peak), where the host call raises."""
    vf = vf_for("tf32")
    eng = vf._engine
    z = torch.zeros(5 * SR, device=DEV)
    got = vf._vocoder.oracle_many([z])[0]
    ref = eng.oracle(z[None], lens=torch.tensor([5 * SR], dtype=torch.int32, device=DEV))
    assert torch.equal(got.view(torch.int32), ref[:, :got.shape[1]].view(torch.int32))
    with pytest.raises(ValueError, match="all zeros"):
        vf._vocoder.oracle_many([z.cpu().numpy()])


# ============================================================================ 2. strided input, read in place
def test_strided_channel_equals_its_contiguous_copy_and_is_not_written(vf_for):
    vf = vf_for("tf32")
    x = torch.stack([_wav(int(33.5 * SR), 7), _wav(int(33.5 * SR), 8)], 1).to(DEV)     # (L, 2) interleaved
    y = torch.stack([_wav(int(6.1 * 16000), 9), _wav(int(6.1 * 16000), 10)], 1).to(DEV)
    before = (x.double().sum().item(), y.double().sum().item(), x.clone(), y.clone())
    assert x[:, 1].stride(0) == 2
    for mode in (0, 1, 2):
        got = vf.restore_many([x[:, 1], y[:, 0]], mode=mode, drop_masks_fn=False, sample_rate=[SR, 16000])
        want = vf.restore_many([x[:, 1].contiguous(), y[:, 0].contiguous()], mode=mode, drop_masks_fn=False,
                               sample_rate=[SR, 16000])
        for g, w in zip(got, want):
            assert torch.equal(g.view(torch.int32), w.view(torch.int32)), f"mode {mode}"
    got = vf._vocoder.oracle_many([x[:, 1], y[:, 1]], sample_rate=[SR, 16000])
    want = vf._vocoder.oracle_many([x[:, 1].contiguous(), y[:, 1].contiguous()], sample_rate=[SR, 16000])
    for g, w in zip(got, want):
        assert torch.equal(g.view(torch.int32), w.view(torch.int32))
    torch.cuda.synchronize()
    assert (x.double().sum().item(), y.double().sum().item()) == before[:2]
    assert torch.equal(x, before[2]) and torch.equal(y, before[3])


# ============================================================================ 4. no host wait
@pytest.mark.parametrize("rate", [SR, 16000])
def test_no_host_synchronisation(vf_for, rate):
    vf = vf_for("tf32")
    wavs = [_wav(int(s * rate), 20 + k).to(DEV) for k, s in enumerate((31.0, 3.5))]
    torch.cuda.synchronize()
    outs = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for mode in (0, 1, 2):                           # mode 2 with the default masks: uploaded from pinned memory
            outs.append(vf.restore_many(wavs, mode=mode, sample_rate=rate))
        outs.append(vf._vocoder.oracle_many(wavs, sample_rate=rate))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    for o in outs:
        assert all(bool(torch.isfinite(t).all()) for t in o)


@pytest.mark.parametrize("rate", [SR, 16000])
def test_calls_return_while_earlier_work_still_runs(vf_for, rate):
    """The sync debug mode does not see every synchronising call (e.g. the library's own), so also: with a kernel that
    spins for about a second queued first, each call returns while that kernel is still running."""
    vf = vf_for("tf32")
    wavs = [_wav(int(s * rate), 60 + k).to(DEV) for k, s in enumerate((31.0, 3.5))]
    calls = [lambda m=m: vf.restore_many(wavs, mode=m, sample_rate=rate) for m in (0, 1, 2)]
    calls.append(lambda: vf._vocoder.oracle_many(wavs, sample_rate=rate))
    for k, call in enumerate(calls):
        call()                                           # warm: buffers, workspace and taps exist
        torch.cuda.synchronize()
        torch.cuda._sleep(2 * 10 ** 9)                   # ~1 s at 1.98 GHz
        call()
        busy = not torch.cuda.current_stream().query()
        torch.cuda.synchronize()
        assert busy, f"call {k} waited for the work queued before it"


# ============================================================================ 5. launch accounting
@pytest.mark.parametrize("rate", [SR, 16000])
def test_each_batch_launches_the_new_kernels_once(vf_for, monkeypatch, rate):
    vf = vf_for("tf32")
    eng = vf._engine
    monkeypatch.setattr(eng, "_fit", lambda per_item, cap, reserve: 2)     # the same plan on both paths: 2 per batch
    wavs = [_wav(int(s * rate), 30 + k).to(DEV) for k, s in enumerate((61.0, 3.5, 12.0, 5.0))]
    host = [w.cpu().numpy() for w in wavs]
    lengths = [resample.out_len(w.shape[0], rate) for w in wavs]
    extra = 2 if rate == SR else 1                       # at another rate the host path runs vfx_resample per batch
    for mode in (0, 1):
        batches = len(plan_many(lengths, mode, lambda L: 2))
        torch.cuda.synchronize()
        n0 = eng.launch_count()
        vf.restore_many(host, mode=mode, sample_rate=rate)
        n1 = eng.launch_count()
        vf.restore_many(wavs, mode=mode, sample_rate=rate)
        n2 = eng.launch_count()
        assert (n2 - n1) - (n1 - n0) == extra * batches, f"mode {mode}: {batches} batches"
    batches = len(_pack(lengths, lambda L: 2))
    n0 = eng.launch_count()
    vf._vocoder.oracle_many(host, sample_rate=rate)
    n1 = eng.launch_count()
    vf._vocoder.oracle_many(wavs, sample_rate=rate)
    n2 = eng.launch_count()
    assert (n2 - n1) - (n1 - n0) == extra * batches
    torch.cuda.synchronize()


# ============================================================================ 6. a side stream
def test_work_on_a_side_stream(vf_for):
    vf = vf_for("tf32")
    wavs = [_wav(int(s * 48000), 50 + k).to(DEV) for k, s in enumerate((40.0, 2.5))]
    want = vf.restore_many([w.cpu().numpy() for w in wavs], mode=1, sample_rate=48000)
    want_o = vf._vocoder.oracle_many([w.cpu().numpy() for w in wavs], sample_rate=48000)
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = vf.restore_many(wavs, mode=1, sample_rate=48000)
        got_o = vf._vocoder.oracle_many(wavs, sample_rate=48000)
    s.synchronize()
    for g, w in zip(got + got_o, want + want_o):
        assert _same_bits(g, w)


# ============================================================================ 6b. the engine's shared buffers
def test_buffers_replaced_on_a_side_stream_are_not_reused_early(weights, monkeypatch):
    """A fresh engine sizes its workspace and uploads the 48 kHz taps on the default stream.  A call on a side stream,
    queued behind a kernel that spins for about two seconds, then outgrows that workspace and brings a new ratio, so both
    buffers are replaced while the side stream has not yet run the launches that read them.  Blocks of their sizes
    allocated on the default stream right after must be other memory, and the results must equal the host call's."""
    eng = Engine(weights[0], weights[1], precision="tf32")
    vf = VoiceFixer.from_engine(eng)
    vf.restore_many([_wav(2 * 48000, 70).to(DEV)], sample_rate=48000)         # small workspace, 48 kHz taps
    torch.cuda.synchronize()
    old = [(eng._ws.data_ptr(), eng._ws.numel()), (eng._taps_dev.data_ptr(), 4 * eng._taps_dev.numel())]
    monkeypatch.setattr(eng, "_fit", lambda per_item, cap, reserve: 1)    # one segment per batch: 48 kHz, then 16 kHz
    wavs = [_wav(30 * 48000, 71).to(DEV), _wav(12 * 16000, 72).to(DEV)]
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(4 * 10 ** 9)                                      # ~2 s at 1.98 GHz
        got = vf.restore_many(wavs, sample_rate=[48000, 16000])
    pending = not s.query()
    fresh = [torch.empty(n, dtype=torch.uint8, device=DEV) for _, n in old]
    for (p, n), t in zip(old, fresh):
        assert t.data_ptr() + t.numel() <= p or p + n <= t.data_ptr(), "a replaced buffer was handed out early"
        t.fill_(0xFF)                                                       # NaN bits, on memory nobody else reads
    s.synchronize()
    assert pending, "the side stream finished before the check: the test saw nothing"
    assert old[0][0] != eng._ws.data_ptr() and old[1][0] != eng._taps_dev.data_ptr(), "nothing was replaced"
    want = vf.restore_many([w.cpu().numpy() for w in wavs], sample_rate=[48000, 16000])
    for g, w in zip(got, want):
        assert _same_bits(g, w)


def test_calls_on_two_streams_run_in_call_order(vf_for):
    """One engine, two streams, calls issued back to back: the second call's stream waits for the first's on the
    device (the spin kernel queued first on s1 keeps s2 busy too), and both results equal the host calls'."""
    vf = vf_for("tf32")
    a = [_wav(int(s * 16000), 80 + k).to(DEV) for k, s in enumerate((33.0, 5.0))]
    b = [_wav(int(s * SR), 90 + k).to(DEV) for k, s in enumerate((8.0, 41.0))]
    s1, s2 = torch.cuda.Stream(device=DEV), torch.cuda.Stream(device=DEV)
    for st in (s1, s2):
        st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        torch.cuda._sleep(4 * 10 ** 9)
        got_a = vf.restore_many(a, mode=1, sample_rate=16000)
    with torch.cuda.stream(s2):
        got_b = vf._vocoder.oracle_many(b)
    ordered = not s2.query()
    s1.synchronize()
    s2.synchronize()
    assert ordered, "the second call did not wait for the first"
    for g, w in zip(got_a, vf.restore_many([w.cpu().numpy() for w in a], mode=1, sample_rate=16000)):
        assert _same_bits(g, w)
    for g, w in zip(got_b, vf._vocoder.oracle_many([w.cpu().numpy() for w in b])):
        assert _same_bits(g, w)


def test_one_shot_iterables_are_taken_like_lists(vf_for):
    vf = vf_for("tf32")
    host = [_wav(int(s * SR), 100 + k).numpy() for k, s in enumerate((3.0, 6.5))]
    for call in (vf.restore_many, vf._vocoder.oracle_many):
        want = call(host)
        for g, w in zip(call(iter(host)), want):
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32))
        for g, w in zip(call(torch.from_numpy(h).to(DEV) for h in host), want):
            assert _same_bits(g, w)


# ============================================================================ 7 + 8. the library entries
def _src_table(rows, h_info):
    """rows: [(src, rate, y_first, y_len)] -> ctypes table of vfx_resample_src_item; h_info: {(up, down): (off, len)}."""
    table = (_lib.ResampleSrcItem * len(rows))()
    for b, (src, rate, y_first, y_len) in enumerate(rows):
        up, down = resample.ratio(rate)
        t = table[b]
        t.src, t.stride, t.n_in, t.y_first, t.y_len = src.data_ptr(), src.stride(0), src.shape[0], y_first, y_len
        t.up, t.down, t.rem = up, down, resample.taps(rate)[1]
        t.h_off, t.h_len = h_info.get((up, down), (0, 0))
    return table


@pytest.mark.parametrize("fields,match", [
    (dict(src=None), "item 1: src is null"),
    (dict(stride=0), "item 1: stride 0"),
    (dict(up=0), "item 1: ratio"),
    (dict(h_off=10 ** 6), "item 1: taps"),
    (dict(y_len=SR + 1), "item 1: y_len"),
    (dict(y_first=10 ** 7), "item 1: outputs"),
])
def test_resample_src_refuses_a_bad_item_and_writes_nothing(vf_for, fields, match):
    eng = vf_for("tf32")._engine
    x = _wav(40000, 3).to(DEV)
    h = torch.from_numpy(resample.taps(16000)[0].copy()).to(DEV)
    table = _src_table([(x, 16000, 0, 1000), (x[::2], 16000, 100, 2000)], {resample.ratio(16000): (0, h.numel())})
    for f, v in fields.items():
        setattr(table[1], f, v)
    y = torch.full((2, SR), -1920.0, device=DEV)
    lens = torch.full((2,), -5, dtype=torch.int32, device=DEV)
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    rc = eng.lib.vfx_resample_src(eng.h, _ptr(h), h.numel(), table, 2, _ptr(y), SR, _ptr(lens), _ptr(ws), 4096,
                                  _stream())
    torch.cuda.synchronize()
    assert rc == -1 and match.encode() in eng.lib.vfx_last_error(), eng.lib.vfx_last_error()
    assert eng.launch_count() == n0
    assert bool((y == -1920.0).all()) and bool((lens == -5).all()), "a refused call wrote its output"


@pytest.mark.parametrize("case,match", [
    ("null", "item 1: dst is null"),
    ("long", "item 1: len 4097 is not in [0, ldx = 4096]"),
    ("outside", "item 1: destination [9000, 10100) is not inside its 10000 elements"),
    ("overlap", "item 1: its destination overlaps item 0's"),
])
def test_scatter_rows_refuses_a_bad_item_and_writes_nothing(vf_for, case, match):
    eng = vf_for("tf32")._engine
    x = torch.randn(2, 4096, device=DEV)
    dst = torch.full((10000,), -1920.0, device=DEV)
    items = [(dst, 0, 1000), (dst, 5000, 1100)]
    table = (_lib.ScatterItem * 2)()
    for b, (d, off, n) in enumerate(items):
        table[b].dst, table[b].dst_elems, table[b].dst_off, table[b].len = d.data_ptr(), d.numel(), off, n
    if case == "null":
        table[1].dst = None
    elif case == "long":
        table[1].len = 4097
    elif case == "outside":
        table[1].dst_off = 9000
    else:
        table[1].dst_off = 999
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    rc = eng.lib.vfx_scatter_rows(_ptr(x), 2, 4096, table, _ptr(ws), 4096, _stream())
    torch.cuda.synchronize()
    assert rc == -1 and match.encode() in eng.lib.vfx_last_error(), eng.lib.vfx_last_error()
    assert eng.launch_count() == n0
    assert bool((dst == -1920.0).all()), "a refused call wrote its output"


def test_resample_src_matches_indexing_and_the_staged_resampler_on_random_tables(vf_for):
    eng = vf_for("tf32")._engine
    rng = np.random.default_rng(5)
    base = torch.randn(3, 300000, device=DEV)
    rows, copies = [], []
    for b in range(40):
        rate = int(rng.choice([SR, SR, 16000, 48000, 22050, 96000]))
        stride = int(rng.integers(1, 4))
        n = int(rng.integers(1, 300000 // stride))
        src = base[int(rng.integers(0, 3)), ::stride][:n]
        n_out = resample.out_len(n, rate)
        y_first = int(rng.integers(0, n_out))
        y_len = int(rng.integers(0, min(n_out - y_first, 20000) + 1))
        rows.append((src, rate, y_first, y_len))
    L_cap = 20003
    y, lens = eng.resample_src(rows, L_cap)
    # copies (44.1 kHz) against torch indexing; other rates against vfx_resample on staged windows
    staged = [(k, r) for k, r in enumerate(rows) if r[1] != SR]
    items = [r[0].cpu().numpy() for _, r in staged]
    x, table = _stage(items, [r[1] for _, r in staged], [(j, r[2], r[2] + r[3]) for j, (_, r) in enumerate(staged)], DEV)
    want, _ = eng.resample(x, table, L_cap)
    torch.cuda.synchronize()
    assert lens.tolist() == [r[3] for r in rows]
    for b, (src, rate, y_first, y_len) in enumerate(rows):
        assert bool((y[b, y_len:] == 0).all()), f"row {b}: tail"
        if rate == SR:
            assert torch.equal(y[b, :y_len], src[y_first:y_first + y_len]), f"row {b}"
    for j, (b, (_, _, _, y_len)) in enumerate(staged):
        assert torch.equal(y[b].view(torch.int32), want[j].view(torch.int32)), f"row {b} ({rows[b][1]} Hz)"


def test_scatter_rows_matches_indexing_on_random_tables(vf_for):
    eng = vf_for("tf32")._engine
    rng = np.random.default_rng(6)
    B, ldx = 37, 5000
    x = torch.randn(B, ldx, device=DEV)
    dsts = [torch.full((int(rng.integers(5000, 40000)),), float("nan"), device=DEV) for _ in range(5)]
    want = [d.clone() for d in dsts]
    free = {k: 0 for k in range(len(dsts))}                  # next free offset per destination: ranges never overlap
    items = []
    for b in range(B):
        k = int(rng.integers(0, len(dsts)))
        n = int(rng.integers(0, ldx + 1))
        off = free[k] + int(rng.integers(0, 50))
        if off + n > dsts[k].numel():
            n, off = 0, 0
        else:
            free[k] = off + n
        items.append((dsts[k], off, n))
        want[k][off:off + n] = x[b, :n]
    eng.scatter_rows(x, items)
    torch.cuda.synchronize()
    for d, w in zip(dsts, want):
        assert torch.equal(d.view(torch.int32), w.view(torch.int32))


# ============================================================================ 9. refusals before any launch
def test_bad_lists_raise_before_any_launch(vf_for):
    vf = vf_for("tf32")
    eng = vf._engine
    good = _wav(3 * SR, 1).to(DEV)
    cases = [([good, good.cpu().numpy()], "recording 1 is not a CUDA tensor but recording 0 is"),
             ([good, good.double()], "recording 1 has dtype torch.float64"),
             ([good, good.half()], "recording 1 has dtype torch.float16"),
             ([good[None], good], r"recording 0 has shape \(1, 132300\)"),
             ([good, torch.zeros(SR, 2, device=DEV)], r"recording 1 has shape \(44100, 2\)"),
             ([good, good[:1].expand(3 * SR)], "recording 1 has element stride 0")]
    if torch.cuda.device_count() > 1:
        cases.append(([good, good.to("cuda:1")], "recording 1 is on cuda:1"))
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    for items, match in cases:
        with pytest.raises(ValueError, match="restore_many: " + match):
            vf.restore_many(items)
        with pytest.raises(ValueError, match="oracle_many: " + match):
            vf._vocoder.oracle_many(items)
    with pytest.raises(ValueError, match="restore_many: recording 0"):     # plan_many's own checks still apply
        vf.restore_many([good[:1024], good])
    with pytest.raises(ValueError, match="oracle_many: item 1 is empty"):
        vf._vocoder.oracle_many([good, good[:0]])
    assert eng.launch_count() == n0
