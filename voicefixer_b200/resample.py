"""Sample-rate conversion to the model's 44.1 kHz on the device (vfx_resample): the host half, i.e. the filter taps and
the index arithmetic.  Pure functions, no GPU.

The device restates wavio._resample, scipy.signal.resample_poly(x, up, down) on float32 input, bit for bit.  For a
rate r, g = gcd(r, 44100), up = 44100 / g and down = r / g; up == down == 1 is a copy.  Otherwise scipy designs
h = float32(firwin(2 * half + 1, 1 / max(up, down), window=("kaiser", 5.0))) * float32(up), half = 10 * max(up, down),
and prepends pre = down - half % down zeros (h' below).  Output j of the n_out = ceil(n_in * up / down) samples is

    p = (j + rem) * down,  rem = (half + pre) // down
    y[j] = sum over i = max(0, ceil((p - len(h') + 1) / up)) .. min(n_in - 1, floor(p / up)), ascending, of x[i] * h'[p - i * up]

accumulated in float32 from 0, one separate multiply and add per tap (no fused multiply-add), as scipy's upfirdn loop
does for float32.  Samples [a, b) of the output read only the inputs window(n_in, rate, a, b), so a 30 s segment is
resampled from its own stretch of input plus a few dozen samples of halo."""
import numbers
from functools import lru_cache
from math import gcd

import numpy as np

RATE = 44100                       # the rate every model input has (the reference's librosa.load(path, sr=44100))
MAX_RATE = 2 ** 31 - 1             # ratios travel as C ints


def ratio(rate):
    """(up, down): 44100 / rate in lowest terms."""
    g = gcd(int(rate), RATE)
    return RATE // g, int(rate) // g


@lru_cache(maxsize=None)
def _taps(up, down):
    from scipy.signal import firwin
    half = 10 * max(up, down)
    h = np.asarray(firwin(2 * half + 1, 1.0 / max(up, down), window=("kaiser", 5.0)), dtype=np.float32)
    h *= np.float32(up)
    pre = down - half % down
    hp = np.concatenate([np.zeros(pre, np.float32), h])
    hp.setflags(write=False)
    return hp, (half + pre) // down


def taps(rate):
    """(h', rem) of a rate: the pre-padded, scaled float32 taps (read-only; cached per ratio) and the output offset rem.
    A copy (rate 44100) has no taps: (empty array, 0)."""
    up, down = ratio(rate)
    if up == down == 1:
        return np.zeros(0, np.float32), 0
    return _taps(up, down)


def out_len(n_in, rate):
    """Samples at 44.1 kHz of a recording of n_in samples at `rate`: ceil(n_in * up / down)."""
    up, down = ratio(rate)
    return -(-int(n_in) * up // down)


def available(n_in, rate):
    """Samples at 44.1 kHz that the first n_in input samples of a recording still arriving determine: the prefix [0, m)
    whose window(n, rate, 0, m) ends at or before n_in for every n >= n_in, i.e. every output whose last input,
    (j + rem) * down // up, has arrived.  That is out_len(n_in, rate) - rem (at least 0), and n_in for a copy; once the
    recording has ended, all out_len(n_in, rate) samples are determined."""
    up, down = ratio(rate)
    if up == down == 1:
        return int(n_in)
    return max(0, out_len(n_in, rate) - taps(rate)[1])


def window(n_in, rate, a, b):
    """(first, stop): the inputs [first, stop) that output samples [a, b) read, clipped to [0, n_in).  Empty (first ==
    stop) when b <= a or no input contributes."""
    n_in, a, b = int(n_in), int(a), int(b)
    up, down = ratio(rate)
    if b <= a:
        return 0, 0
    if up == down == 1:
        first, last = a, b - 1
    else:
        h, rem = taps(rate)
        num = (a + rem) * down - len(h) + 1
        first = max(0, -(-num // up))
        last = (b - 1 + rem) * down // up
    first, last = max(0, first), min(n_in - 1, last)
    return (first, last + 1) if first <= last else (0, 0)


def rates(sample_rate, n, what):
    """One sample rate per recording from `sample_rate` (one positive int for all n recordings, or a list / tuple /
    array of n of them).  Raises ValueError naming the recording; nothing else is checked or launched first."""
    if isinstance(sample_rate, (list, tuple, np.ndarray)):
        rs = list(np.asarray(sample_rate, dtype=object).reshape(-1)) if isinstance(sample_rate, np.ndarray) else list(sample_rate)
        if len(rs) != n:
            raise ValueError(f"{what}: sample_rate has {len(rs)} entries for {n} recordings; give one rate, or one per recording")
    else:
        rs = [sample_rate] * n
    return [check_rate(r, f"{what}: recording {i}") for i, r in enumerate(rs)]


def check_rate(r, who):
    """r as an int if it is a valid sample rate; else raises ValueError `<who> has sample_rate ...`."""
    if isinstance(r, (bool, np.bool_)) or not isinstance(r, numbers.Integral) or not 0 < r <= MAX_RATE:
        raise ValueError(f"{who} has sample_rate {r!r}; a sample rate is a positive integer number of Hz (at most {MAX_RATE})")
    return int(r)


def staging_bound(L, rate):
    """Upper bound of window(n_in, rate, a, a + L)'s length for any n_in and a: the staging samples one item of L output
    samples needs."""
    up, down = ratio(rate)
    if up == down == 1:
        return int(L)
    return ((int(L) - 1) * down + len(taps(rate)[0])) // up + 3
