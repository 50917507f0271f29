"""Host restatement of mode 2's seeded dropout (csrc/philox.cuh, dropout_seeded_kernel; DESIGN.md §3) in numpy.

philox4x32_10 is Philox4x32-10 (Salmon et al., SC'11), the function of curand_Philox4x32_10, vectorised over any
number of counters on uint64 arithmetic.  seeded_masks gives the keep-masks the seeded kernels apply, as an explicit
mask tensor: the reference the kernels are tested against, and a drop_masks_fn / Engine.restore(drop_masks=...) input
that reproduces a seeded call through the explicit-mask path."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(counter, key):
    """counter: (..., 4) integers < 2^32, key: (2,) or (..., 2) -> uint32 (..., 4) output words."""
    c = [w.astype(np.uint64) for w in np.moveaxis(np.asarray(counter, dtype=np.uint64), -1, 0)]
    k0, k1 = (w.astype(np.uint64) for w in np.moveaxis(np.asarray(key, dtype=np.uint64), -1, 0))
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]                 # exact: both factors are below 2^32
        c = [(p1 >> _S32) ^ c[1] ^ k0, p1 & _LO, (p0 >> _S32) ^ c[3] ^ k1, p0 & _LO]
        k0, k1 = (k0 + W0) & _LO, (k1 + W1) & _LO
    return np.stack(c, -1).astype(np.uint32)


def seeded_masks(seed, stream, T):
    """Keep-masks uint8 (2, T, 512) of one item with key (seed, stream), both in [0, 2^64): [l, t, j] is the keep bit of
    unit j of frame t at dropout layer l (0: after dn.lin4, 1: after dn.lin11), i.e. bit j % 32 of word (j % 128) // 32
    of philox4x32_10((t, 4 l + j // 128, stream & 0xffffffff, stream >> 32), (seed & 0xffffffff, seed >> 32))."""
    seed, stream = int(seed), int(stream)
    if not (0 <= seed < 1 << 64 and 0 <= stream < 1 << 64):
        raise ValueError("seed and stream must lie in [0, 2^64)")
    t, g = np.meshgrid(np.arange(int(T), dtype=np.uint64), np.arange(8, dtype=np.uint64), indexing="ij")   # g = 4 l + j // 128
    ctr = np.stack([t, g, np.full_like(t, stream & 0xFFFFFFFF), np.full_like(t, stream >> 32)], -1)
    w = philox4x32_10(ctr, [seed & 0xFFFFFFFF, seed >> 32])                               # (T, 8, 4)
    bits = (w[..., None] >> np.arange(32, dtype=np.uint32)) & 1                           # (T, 8, 4, 32): j % 128 = 32 word + bit
    return bits.reshape(int(T), 2, 512).transpose(1, 0, 2).astype(np.uint8)
