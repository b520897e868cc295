"""numpy restatement of the library's dropout masks (include/beatthis.h, "training mode"): Philox4x32-10 and the
keep rule.  Test infrastructure only; the product package does not import it."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """counter: 4 uint32 arrays (broadcastable), key: 2 uint32 scalars or arrays -> 4 uint32 arrays (Salmon et al.,
    Random123; curand_Philox4x32_10)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in counter)
    k0, k1 = (np.asarray(k, dtype=np.uint32) for k in key)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & MASK32).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & MASK32).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0, k1 = k0 + W0, k1 + W1
    return c0, c1, c2, c3


def rate(p: float) -> float:
    """The rate as the library holds it: a float (bt_train_mode's fields)."""
    return float(np.float32(p))


def threshold(p: float) -> int:
    """floor(p 2^32) of the float rate: an element is kept iff its word is at least this."""
    return int(np.floor(rate(p) * 2.0 ** 32))


def scale(p: float) -> float:
    """1 / (1 - p) of the float rate, rounded to float: the factor of kept values."""
    return float(np.float32(1.0 / (1.0 - rate(p))))


def words(seed: int, site: int, e0: int, n: int) -> np.ndarray:
    """The 32-bit words of elements e0 .. e0 + n - 1 of `site` under `seed`: word e mod 4 of
    Philox(counter (lo32(e / 4), hi32(e / 4), site, 0), key (lo32(seed), hi32(seed)))."""
    e = np.arange(e0, e0 + n, dtype=np.uint64)
    g = np.unique(e >> np.uint64(2))
    out = philox4x32_10((g & MASK32, g >> np.uint64(32), np.full(g.shape, site, np.uint64) & MASK32, np.zeros_like(g)),
                        (np.uint32(seed & 0xFFFFFFFF), np.uint32((seed >> 32) & 0xFFFFFFFF)))
    table = np.stack(out, axis=1)  # [groups, 4]
    return table[(e >> np.uint64(2)) - g[0], (e & np.uint64(3)).astype(np.int64)]


def keep(seed: int, site: int, p: float, n: int, e0: int = 0) -> np.ndarray:
    """Boolean keep mask of elements e0 .. e0 + n - 1 (rate 0: all kept)."""
    t = threshold(p)
    if t == 0:
        return np.ones(n, dtype=bool)
    return words(seed, site, e0, n) >= np.uint32(t)
