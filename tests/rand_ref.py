"""NumPy restatement of the random-number contract (DESIGN.md section 3), in uint64 arithmetic.

Philox4x32-10 over arrays of counters; the RAND / RAND_INTEGER values of rows; the TABLESAMPLE BERNOULLI mask
and the SYSTEM choice.  Written from the contract alone, independently of dask-sql_b200/rand.py.
"""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)


def philox(c0, c1, c2, c3, key):
    """Words (w0, w1, w2, w3) of Philox4x32-10 for arrays of counter words (any int dtype, broadcast) under the
    64-bit key (a python int, negative = two's complement)."""
    c = [np.asarray(x).astype(np.uint64) & M32 for x in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c0, c1, c2, c3 = (x.copy() for x in c)
    k = int(key) & ((1 << 64) - 1)
    k0, k1 = np.uint64(k & 0xFFFFFFFF), np.uint64(k >> 32)
    for i in range(10):
        if i:
            k0 = (k0 + np.uint64(0x9E3779B9)) & M32
            k1 = (k1 + np.uint64(0xBB67AE85)) & M32
        p0 = np.uint64(0xD2511F53) * c0            # < 2^64: both factors are 32-bit
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & M32, p1 & M32, \
                         ((p0 >> np.uint64(32)) ^ c3 ^ k1) & M32, p0 & M32
    return c0, c1, c2, c3


def _rows(rows):
    r = np.asarray(rows, dtype=np.int64).astype(np.uint64)
    return r & M32, r >> np.uint64(32)


def rand_u64(rows, key, site):
    lo, hi = _rows(rows)
    w0, w1, _, _ = philox(lo, hi, site, 0, key)
    return w0 | (w1 << np.uint64(32))


def rand(rows, key, site):
    """RAND: (u >> 11) * 2^-53 as float64."""
    return (rand_u64(rows, key, site) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def mulhi64(a, b):
    """High 64 bits of the 128-bit product of uint64 arrays a and b."""
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    lo32 = np.uint64(0xFFFFFFFF)
    s32 = np.uint64(32)
    a0, a1, b0, b1 = a & lo32, a >> s32, b & lo32, b >> s32
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> s32) + (p01 & lo32) + (p10 & lo32)
    return p11 + (p01 >> s32) + (p10 >> s32) + (mid >> s32)


def rand_integer(rows, key, site, h):
    """RAND_INTEGER: (u * h) >> 64 as int64, h > 0."""
    return mulhi64(rand_u64(rows, key, site), np.uint64(h)).astype(np.int64)


def threshold(p):
    return int(round(float(p) / 100.0 * 2.0 ** 32))


def bernoulli_mask(rows, key, site, p):
    """TABLESAMPLE BERNOULLI (p): keep row r iff word r & 3 of Philox((r >> 2) lo, hi, site, 1) < T."""
    t = threshold(p)
    r = np.asarray(rows, dtype=np.int64)
    if t <= 0:
        return np.zeros(r.shape, dtype=bool)
    if t >= 1 << 32:
        return np.ones(r.shape, dtype=bool)
    g = (r >> 2).astype(np.uint64)
    w = np.stack(philox(g & M32, g >> np.uint64(32), site, 1, key))
    return w[r & 3, np.arange(r.size).reshape(r.shape)] < np.uint64(t)


def system_keep(nparts, key, site, p):
    """TABLESAMPLE SYSTEM (p): which of nparts partitions (in table order) are kept."""
    t = threshold(p)
    if t >= 1 << 32:
        return np.ones(nparts, dtype=bool)
    w0 = philox(np.arange(nparts), 0, site, 2, key)[0]
    return w0 < np.uint64(t)


def key_of(seed):
    k = int(seed) & ((1 << 64) - 1)
    return k - (1 << 64) if k >> 63 else k
