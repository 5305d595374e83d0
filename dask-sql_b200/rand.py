"""Seeds, keys and sample rules of RAND / RANDOM / RAND_INTEGER and TABLESAMPLE.

Every row of a base table has a number 0 ... N-1, its position in the table as ingested (DESIGN.md section 3).
The device draws Philox4x32-10 with that number as counter and the statement's 64-bit key, so a value belongs
to the row and not to the partition it happens to sit in.  This module holds the host half of that contract:
the seed -> key rule, the BERNOULLI threshold, the SYSTEM choice of partitions, and each partition's first
row number.
"""
import os
from typing import List, Optional, Sequence

_M32 = 0xFFFFFFFF
_M64 = (1 << 64) - 1

# Philox counter word 3: which stream of a call site a draw belongs to
STREAM_VALUE, STREAM_BERNOULLI, STREAM_SYSTEM = 0, 1, 2


def key_of(seed: Optional[int]) -> int:
    """The 64-bit Philox key of an integer seed (two's complement for a negative one), as a signed int64
    (the b2_instr_t.imm_i / b2_sample_mask argument).  None: a key drawn from os.urandom."""
    k = int.from_bytes(os.urandom(8), "little") if seed is None else int(seed) & _M64
    return k - (1 << 64) if k >> 63 else k


def philox4x32_10(ctr: Sequence[int], key: int) -> List[int]:
    """Philox4x32-10 of one counter (four 32-bit words) under a 64-bit key: the host twin of
    csrc/rand.cuh b2_philox4x32_10, for the few draws SYSTEM makes per table."""
    c0, c1, c2, c3 = (int(w) & _M32 for w in ctr)
    k0, k1 = key & _M32, (key >> 32) & _M32
    for i in range(10):
        if i:
            k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _M32, p1 & _M32, ((p0 >> 32) ^ c3 ^ k1) & _M32, p0 & _M32
    return [c0, c1, c2, c3]


def threshold(p: float) -> int:
    """TABLESAMPLE's p (percent, 0 ... 100) as the 32-bit word a draw must stay below: round(p / 100 * 2^32)."""
    return int(round(float(p) / 100.0 * 2.0 ** 32))


def system_keeps(k: int, key: int, site: int, p: float) -> bool:
    """Does TABLESAMPLE SYSTEM (p) keep partition k (counted in table order)?"""
    t = threshold(p)
    if t >= 1 << 32:
        return True
    return philox4x32_10((k, 0, site, STREAM_SYSTEM), key)[0] < t


def row_bases(sizes: Sequence[int], start: int = 0) -> List[int]:
    """First row number of each partition: `start` plus the sizes of the partitions before it."""
    out, r = [], int(start)
    for n in sizes:
        out.append(r)
        r += int(n)
    return out


class Sample:
    """One TABLESAMPLE clause: method "bernoulli" | "system", p in percent, the statement's key and the
    clause's call-site number."""
    __slots__ = ("method", "p", "key", "site")

    def __init__(self, method: str, p: float, key: int, site: int):
        self.method, self.p, self.key, self.site = method, float(p), int(key), int(site)

    def __repr__(self):
        return f"{self.method}({self.p}; key={self.key}, site={self.site})"

    def __eq__(self, o):
        return isinstance(o, Sample) and (self.method, self.p, self.key, self.site) == (o.method, o.p, o.key, o.site)

    def __hash__(self):
        return hash((self.method, self.p, self.key, self.site))
