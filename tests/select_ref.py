"""NumPy restatement of b2_select_hist (one pass of the multi-target MSD radix select) and of the host's walk
to the wanted ranks (executor.order_statistics).  The kernels are checked bin for bin against hist_pass; the
walk is checked here against np.partition, and on the GPU the driver's answers are checked against it too."""
import numpy as np

SIGN = np.uint64(1 << 63)
MAX_BITS = 11


def images(values, valid=None) -> np.ndarray:
    """uint64 order-preserving images of the non-NULL, non-NaN rows of an int64 / float64 array, in row order:
    int64 sign-flipped; float64 as the ordered image (bits ^ ((bits >> 63) & 0x7fff...)) sign-flipped."""
    values = np.asarray(values)
    keep = np.ones(values.shape[0], bool) if valid is None else np.asarray(valid, bool).copy()
    if values.dtype == np.float64:
        keep &= ~np.isnan(values)
        b = values.view(np.int64)
        key = b ^ ((b >> np.int64(63)) & np.int64(0x7FFFFFFFFFFFFFFF))
    else:
        key = values.astype(np.int64)
    return key[keep].view(np.uint64) ^ SIGN


def hist_pass(u: np.ndarray, prefixes, shift: int, bits: int) -> np.ndarray:
    """hist[k * 2^bits + digit] over the images u: digit = (u >> shift) & (2^bits - 1) of the rows with
    u >> (shift + bits) == prefixes[k] (every row when shift + bits == 64).  uint64[len(prefixes) << bits]."""
    hs = shift + bits
    out = np.zeros(len(prefixes) << bits, np.uint64)
    d = ((u >> np.uint64(shift)) & np.uint64((1 << bits) - 1)).astype(np.int64)
    p = np.zeros_like(u) if hs == 64 else u >> np.uint64(hs)
    for k, pk in enumerate(prefixes):
        m = p == np.uint64(pk)
        out[k << bits:(k + 1) << bits] += np.bincount(d[m], minlength=1 << bits).astype(np.uint64)
    return out


def passes(umin: int, umax: int) -> int:
    """passes of the select between these min / max images: ceil(highest differing bit / MAX_BITS)"""
    return -(-(umin ^ umax).bit_length() // MAX_BITS)


def select(u: np.ndarray, ranks, umin=None, umax=None):
    """k -> image of the k-th smallest (0-based) of u, by the same passes and walk as the driver.  Returns
    (answers, number of passes)."""
    targets = sorted({int(k) for k in ranks})
    umin = int(u.min()) if umin is None else umin
    umax = int(u.max()) if umax is None else umax
    level = (umin ^ umax).bit_length()
    if level == 0:
        return {k: umin for k in targets}, 0
    prefix = {k: umin >> level if level < 64 else 0 for k in targets}
    rank = {k: k for k in targets}
    npass = 0
    while level > 0:
        bits = min(MAX_BITS, level)
        shift = level - bits
        groups = sorted(set(prefix.values()))
        h = hist_pass(u, groups, shift, bits).reshape(len(groups), 1 << bits)
        npass += 1
        for k in targets:
            row = h[groups.index(prefix[k])]
            cum = np.cumsum(row.astype(np.int64))
            d = int(np.searchsorted(cum, rank[k], side="right"))
            rank[k] -= int(cum[d] - row[d])
            prefix[k] = (prefix[k] << bits) | d
        level = shift
    return prefix, npass


def value_of(image: int, dtype):
    """images() inverted for one value"""
    key = np.array([image], np.uint64) ^ SIGN
    if np.dtype(dtype) == np.float64:
        k = key.view(np.int64)
        b = k ^ ((k >> np.int64(63)) & np.int64(0x7FFFFFFFFFFFFFFF))
        return b.view(np.float64)[0]
    return key.view(np.int64)[0]
