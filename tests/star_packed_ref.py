"""NumPy reference of the packed slot array of the ranked-bitmap star lookup (include/b200sql.h,
b2_star_build_mark): the width rule and the packing of the (dir, slots) that
groupagg_ref.star_build_bitmap returns."""
import numpy as np

from tests import groupagg_ref as G


def slot_bits(null_slot):
    """the narrowest of 16, 21, 32 bits that holds every slot, null_slot being the largest"""
    return 16 if null_slot < (1 << 16) else 21 if null_slot < (1 << 21) else 32


def pack_slots(slots, bits, nentries=None):
    """uint64 words of `slots` packed `bits` wide: k = 64 // bits entries per word, entry i at bit
    (i % k) * bits of word i // k; unused bits and entries are 0.  `nentries` (>= len(slots)) sizes the
    array as the caller allocates it, so that words past the used ones are covered too."""
    k = 64 // bits
    n = len(slots) if nentries is None else nentries
    vals = np.zeros(-(-n // k) * k, np.uint64)
    vals[:len(slots)] = np.asarray(slots, np.int64).astype(np.uint64) & np.uint64((1 << bits) - 1)
    vals = vals.reshape(-1, k)
    shifts = (np.arange(k, dtype=np.uint64) * np.uint64(bits))
    return np.bitwise_or.reduce(vals << shifts, axis=1)


def unpack_slots(words, bits, n):
    """the first n entries of a packed array, as int64"""
    k = 64 // bits
    i = np.arange(n)
    w = np.asarray(words, np.uint64)[i // k]
    return ((w >> ((i % k) * bits).astype(np.uint64)) & np.uint64((1 << bits) - 1)).astype(np.int64)


def star_build_packed(parts, passing, pk_col, grp_col, pk_min, pk_range, grp_min, null_slot, bits, nentries):
    """b2_star_build_mark / rank / fill_packed over all partitions: (dir words, packed slot words,
    duplicate flag)"""
    dirw, slots, dup = G.star_build_bitmap(parts, passing, pk_col, grp_col, pk_min, pk_range, grp_min, null_slot)
    return dirw, pack_slots(slots, bits, nentries), dup
