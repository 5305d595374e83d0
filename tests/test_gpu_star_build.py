"""The build of the ranked-bitmap star lookup (include/b200sql.h, b2_star_build_mark) word for word against
tests/star_packed_ref.py where its parallel structure has edges: the tiled rank at directory sizes around
one, two and three rank tiles and at the C4 range of 10M keys, and the packed fill when every slot word is
written by the rows of one lane's batch (all its entries race for the same words), with and without
duplicate passing keys."""
import ctypes as C

import numpy as np
import pytest

from tests import rowwise_ref as R
from tests import star_packed_ref as S
from tests.test_gpu_groupagg import DIM_PRED, _eq, _full, _np, _ptr, _stream, _L, _dev, scan_of

pytestmark = pytest.mark.gpu

RANK_TILE = 2048                 # directory words per block of the rank (csrc/groupby.cuh, B2_RANK_TILE)
LANE_ROWS, WARP_ROWS = 8, 256    # rows of one lane's batch in the build scan, and of one warp's tile
PAD = 0x5A5A5A5A5A5A5A5A


def _build(dims, pk_min, pk_range, grp_min, null_slot, bits, nentries):
    """mark every partition, rank, fill every partition: (dir words, slot words, flags) as numpy"""
    import torch
    L = _L()
    k = 64 // bits
    nwords = -(-nentries // k)
    dirw = torch.zeros((pk_range + 31) // 32, dtype=torch.int64, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    slots = _full(nwords + 1, 0)
    slots[nwords] = PAD
    scans = [scan_of(cols, DIM_PRED) for cols in dims]
    for s in scans:
        L.star_build_mark(C.byref(s), 1, pk_min, pk_range, _ptr(dirw), _ptr(flags), _stream())
    L.star_build_rank(_ptr(dirw), pk_range, _stream())
    for s in scans:
        L.star_build_fill_packed(C.byref(s), 1, 2, pk_min, pk_range, grp_min, null_slot, _ptr(dirw), _ptr(slots),
                                 bits, _stream())
    words = _np(slots).view(np.uint64)
    assert words[nwords] == np.uint64(PAD), "the word after the slot array was written"
    return _np(dirw), words[:nwords], _np(flags)


def _dim(pk, flag, grp, grp_null=None):
    return [R.Column(flag.astype(np.int64), None, R.I64), R.Column(pk.astype(np.int64), None, R.I64),
            R.Column(grp.astype(np.int64), grp_null, R.I64)]


def _check_against_ref(dims, pk_min, pk_range, grp_min, null_slot, bits):
    nentries = min(sum(d[0].n for d in dims), pk_range)
    dirw, words, flags = _build(dims, pk_min, pk_range, grp_min, null_slot, bits, nentries)
    passing = [R.eval_terms(cols, DIM_PRED, cols[0].n) for cols in dims]
    exp_dir, exp_words, dup = S.star_build_packed(dims, passing, 1, 2, pk_min, pk_range, grp_min, null_slot, bits,
                                                  nentries)
    assert not dup and not flags.any()
    _eq(dirw, exp_dir, f"dir words (pk_range {pk_range})")
    _eq(words, exp_words, f"slot words ({bits} bits, pk_range {pk_range})")


# every directory size around 1, 2 and 3 rank tiles, words partly used at the end or not
RANGES = [1, 31, 32, 33] + [32 * (t * RANK_TILE + dw) - cut for t in (1, 2, 3) for dw in (-1, 0, 1) for cut in (0, 7)]


@pytest.mark.parametrize("pk_range", RANGES)
def test_rank_tiles(pk_range):
    """two partitions whose keys hit every other key of the range, half of the rows passing"""
    rng = np.random.default_rng(pk_range)
    pk_min = -5
    keys = rng.permutation(np.arange(0, pk_range, 2)) + pk_min
    parts = np.array_split(keys, 2) if len(keys) > 1 else [keys]
    dims = []
    for pk in parts:
        n = len(pk)
        g = rng.integers(0, 1000, n)
        dims.append(_dim(pk, rng.integers(0, 10, n), g + 7, rng.random(n) < 0.05))
    _check_against_ref(dims, pk_min, pk_range, 7, 1000, 16)


def test_c4_sized_build():
    """the C4 build: 10M dim rows over a 10M-key range in 3 partitions, 1M groups (21-bit slots)"""
    rng = np.random.default_rng(10)
    nd, ng = 10_000_000, 1_000_000
    pk = rng.permutation(nd)
    flag, grp = rng.integers(0, 10, nd), rng.integers(0, ng, nd)
    dims = [_dim(p, f, g) for p, f, g in zip(np.array_split(pk, 3), np.array_split(flag, 3), np.array_split(grp, 3))]
    assert S.slot_bits(ng) == 21
    _check_against_ref(dims, 0, nd, 0, ng, 21)


# (null_slot, width): the largest slots use the top bits of their entries
WIDTHS = [(2 ** 16 - 1, 16), (2 ** 21 - 1, 21), (2 ** 21 + 5, 32)]


def _contended(bits, warps, rng, pk_min):
    """rows laid out so that lane l of warp tile t holds the live rows j < per of its batch (per = the
    largest multiple of k = 64 / bits in a batch) and their keys are consecutive: the slot words of a lane
    are written by that lane only, every entry of them in the same batch.  Rows j >= per fail the
    predicate.  Returns (pk, flag, key rank of each row or -1)."""
    k = 64 // bits
    per = (LANE_ROWS // k) * k
    r = np.arange(warps * WARP_ROWS)
    t, lane, j = r // WARP_ROWS, r % 32, (r % WARP_ROWS) // 32
    live = j < per
    pos = np.where(live, (t * 32 + lane) * per + j, -1)
    pk = np.where(live, pos, warps * WARP_ROWS + r) + pk_min
    flag = np.where(live, rng.integers(0, 5, len(r)), 9)
    return pk, flag, pos


@pytest.mark.parametrize("null_slot,bits", WIDTHS)
def test_fill_one_lane_per_word(null_slot, bits):
    rng = np.random.default_rng(bits)
    pk_min, warps = 1 << 40, 97
    pk, flag, pos = _contended(bits, warps, rng, pk_min)
    g = rng.integers(0, null_slot, len(pk))
    g[rng.random(len(pk)) < 0.3] = null_slot - 1
    dims = [_dim(pk, flag, g + 3, rng.random(len(pk)) < 0.05)]
    _check_against_ref(dims, pk_min, int(pos.max()) + 1, 3, null_slot, bits)


@pytest.mark.parametrize("null_slot,bits", WIDTHS)
def test_fill_one_lane_per_word_duplicates(null_slot, bits):
    """the contended layout with the second live row of every lane given the key of its first: the pair
    shares one entry, which must hold one of the pair's slots and never a mix of them, while every other
    entry of the same word keeps its own slot"""
    rng = np.random.default_rng(bits + 1)
    pk_min, warps = -(1 << 33), 41
    pk, flag, pos = _contended(bits, warps, rng, pk_min)
    n = len(pk)
    r = np.arange(n)
    first = (pos >= 0) & ((r % WARP_ROWS) // 32 == 0)
    pk[r[first] + 32] = pk[first]                      # row j = 1 of the lane gets the key of row j = 0
    g = rng.integers(0, null_slot, n)
    # the pair's slots have no bit in common: an OR of them is neither
    g[first], g[r[first] + 32] = (null_slot - 1) & 0xAAAAAAAA, (null_slot - 1) & 0x55555555
    dims = [_dim(pk, flag, g)]
    pk_range = int(pos.max()) + 1
    k = 64 // bits
    passing = flag < 5
    keys = np.unique(pk[passing] - pk_min)
    _, words, flags = _build(dims, pk_min, pk_range, 0, null_slot, bits, len(keys))
    assert flags[0] == 1
    entries = S.unpack_slots(words, bits, len(keys))
    assert entries.min() >= 0 and entries.max() <= null_slot, entries.max()
    at = np.searchsorted(keys, pk - pk_min)             # entry of each row's key
    dup = first & passing & passing[np.minimum(r + 32, n - 1)]
    single = passing & ~dup & ~np.isin(r, r[dup] + 32)
    _eq(entries[at[single]], g[single], f"entries of unique keys ({bits} bits)")
    got = entries[at[dup]]
    ok = (got == g[dup]) | (got == g[r[dup] + 32])
    assert ok.all(), f"{(~ok).sum()} duplicated entries hold neither slot, e.g. {got[~ok][:4]}"
    assert len(words) == -(-len(keys) // k)
