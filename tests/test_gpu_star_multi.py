"""The probe over several fact partitions in one launch (b2_star_agg_multi) and the 21-bit lookup filled through
an int32 staging array and packed (b2_star_build_fill_narrow at 32 bits + b2_star_build_pack).  The staged
slot words word for word against tests/star_packed_ref.py, with and without a duplicate passing pk; then the
multi-partition probe over that lookup against tests/groupagg_ref.py: uneven partitions, empty ones, sizes on
and off the 4096-row tile, one partition, partitions streamed as 32-bit images next to int64 ones, more
partitions than one launch takes, and enough tiles that some are strided statically and the rest handed out
by the ticket."""
import ctypes as C

import numpy as np
import pytest

from tests import groupagg_ref as G
from tests import rowwise_ref as R
from tests import star_packed_ref as S
from tests.test_gpu_groupagg import (COUNT, DIM_PRED, GRP_MIN, PRED, SUM, AMAX, AMIN, _concat_inputs, _dtypes, _eq,
                                     _full, _np, _ptr, _stream, _L, _dev, State, _aggs, fact_part, scan_of)
from tests.test_gpu_star_packed import _dims, _slot_of

pytestmark = pytest.mark.gpu

SPECS = [(-1, COUNT), (2, SUM), (2, AMIN), (4, AMAX), (3, COUNT), (3, SUM)]
NULL_SLOT = 2 ** 16 + 7            # 21-bit slots
PAD = 0x5A5A5A5A


def _staged_lookup(rng, nparts=2, nd=3001, dup=False):
    """(dir, slot words, flags, dims, passing, pk_min, pk_range, nentries) of a 21-bit lookup built through the
    staging array; dup: the first two rows of dims[0] pass with the same pk"""
    import torch
    L = _L()
    pk_min = -77
    dims = _dims(nparts, nd, rng, pk_min, NULL_SLOT)
    if dup:
        flag, pk = dims[0][0], dims[0][1]
        pk.values[1], flag.values[:2] = pk.values[0], 0
        pk.null[:2] = False
        dims[0][2].values[:2] = GRP_MIN + np.array([5, 9])     # two different slots for the one pk
        dims[0][2].null[:2] = False
    pk_range = 2 * nd * nparts
    nentries = min(nd * nparts, pk_range)
    nwords = -(-nentries // 3)
    dirw = torch.zeros((pk_range + 31) // 32, dtype=torch.int64, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    stage = _full(nentries, PAD, dtype=torch.int32)          # entries past the used ones hold garbage
    slots = _full(nwords + 1, 0x5A5A5A5A5A5A5A5A)            # no zeroing: the pack writes every word
    scans = [scan_of(cols, DIM_PRED) for cols in dims]
    for s in scans:
        L.star_build_mark(C.byref(s), 1, pk_min, pk_range, _ptr(dirw), _ptr(flags), _stream())
    L.star_build_rank(_ptr(dirw), pk_range, _stream())
    for s in scans:
        L.star_build_fill_packed(C.byref(s), 1, 2, pk_min, pk_range, GRP_MIN, NULL_SLOT, _ptr(dirw), _ptr(stage), 32,
                                 _stream())
    L.star_build_pack(_ptr(dirw), pk_range, _ptr(stage), nentries, _ptr(slots), 21, _stream())
    passing = [R.eval_terms(cols, DIM_PRED, nd) for cols in dims]
    return dirw, slots, flags, dims, passing, pk_min, pk_range, nentries


@pytest.mark.parametrize("dup", [False, True])
def test_staged_fill_and_pack(dup):
    rng = np.random.default_rng(11 + dup)
    dirw, slots, flags, dims, passing, pk_min, pk_range, nentries = _staged_lookup(rng, dup=dup)
    assert bool(_np(flags)[0]) == dup
    # the reference without the duplicate's second row: the directory is the same, and so is every entry
    # but the duplicate's, which holds one of its two passing rows' slots (the last store wins)
    ref_passing = [ok.copy() for ok in passing]
    ref_passing[0][1] = not dup and ref_passing[0][1]
    exp_dir, exp_words, exp_dup = S.star_build_packed(dims, ref_passing, 1, 2, pk_min, pk_range, GRP_MIN, NULL_SLOT,
                                                      21, nentries)
    assert not exp_dup
    _eq(_np(dirw), exp_dir, "dir words")
    got = _np(slots).view(np.uint64)
    nwords = -(-nentries // 3)
    assert got[nwords] == np.uint64(0x5A5A5A5A5A5A5A5A), "the word after the slot array was written"
    got = got[:nwords]
    if not dup:
        _eq(got, exp_words, "staged 21-bit slot words")
        return
    d = int(dims[0][1].values[0]) - pk_min
    w = _np(dirw).view(np.uint64)[d >> 5]
    pos = int(w >> np.uint64(32)) + bin(int(w) & 0xFFFFFFFF & ((1 << (d & 31)) - 1)).count("1")
    got_e, exp_e = S.unpack_slots(got, 21, nwords * 3), S.unpack_slots(exp_words, 21, nwords * 3)
    assert got_e[pos] in (5, 9), got_e[pos]
    keep = np.arange(nwords * 3) != pos
    _eq(got_e[keep], exp_e[keep], "staged 21-bit entries")


def _image(dev_col, base):
    """a B2_U32 image of an int64 Dev column (NULL rows 0), kept alive on the Dev"""
    import torch
    L = _L()
    v = dev_col.col.values.astype(np.int64) - np.int64(base)
    assert v.min(initial=0) >= 0 and v.max(initial=0) < 2 ** 32
    v = v.astype(np.uint32)
    if dev_col.col.null is not None:
        v[dev_col.col.null] = 0
    dev_col.image = torch.from_numpy(v.view(np.int32)).to(_dev())
    c = dev_col.struct()
    c.data, c.dtype = (dev_col.image.data_ptr() if v.size else 0), L.U32
    return c


LAYOUTS = {
    "uneven": ([5000, 0, 3 * 4096, 1, 4097, 12_345], ()),
    "one": ([20_011], ()),
    "images": ([7000, 5000, 0, 9001], (0, 3)),
    "over_cap": ([int(x) for x in np.random.default_rng(5).integers(0, 3000, 37)] + [0], (2, 20, 33)),
    "static_and_ticket": ([1_000_003, 0, 700_001, 333_333], (2,)),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_multi_partition_probe(layout):
    import torch
    L = _L()
    sizes, imaged = LAYOUTS[layout]
    rng = np.random.default_rng(len(sizes))
    dirw, slots, flags, dims, passing, pk_min, pk_range, _ = _staged_lookup(rng)
    assert not _np(flags).any()
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir, lk.slot_bits = 2, slots.data_ptr(), pk_min, pk_range, \
        dirw.data_ptr(), 21
    m = {}
    for cols, ok in zip(dims, passing):
        r = np.flatnonzero(ok)
        m.update(G.star_map(cols[1], r, _slot_of(cols[2], r, NULL_SLOT))[0])
    facts = []
    for p, n in enumerate(sizes):
        cols = fact_part(n, rng, pk_min, pk_range)
        if p in imaged:
            cols[1].values[cols[1].values == np.iinfo(np.int64).min] = pk_min     # an image spans 2^32 values
        facts.append(cols)
    nt = -(-len(sizes) // L.STAR_MAX_PARTS)
    for terms, what in [(PRED, "predicate"), ([], "no predicate")]:
        scans = (L.Scan * len(sizes))()
        bases = (C.c_void_p * len(sizes))()
        keep = []
        for p, cols in enumerate(facts):
            s = scan_of(cols, terms)
            if p in imaged:
                b = (C.c_int64 * s.ncols)()
                b[0], b[1] = -3, pk_min - 5
                s.cols[0], s.cols[1] = _image(s.devs[0], b[0]), _image(s.devs[1], b[1])
                bases[p] = C.addressof(b)
                keep.append(b)
            scans[p] = s
            keep.append(s)
        tickets = torch.zeros(nt, dtype=torch.int64, device=_dev())
        st = State(SPECS, _dtypes(facts[0], SPECS), NULL_SLOT + 1, rows=True, present=False)
        rc = L.star_agg_multi(scans, bases, len(sizes), 1, C.byref(lk), _aggs(SPECS), len(SPECS),
                              st.with_out_slot(None), _ptr(tickets), _stream())
        assert rc == 0
        gids = [G.star_slots(cols[1], R.eval_terms(cols, terms, cols[0].n), m) for cols in facts]
        ex = G.aggregate(_concat_inputs(facts, SPECS), [op for _, op in SPECS], np.concatenate(gids), NULL_SLOT + 1)
        st.check(ex, True, f"{layout}, {what}")


@pytest.mark.parametrize("nparts", [1, 5, 100])
def test_c4_shape_over_partitions(nparts):
    """The C4 query through Context.sql() over a fact table of 1, 5 and 100 partitions: one probe launch, or
    (100 > B2_STAR_MAX_PARTS) seven, each with its own ticket, and the 21-bit lookup staged and packed; twice,
    so that the second run rebuilds into the same buffer and re-zeroes the tickets.  The lookup buffer, which a
    'root' dim broadcasts, is sized by the key range, the dim rows and the slot width alone, as every rank
    agrees on, never by this rank's fact partitions."""
    from dask_sql_b200 import Context, executor
    from tests.test_gpu_star_packed import _c4, _check, _expected
    rng = np.random.default_rng(nparts)
    dim, fact = _c4(2 ** 16, rng)
    c = Context()
    c.create_table("fact", fact, npartitions=nparts, persist=True)
    c.create_table("dim", dim, npartitions=2, persist=True)
    q = ("SELECT d.grp, SUM(f.val) AS rev, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
         "WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp")
    exp = _expected(fact, dim)
    for _ in range(2):
        fused = executor.stats["star_fused"]
        _check(c.sql(q).compute(), exp)
        assert executor.stats["star_fused"] == fused + 1
    prep = executor.PreparedStar._live[-1]
    assert prep.multi and prep.tickets.numel() == -(-nparts // 16) and prep.stage_n > 0
    assert prep.lookup.numel() == executor._star_bitmap_words(prep.q.prange, prep.q.dn, 21)[2]


def test_out_slot_needs_one_partition():
    """out_slot is indexed by the row within a partition, so b2_star_agg_multi refuses it over several"""
    import torch
    L = _L()
    rng = np.random.default_rng(3)
    dirw, slots, _, _, _, pk_min, pk_range, _ = _staged_lookup(rng)
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir, lk.slot_bits = 2, slots.data_ptr(), pk_min, pk_range, \
        dirw.data_ptr(), 21
    facts = [fact_part(100, rng, pk_min, pk_range) for _ in range(2)]
    keep = [scan_of(cols, PRED) for cols in facts]
    scans = (L.Scan * 2)(*keep)
    st = State(SPECS, _dtypes(facts[0], SPECS), NULL_SLOT + 1, rows=True, present=False)
    buf = _full(100, 0, dtype=torch.int32)
    tickets = torch.zeros(1, dtype=torch.int64, device=_dev())
    with pytest.raises(L.B200SqlError, match=r"\(-2\).*out_slot"):
        L.star_agg_multi(scans, None, 2, 1, C.byref(lk), _aggs(SPECS), len(SPECS), st.with_out_slot(buf),
                         _ptr(tickets), _stream())
