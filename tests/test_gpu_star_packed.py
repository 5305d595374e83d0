"""The packed slot array of the ranked-bitmap star lookup (include/b200sql.h, b2_star_build_mark) at 16,
21 and 32 bits: b2_star_build_fill_packed word for word against tests/star_packed_ref.py, then b2_star_agg
probing it (per-row slots and aggregates against the reference), with null_slot at and next to each width's
edge.  Then end-to-end SQL in the C4 shape with group-key ranges that select each width, through a prepared
plan whose lookup buffer holds garbage before its second run, and through the TMA-staged instance."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

from tests import groupagg_ref as G
from tests import rowwise_ref as R
from tests import star_packed_ref as S
from tests.test_gpu_groupagg import (COUNT, DIM_PRED, GRP_MIN, PRED, SUM, AMAX, AMIN, _concat_inputs, _dtypes, _eq,
                                     _full, _np, _ptr, _stream, _L, _dev, State, _aggs, check_out_slots, dim_part,
                                     fact_part, scan_of)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (null_slot, width): at and next to each class edge
EDGES = [(2 ** 16 - 2, 16), (2 ** 16 - 1, 16), (2 ** 16, 21), (2 ** 21 - 1, 21), (2 ** 21, 32), (2 ** 21 + 1, 32)]
SPECS = [(-1, COUNT), (2, SUM), (2, AMIN), (4, AMAX), (3, COUNT)]
PAD = 0x5A5A5A5A5A5A5A5A


def _dims(nparts, nd, rng, pk_min, null_slot):
    """dim_part partitions whose group keys span [GRP_MIN, GRP_MIN + null_slot): both ends present, the
    top of the range frequent (its entries use the highest bits of the width), 5 % NULL (-> null_slot)"""
    dims = []
    for p in range(nparts):
        cols = dim_part(nd, rng, pk_min + 2 * nd * p)
        g = rng.integers(0, null_slot, nd)
        g[rng.random(nd) < 0.3] = null_slot - 1
        g[:2] = 0, null_slot - 1
        cols[2] = R.Column((g + GRP_MIN).astype(np.int64), rng.random(nd) < 0.05, R.I64)
        dims.append(cols)
    return dims


def _slot_of(g: R.Column, rows, null_slot):
    return np.where(g.null_mask()[rows], null_slot, g.values[rows] - GRP_MIN).astype(np.int64)


@pytest.mark.parametrize("nparts", [2, 3])
@pytest.mark.parametrize("null_slot,bits", EDGES)
def test_packed_build_and_probe(null_slot, bits, nparts):
    import torch
    L = _L()
    assert S.slot_bits(null_slot) == bits
    rng = np.random.default_rng(null_slot + nparts)
    pk_min, nd = -77, 3001
    dims = _dims(nparts, nd, rng, pk_min, null_slot)
    pk_range = 2 * nd * nparts
    nentries = min(nd * nparts, pk_range)
    k = 64 // bits
    nwords = -(-nentries // k)
    dirw = torch.zeros((pk_range + 31) // 32, dtype=torch.int64, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    # below 32 bits the caller zeroes the slot words; at 32 bits FILL stores and the padding must survive.
    # One extra word after the array must survive at every width.
    slots = _full(nwords + 1, 0 if bits < 32 else PAD)
    slots[nwords] = PAD
    scans = [scan_of(cols, DIM_PRED) for cols in dims]
    for s in scans:
        L.star_build_mark(C.byref(s), 1, pk_min, pk_range, _ptr(dirw), _ptr(flags), _stream())
    L.star_build_rank(_ptr(dirw), pk_range, _stream())
    for s in scans:
        L.star_build_fill_packed(C.byref(s), 1, 2, pk_min, pk_range, GRP_MIN, null_slot, _ptr(dirw), _ptr(slots),
                                 bits, _stream())
    passing = [R.eval_terms(cols, DIM_PRED, nd) for cols in dims]
    exp_dir, exp_words, dup = S.star_build_packed(dims, passing, 1, 2, pk_min, pk_range, GRP_MIN, null_slot, bits,
                                                  nentries)
    assert not dup and not _np(flags).any()
    _eq(_np(dirw), exp_dir, "dir words")
    got = _np(slots).view(np.uint64)
    assert got[nwords] == np.uint64(PAD), "the word after the slot array was written"
    got = got[:nwords]
    if bits == 32:
        nused = len(G.star_build_bitmap(dims, passing, 1, 2, pk_min, pk_range, GRP_MIN, null_slot)[1])
        exp_words = exp_words.copy()
        pad = np.full(nwords * 2, 0x5A5A5A5A, np.uint32)
        pad[:nused] = exp_words.view(np.uint32)[:nused]
        exp_words = pad.view(np.uint64)
    _eq(got, exp_words, f"slot words ({bits} bits)")

    # b2_star_agg over the packed lookup
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir = 2, slots.data_ptr(), pk_min, pk_range, dirw.data_ptr()
    lk.slot_bits = bits
    m = {}
    for cols, ok in zip(dims, passing):
        r = np.flatnonzero(ok)
        m.update(G.star_map(cols[1], r, _slot_of(cols[2], r, null_slot))[0])
    assert null_slot in m.values() and null_slot - 1 in m.values()
    facts = [fact_part(20_011, rng, pk_min, pk_range) for _ in range(nparts)]
    for terms, what in [(PRED, "predicate"), ([], "no predicate")]:
        st = State(SPECS, _dtypes(facts[0], SPECS), null_slot + 1, rows=True, present=False)
        outs = []
        for cols in facts:
            n = cols[0].n
            buf = _full(n, 0x5A5A5A5A, dtype=torch.int32)
            L.star_agg(C.byref(scan_of(cols, terms)), 1, C.byref(lk), _aggs(SPECS), len(SPECS), st.with_out_slot(buf),
                       _stream())
            outs.append((buf, n))
        gids = [G.star_slots(cols[1], R.eval_terms(cols, terms, cols[0].n), m) for cols in facts]
        ex = G.aggregate(_concat_inputs(facts, SPECS), [op for _, op in SPECS], np.concatenate(gids), null_slot + 1)
        what = f"{bits} bits, null_slot {null_slot}, {what}"
        check_out_slots(outs, gids, what)
        st.check(ex, True, what)


# (null_slot, width, the two group slots of a duplicated pk): below 32 bits a | b > null_slot
DUP_CASES = [(60_000, 16, 32_768, 30_000), (1_000_000, 21, 524_288, 500_000), (2 ** 21 + 5, 32, 2 ** 20, 2 ** 20 - 1)]


@pytest.mark.parametrize("null_slot,bits,a,b", DUP_CASES)
def test_duplicate_passing_pk_keeps_one_valid_slot(null_slot, bits, a, b):
    """Two passing dim rows with one pk share a directory bit and so one slot entry.  The duplicate flag is
    read by the host only after the probe, so the entry must hold one of the two slots -- never a mix of
    them, which could exceed null_slot and send the probe's atomics past the group table."""
    import torch
    L = _L()
    assert a < null_slot and b < null_slot and (bits == 32 or (a | b) > null_slot)
    rng = np.random.default_rng(null_slot)
    pk_min, nd = 11, 2003
    dims = _dims(2, nd, rng, pk_min, null_slot)
    flag, pk, grp = dims[0]
    pkv, pkn = pk.values.copy(), pk.null_mask().copy()
    fl, g, gn = flag.values.copy(), grp.values.copy(), grp.null_mask().copy()
    pkv[1], pkn[:2], fl[:2], gn[:2] = pkv[0], False, 0, False
    g[0], g[1] = GRP_MIN + a, GRP_MIN + b
    dims[0] = [R.Column(fl, None, R.I64), R.Column(pkv, pkn, R.I64), R.Column(g, gn, R.I64)]
    pk_range = 4 * nd
    nwords = -(-min(2 * nd, pk_range) // (64 // bits))
    dirw = torch.zeros((pk_range + 31) // 32, dtype=torch.int64, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    slots = _full(nwords + 1, 0)
    slots[nwords] = PAD
    scans = [scan_of(cols, DIM_PRED) for cols in dims]
    for s in scans:
        L.star_build_mark(C.byref(s), 1, pk_min, pk_range, _ptr(dirw), _ptr(flags), _stream())
    L.star_build_rank(_ptr(dirw), pk_range, _stream())
    for s in scans:
        L.star_build_fill_packed(C.byref(s), 1, 2, pk_min, pk_range, GRP_MIN, null_slot, _ptr(dirw), _ptr(slots),
                                 bits, _stream())
    assert _np(flags)[0] == 1
    words = _np(slots).view(np.uint64)
    assert words[nwords] == np.uint64(PAD)
    dirs = _np(dirw).view(np.uint64)
    nused = int(sum(bin(int(w) & 0xFFFFFFFF).count("1") for w in dirs))
    entries = S.unpack_slots(words[:nwords], bits, nused)
    assert entries.min() >= 0 and entries.max() <= null_slot, entries.max()
    d0 = int(pkv[0]) - pk_min
    w0 = int(dirs[d0 >> 5])
    pos = (w0 >> 32) + bin(w0 & ((1 << (d0 & 31)) - 1)).count("1")
    assert entries[pos] in (a, b), entries[pos]

    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir = 2, slots.data_ptr(), pk_min, pk_range, dirw.data_ptr()
    lk.slot_bits = bits
    cols = fact_part(20_011, rng, pk_min, pk_range)
    fk = cols[1]
    fkv, fkn = fk.values.copy(), fk.null_mask().copy()
    fkv[::7], fkn[::7] = pkv[0], False
    cols[1] = R.Column(fkv, fkn, R.I64)
    n = cols[0].n
    st = State(SPECS, _dtypes(cols, SPECS), null_slot + 1, present=False)
    buf = _full(n, 0x5A5A5A5A, dtype=torch.int32)
    L.star_agg(C.byref(scan_of(cols, [])), 1, C.byref(lk), _aggs(SPECS), len(SPECS), st.with_out_slot(buf), _stream())
    out = _np(buf, n)
    assert out.min() >= -1 and out.max() <= null_slot, out.max()
    assert np.isin(out[::7], [a, b]).all() and out[::7][0] == entries[pos]


def test_star_agg_rejects_other_widths():
    import torch
    from dask_sql_b200._lib import B200SqlError
    L = _L()
    cols = fact_part(10, np.random.default_rng(0), 0, 64)
    words = torch.zeros(8, dtype=torch.int64, device=_dev())
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir = 2, words.data_ptr(), 0, 64, words.data_ptr()
    st = State(SPECS, _dtypes(cols, SPECS), 4)
    for bits in (1, 8, 20, 24, 31, 33, 64, -1):
        lk.slot_bits = bits
        with pytest.raises(B200SqlError, match="slot_bits"):
            L.star_agg(C.byref(scan_of(cols, [])), 1, C.byref(lk), _aggs(SPECS), len(SPECS), st.with_out_slot(None),
                       _stream())


# ---- end to end: C4 shape -----------------------------------------------------------------------------------
def _c4(ng, rng):
    """dim with 300k rows whose group key spans exactly [0, ng) (NULLs too), fact of 1M rows"""
    nd, nf = 300_000, 1_000_000
    pk = rng.permutation(nd).astype(np.int64) * 2 + 5
    grp = rng.integers(0, ng, nd)
    grp[rng.random(nd) < 0.2] = ng - 1
    grp[:2] = 0, ng - 1
    dim = pd.DataFrame({"pk": pk, "flag": rng.integers(0, 10, nd), "grp": pd.array(grp, dtype="Int64")})
    dim.loc[2 + np.flatnonzero(rng.random(nd - 2) < 0.03), "grp"] = pd.NA
    fact = pd.DataFrame({"fk": pk[rng.integers(0, nd, nf)], "x": rng.integers(-2**31, 2**31, nf),
                         "val": rng.random(nf)})
    return dim, fact


def _expected(fact, dim):
    f = fact[fact["x"] > 0]
    d = dim[dim["flag"] < 5]
    j = f.merge(d, left_on="fk", right_on="pk", how="inner")
    return j.groupby("grp", dropna=False).agg(rev=("val", "sum"), n=("val", "size")).reset_index()


def _check(got, exp):
    got = got.sort_values("grp", na_position="last").reset_index(drop=True)
    exp = exp.sort_values("grp", na_position="last").reset_index(drop=True)
    assert len(got) == len(exp), f"{len(got)} groups vs {len(exp)}"
    np.testing.assert_array_equal(got["grp"].to_numpy(dtype=float, na_value=np.nan),
                                  exp["grp"].to_numpy(dtype=float, na_value=np.nan))
    np.testing.assert_array_equal(got["n"].to_numpy(dtype=np.int64), exp["n"].to_numpy(dtype=np.int64))
    np.testing.assert_allclose(got["rev"].to_numpy(dtype=float), exp["rev"].to_numpy(dtype=float), rtol=1e-9)


# group-key range -> null_slot = range (one slot per key, then the NULL slot)
C4_RANGES = [(2 ** 16 - 1, 16), (2 ** 16, 21), (2 ** 21 - 1, 21), (2 ** 21, 32)]


@pytest.mark.parametrize("ng,bits", C4_RANGES)
def test_c4_shape_prepared_twice(ng, bits):
    """Two runs of one prepared plan; before the second, every byte of its lookup buffer is set, so a
    rebuild that does not zero the slot words (FILL ORs into them) or the directory shows up."""
    from dask_sql_b200 import Context, executor
    rng = np.random.default_rng(ng)
    dim, fact = _c4(ng, rng)
    c = Context()
    c.create_table("fact", fact, npartitions=4, persist=True)    # resident columns: the prepared path
    c.create_table("dim", dim, npartitions=3, persist=True)
    q = ("SELECT d.grp, SUM(f.val) AS rev, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
         "WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp")
    exp = _expected(fact, dim)
    before = executor.stats["star_fused"]
    _check(c.sql(q).compute(), exp)
    prep = executor.PreparedStar._live[-1]
    assert prep.slot_bits == bits
    prep.lookup.fill_(-1)
    _check(c.sql(q).compute(), exp)
    assert executor.PreparedStar._live[-1] is prep
    assert executor.stats["star_fused"] == before + 2


@pytest.mark.parametrize("ng,bits", C4_RANGES)
def test_c4_shape_unprepared(ng, bits, monkeypatch):
    """the same query on the per-query path (a plan built for one execution, fresh lookup buffer, then
    dropped) issues the launches of the prepared plan and caches nothing; so does a computed aggregate
    input over the same resident tables"""
    from dask_sql_b200 import Context, executor
    rng = np.random.default_rng(ng + 1)
    dim, fact = _c4(ng, rng)
    c = Context()
    c.create_table("fact", fact, npartitions=4, persist=True)
    c.create_table("dim", dim, npartitions=2, persist=True)
    q = ("SELECT d.grp, SUM(f.val{}) AS rev, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
         "WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp")
    exp = _expected(fact, dim)

    def run(sql):
        live, fused, launches = list(executor.PreparedStar._live), executor.stats["star_fused"], \
            executor.stats["launches"]
        got = c.sql(sql).compute()
        assert executor.stats["star_fused"] == fused + 1
        return got, executor.PreparedStar._live == live, executor.stats["launches"] - launches

    monkeypatch.setenv("B200SQL_NO_PREPARED", "1")
    got, nothing_cached, unprepared = run(q.format(""))
    _check(got, exp)
    assert nothing_cached
    monkeypatch.delenv("B200SQL_NO_PREPARED")
    got, nothing_cached, prepared = run(q.format(""))
    _check(got, exp)
    assert not nothing_cached and prepared == unprepared
    got, nothing_cached, _ = run(q.format(" * 2"))
    _check(got.assign(rev=got["rev"] / 2), exp)
    assert nothing_cached


def test_packed_staged_pipeline():
    """Everything above through the TMA-staged instance of b2_star_agg (B200SQL_PIPELINE=1, read once per
    process): in a child process."""
    if os.environ.get("B200SQL_PIPELINE") == "1":
        pytest.skip("already the staged instance")
    env = dict(os.environ, B200SQL_PIPELINE="1")
    res = subprocess.run(
        [sys.executable, "-m", "pytest", "tests/test_gpu_star_packed.py", "-m", "gpu", "-x", "-q", "-k",
         "not staged_pipeline"],
        cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-2000:]
    assert " passed" in res.stdout
