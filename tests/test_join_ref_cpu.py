"""The join reference of tests/join_ref.py checked on its own (no GPU, no library): row for row against
pandas.merge(sort=False) and Series / MultiIndex.isin on random keys with duplicates, NULLs, NaN, ±0.0 and
1-4 mixed int64 / float64 columns, and by hand at the int64 extremes and the uint32 wrap."""
import math

import numpy as np
import pandas as pd
import pytest

from tests import join_ref as J
from tests.rowwise_ref import F64, I64, INT64_MAX, INT64_MIN, U8, Column

MIN, MAX = INT64_MIN, INT64_MAX


def _keys(dtypes, n, rng, pool):
    """key columns drawn from a small pool (so keys repeat) with NULL bitmaps and NaN / ±0.0 in floats"""
    cols = []
    for dt in dtypes:
        if dt == I64:
            v = rng.choice(np.array([0, 1, -1, 7, MIN, MAX, 2 ** 40], np.int64)[:pool], n)
        else:
            v = rng.choice(np.array([0.0, -0.0, 1.5, -2.0, math.inf, -math.inf, math.nan])[:pool], n)
        cols.append(Column(v, rng.random(n) < 0.1, dt))
    return cols


def _frame(cols, tag):
    df = pd.DataFrame({f"k{i}": c.values for i, c in enumerate(cols)})
    df[tag] = np.arange(cols[0].n)
    return df


def _pandas_join(pcols, bcols, passing, how):
    """(probe rows, build rows) of pandas.merge over the rows with no NULL key, as the reference drops them
    before matching (join.py:202-213); probe rows with a NULL key are added back for a left join"""
    _, pnul = J.key_rows(pcols)
    _, bnul = J.key_rows(bcols)
    left = _frame(pcols, "_l")[passing & ~pnul]
    right = _frame(bcols, "_r")[~bnul]
    keys = [f"k{i}" for i in range(len(pcols))]
    m = pd.merge(left, right, on=keys, how=how, sort=False)
    lr = m["_l"].to_numpy(np.int64)
    rr = m["_r"].fillna(-1).to_numpy(np.int64)
    if how == "left":
        extra = np.flatnonzero(passing & pnul)
        lr, rr = np.concatenate([lr, extra]), np.concatenate([rr, np.full(len(extra), -1)])
        order = np.argsort(lr, kind="stable")
        lr, rr = lr[order], rr[order]
    return lr, rr


def _pandas_isin(pcols, bcols, passing):
    _, pnul = J.key_rows(pcols)
    _, bnul = J.key_rows(bcols)
    keys = [f"k{i}" for i in range(len(pcols))]
    left, right = _frame(pcols, "_l"), _frame(bcols, "_r")[~bnul]
    if len(keys) == 1:
        hit = left["k0"].isin(right["k0"]).to_numpy()
    else:
        hit = pd.MultiIndex.from_frame(left[keys]).isin(pd.MultiIndex.from_frame(right[keys]))
    return np.asarray(hit) & ~pnul


DTYPES = [[I64], [F64], [F64, I64], [I64, F64, F64], [F64, I64, F64, I64]]


@pytest.mark.parametrize("dtypes", DTYPES, ids=lambda d: "".join("if"[t] for t in d))
@pytest.mark.parametrize("seed", range(3))
def test_reference_matches_pandas_merge(dtypes, seed):
    rng = np.random.default_rng(seed * 10 + len(dtypes))
    pool = 3 if len(dtypes) > 2 else 7
    npr, nb = 700, 300
    pcols, bcols = _keys(dtypes, npr, rng, pool), _keys(dtypes, nb, rng, pool)
    passing = rng.random(npr) < 0.8
    m = J.hash_matches(pcols, bcols, passing)
    for mode, how in ((J.JOIN_INNER, "inner"), (J.JOIN_LEFT, "left")):
        e = J.emit(mode, passing, m)
        lr, rr = _pandas_join(pcols, bcols, passing, how)
        np.testing.assert_array_equal(e.probe, lr, err_msg=f"{how}: probe rows")
        np.testing.assert_array_equal(e.build, J.sort_runs(lr, rr), err_msg=f"{how}: build runs")
        np.testing.assert_array_equal(J.build_matched(mode, e, nb), np.isin(np.arange(nb), rr).astype(np.uint8))
    hit = _pandas_isin(pcols, bcols, passing)
    semi, anti = J.emit(J.JOIN_SEMI, passing, m), J.emit(J.JOIN_ANTI, passing, m)
    np.testing.assert_array_equal(semi.probe, np.flatnonzero(passing & hit))
    np.testing.assert_array_equal(anti.probe, np.flatnonzero(passing & ~hit))
    assert (semi.build == -1).all() and (anti.build == -1).all()
    assert not J.build_matched(J.JOIN_SEMI, semi, nb).any()


def test_float_keys_by_hand():
    """-0.0 meets +0.0; NaN of any payload and sign meets nothing; ±inf meet themselves only"""
    nan_bits = np.array([0x7FF8000000000000, 0x7FF0000000000001, -0x0008000000000000, 0x7FFFFFFFFFFFFFFF], np.int64)
    b = np.concatenate([[0.0, math.inf, -math.inf], nan_bits.view(np.float64)])
    p = np.concatenate([[-0.0, 0.0, -math.inf, 1.0], nan_bits.view(np.float64)])
    m = J.hash_matches([Column(p, None, F64)], [Column(b, None, F64)], np.ones(len(p), bool))
    assert m.counts.tolist() == [1, 1, 1, 0, 0, 0, 0, 0]
    assert m.rows.tolist() == [0, 0, 2]


def test_int_keys_by_hand():
    """INT64_MIN is an ordinary int key (only float keys fold the -0.0 pattern); a NULL bit hides the value"""
    b = Column(np.array([MIN, 0, MAX, 5], np.int64), np.array([False, False, False, True]), I64)
    p = Column(np.array([0, MIN, MAX, 5, MIN], np.int64), np.array([False, False, False, False, True]), I64)
    m = J.hash_matches([p], [b], np.ones(5, bool))
    assert m.counts.tolist() == [1, 1, 1, 0, 0] and m.rows.tolist() == [1, 0, 2]
    passing = np.array([True, True, False, True, True])
    e = J.emit(J.JOIN_LEFT, passing, J.hash_matches([p], [b], passing))
    assert e.probe.tolist() == [0, 1, 3, 4] and e.build.tolist() == [1, 0, -1, -1]


def test_dense_offsets_wrap():
    """offsets are uint64 key - kmin: the table of kmin = INT64_MIN reaches INT64_MAX, and a key below a
    table near INT64_MAX wraps past 2^64 into range"""
    key = Column(np.array([MIN, MAX, -1, 0, MIN + 1], np.int64), None, I64)
    d, ok = J.offsets(key, MIN, 1 << 63)
    assert ok.tolist() == [True, False, True, False, True]
    assert d[ok].tolist() == [0, (1 << 63) - 1, 1]
    d, ok = J.offsets(key, MAX - 1, 4)
    assert ok.tolist() == [True, True, False, False, True] and d[ok].tolist() == [2, 1, 3]
    lookup, dup, dups = J.dense_build(Column(np.array([MAX, MAX - 2, MAX, MIN], np.int64), None, I64), MAX - 3, 4)
    assert lookup.tolist() == [-1, 1, -1, -1] and dup == 1 and dups == {3: [0, 2]}


def test_key_layout_uint32_wrap():
    """the U32 word is uint32(v - base) with wrap: v - base = 2^32 - 1, 2^32 (-> 0) and 2^64 - 1"""
    key = Column(np.array([10, 11, 12, 13], np.int64), np.array([False, False, False, True]), I64)
    col = Column(np.array([MIN + (1 << 32) - 1, MIN + (1 << 32), MAX, 7], np.int64), None, I64)
    out, valid, present = J.key_layout(key, 10, 5, col, J.U32, MIN, np.full(5, 0xDEADBEEF, np.uint32),
                                       np.zeros(1, np.uint32), np.zeros(1, np.uint32))
    assert out.tolist() == [0xFFFFFFFF, 0, 0xFFFFFFFF, 0xDEADBEEF, 0xDEADBEEF]
    assert present.tolist() == [0b111] and valid.tolist() == [0b111]
    vals, ok = J.gather_build(Column(out, None, J.U32), [0, 1, -1], base=MIN)
    assert vals.tolist() == [MIN + (1 << 32) - 1, MIN, 0] and ok.tolist() == [True, True, False]


def test_gather_fill_and_tiles():
    f = Column(np.array([-0.0, math.nan]), np.array([False, True]), F64)
    vals, ok = J.gather_build(f, [0, -1, 1])
    assert vals.tolist() == [J.NEG_ZERO_BITS, J.NAN_FILL, np.float64(math.nan).view(np.int64)]
    assert ok.tolist() == [True, False, False]
    vals, ok = J.gather_build(Column(np.array([3], np.uint8), None, U8), [-1, 0])
    assert vals.tolist() == [0, 3] and ok.tolist() == [False, True]
    cnt = np.zeros(4097, np.int64)
    cnt[0], cnt[4095], cnt[4096] = 2, 1, 5
    assert J.tile_off(cnt, 4097).tolist() == [0, 3, 8]
    assert J.tile_off(np.zeros(0, np.int64), 0).tolist() == [0]


def test_check_chains_catches_broken_tables():
    keys = [Column(np.array([1, 2, 1, 9], np.int64), np.array([False, False, False, True]), I64)]
    head, nxt = np.array([2, 1, -1, -1]), np.array([-1, -1, 0, -1])
    assert J.check_chains(head, nxt, keys) is None
    assert "buckets" in J.check_chains(np.array([0, 1, 2, -1]), np.array([-1, -1, -1, -1]), keys)
    assert "linked" in J.check_chains(np.array([2, 1, -1, -1]), np.array([-1, -1, -1, -1]), keys)
    assert "NULL" in J.check_chains(head, np.array([-1, -1, 0, 0]), keys)
    assert "linked" in J.check_chains(np.array([2, 1, 0, -1]), nxt, keys)
    cyc = J.check_chains(np.array([1, -1, -1, -1]), np.array([2, -1, 0, -1]), keys)
    assert cyc is not None
