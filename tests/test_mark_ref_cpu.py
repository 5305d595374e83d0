"""tests/mark_ref.py against stdlib sqlite3 running the same subquery predicates on seeded tables with NULLs on
both sides: IN, NOT IN, EXISTS, NOT EXISTS, correlated and uncorrelated, with pair terms, and an empty inner
side.  NOT is the three-valued NOT of the mark.  A pair term of the subquery's WHERE rejects a candidate when
it is NULL; only the IN's own `x = y` term is three-valued."""
import sqlite3

import numpy as np
import pytest

from tests import mark_ref as M


def _table(rng, n, nulls, hi=6):
    cols = {}
    for name in ("a", "b", "c"):
        v = rng.integers(0, hi, n).astype(np.int64)
        ok = rng.random(n) >= nulls
        cols[name] = (v, ok)
    return cols


def _rows(t):
    n = len(t["a"][0])
    return [tuple(int(t[c][0][i]) if t[c][1][i] else None for c in ("a", "b", "c")) for i in range(n)]


def _db(outer, inner):
    db = sqlite3.connect(":memory:")
    db.execute("CREATE TABLE o (a INTEGER, b INTEGER, c INTEGER)")
    db.execute("CREATE TABLE i (a INTEGER, b INTEGER, c INTEGER)")
    db.executemany("INSERT INTO o VALUES (?, ?, ?)", _rows(outer))
    db.executemany("INSERT INTO i VALUES (?, ?, ?)", _rows(inner))
    return db


def _sqlite(db, pred):
    rows = db.execute(f"SELECT ({pred}) FROM o ORDER BY rowid").fetchall()
    return [None if r[0] is None else bool(r[0]) for r in rows]


def _not(v):
    return [None if x is None else not x for x in v]


def _is_true(v):
    return [x is True for x in v]


CASES = [
    # (sqlite predicate over o, probe keys, build keys, pair terms, null_aware, exists)
    ("o.a IN (SELECT i.a FROM i)", ["a"], ["a"], [], True, False),
    ("o.a IN (SELECT i.b FROM i WHERE i.c > 2)", ["a"], ["b"], [], True, False),
    ("EXISTS (SELECT 1 FROM i WHERE i.a = o.a)", ["a"], ["a"], [], False, True),
    ("EXISTS (SELECT 1 FROM i WHERE i.a = o.a AND i.b < o.b)", ["a"], ["a"], [("b", "b", ">", True)], False, True),
    ("EXISTS (SELECT 1 FROM i WHERE i.a = o.a AND i.b <> o.b AND o.c >= i.c)", ["a"], ["a"],
     [("b", "b", "!=", True), ("c", "c", ">=", True)], False, True),
    ("o.c IN (SELECT i.c FROM i WHERE i.a = o.a)", ["a"], ["a"], [("c", "c", "=")], False, False),
    ("o.c IN (SELECT i.c FROM i WHERE i.a = o.a AND i.b = o.b)", ["a", "b"], ["a", "b"], [("c", "c", "=")],
     False, False),
    ("o.b IN (SELECT i.b FROM i WHERE i.a = o.a AND i.c <= o.c)", ["a"], ["a"], [("b", "b", "="), ("c", "c", ">=", True)],
     False, False),
]


def _ref(outer, inner, keep, pk, bk, terms, null_aware, exists):
    inner = {k: (v[keep], ok[keep]) for k, (v, ok) in inner.items()}
    out, valid = M.mark([outer[k] for k in pk], [inner[k] for k in bk],
                        [(outer[t[0]], inner[t[1]]) + tuple(t[2:]) for t in terms], null_aware)
    v = M.sql_value(out, valid)
    return _is_true(v) if exists else v


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("inner_rows", [0, 1, 40])
def test_mark_matches_sqlite(seed, case, inner_rows):
    pred, pk, bk, terms, null_aware, exists = CASES[case]
    rng = np.random.default_rng(seed)
    outer, inner = _table(rng, 60, 0.15), _table(rng, inner_rows, 0.15)
    keep = inner["c"][0] > 2 if "i.c > 2" in pred else np.ones(inner_rows, bool)
    if "i.c > 2" in pred:
        keep &= inner["c"][1]
    db = _db(outer, inner)
    want = _sqlite(db, pred)
    got = _ref(outer, inner, keep, pk, bk, terms, null_aware, exists)
    assert got == want
    assert _not(got) == _sqlite(db, "NOT " + pred)


def test_empty_inner_side_is_false_even_for_null():
    out, valid = M.mark([(np.array([1, 0], np.int64), np.array([True, False]))],
                        [(np.zeros(0, np.int64), None)], null_aware=True)
    assert M.sql_value(out, valid) == [False, False]


def test_float_keys_nan_and_signed_zero():
    p = (np.array([0.0, -0.0, np.nan, 2.0]), None)
    b = (np.array([-0.0, np.nan]), None)
    out, valid = M.mark([p], [b], null_aware=True)
    # NaN is a NULL key: it is never found, and the inner side's NaN makes "not found" NULL
    assert M.sql_value(out, valid) == [True, True, None, None]
    out, valid = M.mark([p], [b])
    assert M.sql_value(out, valid) == [True, True, False, False]


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("negated", [False, True])
def test_correlated_in_on_a_float_column_whose_nulls_are_nan(seed, negated):
    """a NULL float is a NaN without a bitmap: the IN's own x = y term takes it for NULL, as sqlite's NULL"""
    rng = np.random.default_rng(seed)
    n, m = 80, 40

    def floats(k):
        v = rng.integers(0, 4, k).astype(np.float64)
        v[rng.random(k) < 0.2] = np.nan
        return v

    oa, ia = rng.integers(0, 5, n).astype(np.int64), rng.integers(0, 5, m).astype(np.int64)
    of, if_ = floats(n), floats(m)
    db = sqlite3.connect(":memory:")
    db.execute("CREATE TABLE o (a INTEGER, f REAL)")
    db.execute("CREATE TABLE i (a INTEGER, f REAL)")
    db.executemany("INSERT INTO o VALUES (?, ?)", [(int(a), None if np.isnan(f) else float(f)) for a, f in zip(oa, of)])
    db.executemany("INSERT INTO i VALUES (?, ?)", [(int(a), None if np.isnan(f) else float(f)) for a, f in zip(ia, if_)])
    pred = f"o.f {'NOT ' if negated else ''}IN (SELECT i.f FROM i WHERE i.a = o.a)"
    out, valid = M.mark([(oa, None)], [(ia, None)], [((of, None), (if_, None), "=")])
    got = M.sql_value(out, valid)
    assert (_not(got) if negated else got) == _sqlite(db, pred)
