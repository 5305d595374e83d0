"""The query reference of tests/query_ref.py against sqlite3 and hand-computed answers, and its comparator
against corrupted results: each corruption of a correct answer must be caught.  CPU only."""
import math
import sqlite3

import numpy as np
import pandas as pd
import pytest

from tests import query_ref as Q

I64_MAX, I64_MIN = 2 ** 63 - 1, -(2 ** 63)


def _frame(seed=0, n=400):
    rng = np.random.default_rng(seed)
    k = pd.array(np.where(rng.random(n) < 0.1, None, rng.integers(-3, 4, n)), dtype="Int64")
    j = pd.array(np.where(rng.random(n) < 0.1, None, rng.integers(0, 3, n)), dtype="Int64")
    x = pd.array(np.where(rng.random(n) < 0.1, None, rng.integers(-10 ** 6, 10 ** 6, n)), dtype="Int64")
    f = rng.integers(-64, 64, n) * 0.25                     # dyadic: sqlite's sums are exact too
    f[rng.random(n) < 0.1] = np.nan
    s = np.where(rng.random(n) < 0.1, None, rng.choice(["a", "b", "ab", "B", "é"], n)).astype(object)
    return pd.DataFrame({"k": k, "j": j, "x": x, "f": f, "s": s, "i": np.arange(n)})


def _sqlite(sql, **frames):
    con = sqlite3.connect(":memory:")
    for name, df in frames.items():
        d = df.astype(object).where(df.notna(), None)
        d.to_sql(name, con, index=False)
    cur = con.execute(sql)
    names = [c[0] for c in cur.description]
    out = {n: [] for n in names}
    for row in cur.fetchall():
        for n, v in zip(names, row):
            out[n].append(v)
    return out


def _floats(got, *names):
    for n in names:
        got[n] = [math.nan if v is None else float(v) for v in got[n]]
    return got


def test_groupby_matches_sqlite():
    df = _frame()
    rel = Q.table(df)
    exp = Q.aggregate(rel, ["k"], [("n", "count_star"), ("nx", "count", "x"), ("sx", "sum", "x"),
                                   ("lo", "min", "x"), ("hi", "max", "f"), ("sf", "sum", "f"), ("af", "avg", "f")],
                      mask=Q.cmp(rel["i"], ">=", 7))
    assert exp.kinds["sf"] == "float" and exp.kinds["af"] == "float"     # dyadic: determined to the bit
    got = _sqlite("SELECT k, COUNT(*) AS n, COUNT(x) AS nx, SUM(x) AS sx, MIN(x) AS lo, MAX(f) AS hi, "
                  "SUM(f) AS sf, AVG(f) AS af FROM t WHERE i >= 7 GROUP BY k", t=df)
    Q.assert_result(_floats(got, "hi", "sf", "af"), exp)


def test_two_keys_and_varchar_key_match_sqlite():
    df = _frame(1)
    rel = Q.table(df)
    exp = Q.aggregate(rel, ["s", "j"], [("n", "count_star"), ("sx", "sum", "x"), ("d", "count_distinct", "k")])
    got = _sqlite("SELECT s, j, COUNT(*) AS n, SUM(x) AS sx, COUNT(DISTINCT k) AS d FROM t GROUP BY s, j", t=df)
    Q.assert_result(got, exp)


@pytest.mark.parametrize("how", ["inner", "left", "right", "full"])
def test_joins_match_sqlite(how):
    a = _frame(2, 60).rename(columns=lambda c: "a" + c)
    b = _frame(3, 50).rename(columns=lambda c: "b" + c)
    rel = Q.join(Q.table(a), Q.table(b), ["ak", "as"], ["bk", "bs"], how)
    exp = Q.select(rel, ["ai", "bi", "ax", "bf"])
    got = _sqlite(f"SELECT ai, bi, ax, bf FROM a {how.upper()} JOIN b ON ak = bk AND \"as\" = bs", a=a, b=b)
    Q.assert_result(_floats(got, "bf"), exp)


def test_semi_and_anti_join_partition_the_left_rows():
    a, b = _frame(4, 80), _frame(5, 30).rename(columns=lambda c: "b" + c)
    semi = Q.join(Q.table(a), Q.table(b), ["k"], ["bk"], "semi")
    anti = Q.join(Q.table(a), Q.table(b), ["k"], ["bk"], "anti")
    got = _sqlite("SELECT i FROM a WHERE k IN (SELECT bk FROM b WHERE bk IS NOT NULL)", a=a, b=b)
    Q.assert_result(got, Q.select(semi, ["i"]))
    got = _sqlite("SELECT i FROM a WHERE NOT EXISTS (SELECT 1 FROM b WHERE bk = a.k)", a=a, b=b)
    Q.assert_result(got, Q.select(anti, ["i"]))      # a NULL key matches nothing: its row is in ANTI


@pytest.mark.parametrize("order,sql", [
    ([("k", False), ("x", True)], "k NULLS LAST, x DESC NULLS FIRST"),
    ([("k", True, False), ("i", False)], "k DESC NULLS LAST, i"),
    ([("f", False, True), ("i", True)], "f NULLS FIRST, i DESC"),
    ([("s", False), ("i", False)], "s NULLS LAST, i"),
])
@pytest.mark.parametrize("window", [(0, None), (5, 17), (390, 50)])
def test_order_by_limit_offset_match_sqlite(order, sql, window):
    df = _frame(6)
    off, lim = window
    exp = Q.order_by(Q.select(Q.table(df), ["i", "k", "x", "f", "s"]), order, off, lim)
    tail = f" LIMIT {lim if lim is not None else -1} OFFSET {off}"
    got = _sqlite(f"SELECT i, k, x, f, s FROM t ORDER BY {sql}{tail}", t=df)
    Q.assert_result(_floats(got, "f"), exp)
    assert got["i"] == exp.as_got()["i"]            # unique last key: the order itself is determined


# ---- where the engine's semantics are not sqlite's, or sqlite cannot say: hand-computed -------------------------
def test_int64_sum_wraps_and_extreme_keys_group():
    df = pd.DataFrame({"k": [I64_MAX, I64_MAX, I64_MIN, I64_MIN, I64_MAX - 1],
                       "v": [I64_MAX, 2, I64_MIN, -1, 2 ** 53 + 1]})
    exp = Q.aggregate(Q.table(df), ["k"], [("s", "sum", "v"), ("n", "count_star")])
    Q.assert_result({"k": [I64_MAX, I64_MIN, I64_MAX - 1], "s": [I64_MIN + 1, I64_MAX, 2 ** 53 + 1], "n": [2, 2, 1]},
                    exp)


def test_float_keys_signed_zero_nan_and_null_group():
    df = pd.DataFrame({"f": [0.0, -0.0, np.nan, np.inf, -np.inf, -0.0], "g": [1, 2, 3, 4, 5, 6],
                       "v": [-0.0, 0.0, 1.0, 2.0, 3.0, -0.0]})
    exp = Q.aggregate(Q.table(df), ["f"], [("n", "count_star"), ("lo", "min", "v"), ("hi", "max", "v")])
    got = {"f": [0.0, math.nan, math.inf, -math.inf], "n": [3, 1, 1, 1],
           "lo": [-0.0, 1.0, 2.0, 3.0], "hi": [0.0, 1.0, 2.0, 3.0]}
    Q.assert_result(got, exp)
    bad = dict(got, f=[-0.0, math.nan, math.inf, -math.inf])  # the zero group's key is +0.0
    with pytest.raises(AssertionError):
        Q.assert_result(bad, exp)


def test_join_keys_signed_zero_nan_and_mixed_int_float():
    a = pd.DataFrame({"ak": [0.0, np.nan, 2.0 ** 53, 1.5], "ai": [0, 1, 2, 3]})
    b = pd.DataFrame({"bk": [0, 2 ** 53 + 1, 2 ** 53, 7], "bi": [10, 11, 12, 13]})
    a.loc[0, "ak"] = -0.0
    rel = Q.join(Q.table(a), Q.table(b), ["ak"], ["bk"], "inner")
    # -0.0 = 0; 2^53 + 1 rounds to 2^53 in float64 and matches too (DESIGN.md section 6); NaN matches nothing
    Q.assert_result({"ai": [0, 2, 2], "bi": [10, 11, 12]}, Q.select(rel, ["ai", "bi"]))


def test_bit_every_of_an_all_null_group_are_null_and_global_of_no_rows_is_empty():
    df = pd.DataFrame({"k": [1, 1, 2], "x": pd.array([5, 3, None], dtype="Int64"),
                       "b": pd.array([True, False, None], dtype="boolean")})
    exp = Q.aggregate(Q.table(df), ["k"], [("a", "bit_and", "x"), ("o", "bit_or", "x"), ("x1", "bit_xor", "x"),
                                           ("e", "every", "b")])
    Q.assert_result({"k": [1, 2], "a": [1, None], "o": [7, None], "x1": [6, None], "e": [False, None]}, exp)
    # DESIGN.md section 6: a global aggregate over no rows is no row (sqlite: one row of NULL / 0)
    rel = Q.table(df)
    assert Q.aggregate(rel, [], [("n", "count_star"), ("s", "sum", "x")], mask=Q.cmp(rel["k"], ">", 9)).n == 0


def test_variance_is_bounded_against_the_exact_value():
    x = 1e9 + np.array([0.5, 0.25, -0.75, 0.0, 1.0])
    df = pd.DataFrame({"k": [1, 1, 1, 1, 2], "x": x, "y": [1.0, np.nan, 2.0, 3.0, 4.0]})
    exp = Q.aggregate(Q.table(df), ["k"], [("v", "var_samp", "x"), ("p", "var_pop", "x"), ("sd", "stddev_samp", "x"),
                                           ("sxx", "regr_sxx", "y", "x"), ("rc", "regr_count", "y", "x")])
    v = np.var(x[:4] - 1e9, ddof=1)                         # exact: the offsets are dyadic
    sxx = float(np.sum((x[[0, 2, 3]] - np.mean(x[[0, 2, 3]])) ** 2))
    got = {"k": [1, 2], "v": [v, math.nan], "p": [v * 3 / 4, 0.0], "sd": [math.sqrt(v), math.nan],
           "sxx": [sxx, 0.0], "rc": [3, 1]}
    Q.assert_result(got, exp)
    assert exp.cols["v"][0][1] < 1e-6 * v                   # the bound is a bound, not a shrug
    with pytest.raises(AssertionError):
        Q.assert_result(dict(got, v=[v * 3 / 4, math.nan]), exp)     # VAR_POP where VAR_SAMP was asked


# ---- the comparator must fail on each corruption of a correct answer ---------------------------------------------
def _corruption_case():
    rng = np.random.default_rng(9)
    n = 3000
    df = pd.DataFrame({"k": pd.array(np.where(rng.random(n) < 0.05, None, rng.integers(0, 40, n)), dtype="Int64"),
                       "big": rng.integers(2 ** 60, 2 ** 61, n), "z": rng.choice([0.0, -0.0, 1.0], n),
                       "f": rng.random(n) * 1e3 - 500, "x": pd.array(np.where(rng.random(n) < 0.9, None, 1), dtype="Int64")})
    df.loc[df.k == 5, "x"] = None       # a group whose MAX has no input: NULL
    exp = Q.aggregate(Q.table(df), ["k"], [("sb", "sum", "big"), ("lo", "min", "z"), ("sf", "sum", "f"),
                                           ("mx", "max", "x")])
    return exp


def _check_fails(got, exp):
    with pytest.raises(AssertionError):
        Q.assert_result(got, exp)


def test_corruption_low_bit_of_a_large_int64():
    exp = _corruption_case()
    got = exp.as_got()
    Q.assert_result(got, exp)
    i = next(i for i, v in enumerate(got["sb"]) if abs(v) > 2 ** 53)
    got["sb"][i] ^= 1
    assert float(got["sb"][i]) == float(exp.cols["sb"][i])  # invisible once converted to float64
    _check_fails(got, exp)


def test_corruption_min_negative_zero_to_positive_zero():
    exp = _corruption_case()
    got = exp.as_got()
    i = next(i for i, v in enumerate(got["lo"]) if v == 0.0 and math.copysign(1, v) < 0)
    got["lo"][i] = 0.0
    _check_fails(got, exp)


@pytest.mark.parametrize("dup", [False, True])
def test_corruption_group_dropped_or_duplicated(dup):
    exp = _corruption_case()
    got = exp.as_got()
    for k in got:
        got[k] = got[k] + [got[k][3]] if dup else got[k][:3] + got[k][4:]
    _check_fails(got, exp)
    if dup:                            # same row count: one group twice, another missing
        got = exp.as_got()
        for k in got:
            got[k][5] = got[k][3]
        _check_fails(got, exp)


def test_corruption_null_replaced_by_zero():
    exp = _corruption_case()
    got = exp.as_got()
    i = got["mx"].index(None)
    got["mx"][i] = 0
    _check_fails(got, exp)
    got = exp.as_got()                 # and the NULL group's key
    got["k"][got["k"].index(None)] = 0
    _check_fails(got, exp)


def test_corruption_float_sum_just_outside_its_bound():
    exp = _corruption_case()
    assert exp.kinds["sf"] == "bounded"
    e, b = exp.cols["sf"][0]
    assert b > 0
    got = exp.as_got()
    got["sf"][0] = e + b * 0.5         # inside: passes
    Q.assert_result(got, exp)
    g = e + b
    while g - e <= b:                  # the first float past the bound
        g = np.nextafter(g, math.inf)
    got["sf"][0] = float(g)
    _check_fails(got, exp)


def test_corruption_two_rows_of_an_order_by_result_swapped():
    exp = Q.order_by(_corruption_case(), [("sb", True)], 0, 10)
    got = exp.as_got()
    Q.assert_result(got, exp)
    for k in got:
        got[k][2], got[k][3] = got[k][3], got[k][2]
    _check_fails(got, exp)


def test_order_by_ties_may_come_in_any_order():
    df = pd.DataFrame({"a": [1, 1, 1, 2, 2, 3], "b": [0.0, -0.0, 5.0, 1.0, 2.0, np.nan]})
    exp = Q.order_by(Q.select(Q.table(df), ["a", "b"]), [("a", False)])
    got = exp.as_got()
    got["b"][0], got["b"][2] = got["b"][2], got["b"][0]
    Q.assert_result(got, exp)
    exp = Q.order_by(Q.select(Q.table(df), ["a", "b"]), [("b", False)], 0, 2)   # -0.0 ties with 0.0, cut by LIMIT
    Q.assert_result({"a": [1, 1], "b": [-0.0, 0.0]}, exp)
    Q.assert_result({"a": [1, 1], "b": [0.0, -0.0]}, exp)
    _check_fails({"a": [1, 2], "b": [0.0, 1.0]}, exp)


def test_corruption_float_sum_outside_its_bound_in_a_tie_cut_by_limit():
    exp = Q.order_by(_corruption_case(), [("mx", False)], 0, 3)      # MAX is 1 in almost every group: one long tie
    got = exp.as_got()
    Q.assert_result(got, exp)
    e, b = next(c for c, k in zip(exp.cols["sf"], exp.cols["k"]) if k == got["k"][1])
    g = e + b
    while g - e <= b:
        g = np.nextafter(g, math.inf)
    got["sf"][1] = float(g)
    _check_fails(got, exp)
