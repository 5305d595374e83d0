"""BIT_AND / BIT_OR / BIT_XOR / EVERY and REGR_COUNT / REGR_SXX / REGR_SYY without a GPU: the bitwise
accumulators of the group-by reference (tests/groupagg_bits_ref.py) against hand-computed cases, the planner's
typing and errors, the plans the aggregate plugin hands to the executor, and the REGR_* definitions against a
pairwise NumPy computation."""
import numpy as np
import pandas as pd
import pytest

from tests import groupagg_bits_ref as B
from tests import rowwise_ref as R

MIN, MAX = R.INT64_MIN, R.INT64_MAX
AND, OR, XOR = B.AGG_AND, B.AGG_OR, B.AGG_XOR


def col(vals, dtype, null=None):
    dt = {R.I64: np.int64, R.F64: np.float64, R.U8: np.uint8}[dtype]
    return R.Column(np.array(vals, dtype=dt), None if null is None else np.array(null, bool), dtype)


# ---- the reference's bitwise accumulators ------------------------------------------------------------------
def test_and_over_negative_numbers_and_int64_min():
    v = col([-1, -2, MIN, -1, MAX, -6, -3], R.I64)
    ex = B.aggregate([v], [AND], [0, 0, 1, 1, 2, 3, 3], 5)
    # -1 & -2 = -2; INT64_MIN & -1 = INT64_MIN; MAX alone; -6 & -3 = ...11010 & ...11101 = ...11000 = -8
    assert ex.acc[0].tolist() == [-2, MIN, MAX, -8, -1]       # slot 4: no row, keeps all ones
    assert (MIN & MAX) == 0 and B.aggregate([v], [AND], [0, 0, 0, 0, 0, 0, 0], 1).acc[0].tolist() == [0]


def test_xor_parity_and_or_of_booleans():
    v = col([5, 5, 5, 3, 3, MIN, MIN], R.I64)
    ex = B.aggregate([v, v], [XOR, OR], [0, 0, 0, 1, 1, 2, 2], 4)
    assert ex.acc[0].tolist() == [5, 0, 0, 0]                 # odd count keeps the value, even cancels it
    assert ex.acc[1].tolist() == [5, 3, MIN, 0]
    b = col([0, 1, 0, 0, 1, 1], R.U8)
    ex = B.aggregate([b, b, b], [OR, AND, XOR], [0, 0, 1, 1, 2, 2], 4)
    assert ex.acc[0].tolist() == [1, 0, 1, 0]
    assert ex.acc[1].tolist() == [0, 0, 1, -1]                # EVERY: the AND of 0 / 1; untouched: all ones
    assert ex.acc[2].tolist() == [1, 0, 0, 0]


def test_untouched_slots_and_all_null_groups_keep_the_identity():
    v = col([7, 9, 12, 4], R.I64, [False, True, True, False])
    ex = B.aggregate([v, v, v], [AND, OR, XOR], [0, 1, 1, 2], 4)
    assert ex.acc[0].tolist() == [7, -1, 4, -1]               # slot 1: both rows NULL
    assert ex.acc[1].tolist() == [7, 0, 4, 0]
    assert ex.acc[2].tolist() == [7, 0, 4, 0]
    assert ex.cnt[0].tolist() == [1, 0, 1, 0] and ex.rows.tolist() == [1, 2, 1, 0]
    assert [B.initial_word(op, R.I64) for op in (AND, OR, XOR)] == [-1, 0, 0]
    moved = B.permute(ex, [3, 0, 1, 4], 5, inputs=[v, v, v], ops=[AND, OR, XOR])
    assert moved.acc[0].tolist() == [-1, 4, -1, 7, -1] and moved.acc[2].tolist() == [0, 4, 0, 7, 0]


def test_global_words_of_an_empty_input_are_the_identities():
    v = col([], R.I64)
    ex = B.aggregate([v, v, v], [AND, OR, XOR], np.zeros(0, np.int64), 1)
    assert B.global_words(ex, [AND, OR, XOR], [v, v, v]) == ([-1, 0, 0], [0, 0, 0])


# ---- planner typing -----------------------------------------------------------------------------------------
def _ctx():
    from dask_sql_b200 import Context
    c = Context()
    c.create_table("t", pd.DataFrame({"k": [1, 1, 2], "i": [3, 5, 6], "j": pd.array([1, None, 2], dtype="Int32"),
                                      "f": [1.5, 2.5, 3.5], "b": [True, False, True]}))
    return c


def test_planner_types_the_new_aggregates():
    from dask_sql_b200.frame import AggSource
    c = _ctx()
    lf = c.sql("""SELECT k, BIT_AND(i) AS a, BIT_OR(j) AS o, BIT_XOR(i) AS x, EVERY(b) AS e, EVERY(i > 4) AS e2,
                  REGR_COUNT(f, i) AS rc, REGR_SXX(f, i) AS sx, REGR_SYY(f, j) AS sy FROM t GROUP BY k""")
    assert lf.columns == ["k", "a", "o", "x", "e", "e2", "rc", "sx", "sy"]
    plan = c.explain("SELECT BIT_AND(i) AS a, EVERY(b) AS e, REGR_COUNT(f, i) AS rc, REGR_SXX(f, i) AS s FROM t")
    assert "BIT_AND" in plan and "REGR_SXX" in plan
    src = lf.source
    while not isinstance(src, AggSource):
        src = src.child.source
    fns = sorted(f for _, _, f in src.aggs)
    assert fns == ["bit_and", "bit_or", "bit_xor", "count", "every", "every", "regr_sxx", "regr_syy"]
    sch = src.schema
    outs = {f: sch[o] for _, o, f in src.aggs}
    assert outs["every"][1] == "bool" and outs["count"][1] == "int64" and outs["regr_sxx"][1] == "float64"


def test_planner_rejects_wrong_argument_types_by_name():
    from dask_sql_b200.utils import ParsingException
    c = _ctx()
    for q, fn in [("SELECT BIT_AND(f) FROM t", "BIT_AND"), ("SELECT BIT_OR(b) FROM t", "BIT_OR"),
                  ("SELECT BIT_XOR(f) FROM t GROUP BY k", "BIT_XOR"), ("SELECT EVERY(i) FROM t", "EVERY"),
                  ("SELECT EVERY(f) FROM t GROUP BY k", "EVERY"), ("SELECT REGR_SXX(f) FROM t", "REGR_SXX"),
                  ("SELECT REGR_COUNT(f, i, i) FROM t", "REGR_COUNT"), ("SELECT REGR_SYY(f, b) FROM t", "REGR_SYY")]:
        with pytest.raises(ParsingException, match=fn):
            c.sql(q)


def test_regr_inputs_skip_rows_where_the_other_argument_is_null():
    """REGR_SXX(y, x) aggregates x' = CASE WHEN y IS NOT NULL THEN x END, REGR_SYY(y, x) y' likewise, and
    REGR_COUNT(y, x) is COUNT(x')"""
    from dask_sql_b200.frame import AggSource
    c = _ctx()
    lf = c.sql("SELECT k, REGR_COUNT(j, f) AS rc, REGR_SXX(j, f) AS sx, REGR_SYY(j, f) AS sy FROM t GROUP BY k")
    src = lf.source
    while not isinstance(src, AggSource):
        src = src.child.source
    exprs = {f: repr(src.child.exprs[i]) for i, _, f in src.aggs}
    assert "isnull" in exprs["regr_sxx"] and "case" in exprs["regr_sxx"].lower()
    assert exprs["count"] == exprs["regr_sxx"]                 # one shared input: x' (f where j is not NULL)
    assert exprs["regr_syy"] != exprs["regr_sxx"]


def regr_numpy(y, x):
    """pairwise definition: rows where both are non-NULL (NaN = NULL); (count, Sxx, Syy), NULL sums at n = 0"""
    ok = ~(np.isnan(y) | np.isnan(x))
    n = int(ok.sum())
    if n == 0:
        return 0, None, None
    xs, ys = x[ok], y[ok]
    return n, float(((xs - xs.mean()) ** 2).sum()), float(((ys - ys.mean()) ** 2).sum())


def test_regr_shifted_moments_match_the_pairwise_definition():
    """the executor's REGR_SXX finish, max(S2 - S1^2 / n, 0) over x - K with K the midpoint of x's range, against
    the two-pass pairwise sum of squares, on data with a large mean"""
    rng = np.random.default_rng(5)
    x = 1e9 + rng.normal(0, 1, 10_000)
    y = rng.normal(3, 2, 10_000)
    x[rng.random(10_000) < 0.1] = np.nan
    y[rng.random(10_000) < 0.1] = np.nan
    n, sxx, syy = regr_numpy(y, x)
    xp = np.where(np.isnan(y), np.nan, x)
    ok = ~np.isnan(xp)
    k = (np.nanmin(x) + np.nanmax(x)) / 2
    d = xp[ok] - k
    s1, s2 = d.sum(), (d * d).sum()
    assert ok.sum() == n
    assert abs(max(s2 - s1 * s1 / n, 0.0) - sxx) <= 1e-6 * sxx
    assert regr_numpy(np.array([np.nan, 1.0]), np.array([2.0, np.nan])) == (0, None, None)
