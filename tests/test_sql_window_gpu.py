"""Window functions end to end on the GPU: Context.sql() against the exact reference of tests/window_ref.py, over
a base table, a partitioned table, a lazy Parquet table, a filter, a join and a GROUP BY output; VARCHAR and DATE
keys and values; several OVER specs in one SELECT; top-N per group through a subquery; ORDER BY / LIMIT on a
window column; and the reference's known answers (tests/golden/reference_window.py)."""
import math

import numpy as np
import pandas as pd
import pytest

from tests import query_ref as Q
from tests import window_ref as W
from tests.golden import reference_window as GW

pytestmark = pytest.mark.gpu
INF = float("inf")

FRAMES = {
    "": None,                  # with ORDER BY: RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW
    "ROWS BETWEEN 2 PRECEDING AND CURRENT ROW": (False, -2, 0),
    "ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING": (False, -2, 3),
    "ROWS BETWEEN 2 PRECEDING AND UNBOUNDED FOLLOWING": (False, -2, INF),
    "ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING": (False, 0, INF),
    "ROWS BETWEEN UNBOUNDED PRECEDING AND 3 FOLLOWING": (False, -INF, 3),
    "ROWS BETWEEN 3 FOLLOWING AND 3 FOLLOWING": (False, 3, 3),
    "ROWS BETWEEN 3 PRECEDING AND 1 PRECEDING": (False, -3, -1),
    "ROWS 40 PRECEDING": (False, -40, 0),
    "ROWS BETWEEN 2 FOLLOWING AND 1 FOLLOWING": (False, 2, 1),          # empty for every row
    "ROWS BETWEEN 1 PRECEDING AND 3 PRECEDING": (False, -1, -3),        # empty for every row
    "RANGE BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING": (True, 0, INF),
    "RANGE BETWEEN CURRENT ROW AND CURRENT ROW": (True, 0, 0),
}


@pytest.fixture(scope="module")
def c():
    import torch
    torch.cuda.set_device(0)
    from dask_sql_b200 import Context
    return Context()


def _frame(sql_frame, has_order):
    f = FRAMES[sql_frame]
    if f is None:
        return (True, -INF, 0) if has_order else (False, -INF, INF)
    return f


def _got(df: pd.DataFrame, kinds):
    out = {}
    for name, kind in kinds.items():
        s = df[name]
        if kind in ("float", "bounded"):
            out[name] = [math.nan if pd.isna(x) else float(x) for x in s]
        elif kind == "str":
            out[name] = [None if pd.isna(x) else str(x) for x in s]
        elif kind == "bool":
            out[name] = [None if pd.isna(x) else bool(x) for x in s]
        elif pd.api.types.is_datetime64_any_dtype(s.dtype):
            out[name] = [None if pd.isna(x) else int(x) for x in s.to_numpy().astype("datetime64[D]").view(np.int64)]
        else:
            out[name] = [None if pd.isna(x) else int(x) for x in s]
    return out


def _check(c, sql, rel, cols, calls, what=None):
    """cols: plain columns of rel selected first; calls: [(alias, fn, arg, partition, order, frame)]"""
    got = c.sql(sql).compute()
    exp_cols, kinds = {}, {}
    for n in cols:
        kinds[n], exp_cols[n] = Q._cells(rel[n])
    for alias, fn, arg, partition, order, frame in calls:
        kinds[alias], exp_cols[alias] = W.window(rel, partition, order, fn, arg, frame)
    Q.assert_result(_got(got, kinds), Q.Result(exp_cols, kinds), what=what or sql)


def _table(rng, n, nkeys=7):
    k = rng.integers(0, nkeys, n).astype(float)
    k[rng.random(n) < 0.1] = np.nan
    t = rng.integers(0, 20, n).astype(np.int64)
    v = rng.normal(0, 100, n)
    v[rng.random(n) < 0.1] = np.nan
    iv = pd.array(rng.integers(-50, 50, n), dtype="Int64")
    iv[rng.random(n) < 0.1] = pd.NA
    return pd.DataFrame({"k": k, "t": t, "v": v, "iv": iv})


@pytest.mark.parametrize("fn", ["SUM", "AVG", "COUNT", "MIN", "MAX", "FIRST_VALUE", "LAST_VALUE"])
@pytest.mark.parametrize("arg", ["v", "iv"])
def test_frames_against_reference(c, fn, arg):
    rng = np.random.default_rng(1)
    df = _table(rng, 300)
    c.create_table("wt", df)
    rel = Q.table(df)
    items, calls = [], []
    for j, (text, _) in enumerate(FRAMES.items()):
        items.append(f"{fn}({arg}) OVER (PARTITION BY k ORDER BY t {text}) AS o{j}")
        calls.append((f"o{j}", fn, arg, ["k"], [("t", True, False)], _frame(text, True)))
    items.append(f"{fn}({arg}) OVER (PARTITION BY k) AS w")
    calls.append(("w", fn, arg, ["k"], [], _frame("", False)))
    sql = f"SELECT k, t, {', '.join(items)} FROM wt"
    # FIRST_VALUE / LAST_VALUE under tied ORDER BY keys pick a row SQL leaves open: order by a unique key too
    if fn in ("FIRST_VALUE", "LAST_VALUE"):
        df = df.assign(u=np.arange(len(df)))
        c.create_table("wt", df)
        rel = Q.table(df)
        sql = sql.replace("ORDER BY t", "ORDER BY t, u")
        calls = [(a, f, x, p, o + [("u", True, False)] if o else o, fr) for a, f, x, p, o, fr in calls]
    _check(c, sql, rel, ["k", "t"], calls)


def test_ranks_and_several_specs(c):
    rng = np.random.default_rng(2)
    df = _table(rng, 500)
    df["u"] = np.arange(len(df))
    c.create_table("wr", df)
    rel = Q.table(df)
    sql = ("SELECT k, t, ROW_NUMBER() OVER (PARTITION BY k ORDER BY t DESC, u) AS rn, "
           "RANK() OVER (PARTITION BY k ORDER BY t DESC) AS rk, DENSE_RANK() OVER (PARTITION BY k ORDER BY t DESC) "
           "AS dr, RANK() OVER (ORDER BY v NULLS FIRST) AS rv, COUNT(*) OVER () AS n FROM wr")
    desc = [("t", False, True)]
    _check(c, sql, rel, ["k", "t"], [
        ("rn", "ROW_NUMBER", None, ["k"], desc + [("u", True, False)], None),
        ("rk", "RANK", None, ["k"], desc, None),
        ("dr", "DENSE_RANK", None, ["k"], desc, None),
        ("rv", "RANK", None, [], [("v", True, True)], None),
        ("n", "COUNT", None, [], [], (False, -INF, INF))])


@pytest.mark.parametrize("n", [1, 31, 32, 33, 2047, 2049, 3 * 2048 + 5, 20_000])
def test_sizes_one_partition_and_singletons(c, n):
    rng = np.random.default_rng(n)
    x = rng.integers(-(1 << 62), 1 << 62, n)                     # int64 sums wrap
    f = rng.integers(-1000, 1000, n) / 8.0                        # dyadic: sums are exact
    df = pd.DataFrame({"one": np.zeros(n, np.int64), "own": np.arange(n), "x": x, "f": f})
    c.create_table("ws", df)
    rel = Q.table(df)
    fr = (False, -5, 2)
    sql = ("SELECT own, SUM(x) OVER (PARTITION BY one ORDER BY own) AS s, "
           "SUM(f) OVER (PARTITION BY one ORDER BY own ROWS BETWEEN 5 PRECEDING AND 2 FOLLOWING) AS sf, "
           "MAX(x) OVER (PARTITION BY one ORDER BY own ROWS BETWEEN 5 PRECEDING AND 2 FOLLOWING) AS mx, "
           "MIN(f) OVER (PARTITION BY one ORDER BY own ROWS BETWEEN 5 PRECEDING AND UNBOUNDED FOLLOWING) AS mn, "
           "ROW_NUMBER() OVER (PARTITION BY own) AS r1 FROM ws")
    _check(c, sql, rel, ["own"], [
        ("s", "SUM", "x", ["one"], [("own", True, False)], (True, -INF, 0)),
        ("sf", "SUM", "f", ["one"], [("own", True, False)], fr),
        ("mx", "MAX", "x", ["one"], [("own", True, False)], fr),
        ("mn", "MIN", "f", ["one"], [("own", True, False)], (False, -5, INF)),
        ("r1", "ROW_NUMBER", None, ["own"], [], None)])


def test_wide_minmax_frame(c):
    rng = np.random.default_rng(5)
    n = 30_000
    df = pd.DataFrame({"k": rng.integers(0, 3, n), "t": np.arange(n), "v": rng.normal(size=n)})
    c.create_table("wm", df)
    rel = Q.table(df)
    fr = (False, -1000, 0)
    sql = "SELECT t, MAX(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 1000 PRECEDING AND CURRENT ROW) AS m FROM wm"
    got = c.sql(sql).compute()
    perm, pkey, _ = W.sort_positions(rel, ["k"], [("t", True, False)])
    v = df["v"].to_numpy()
    exp = np.empty(n)
    for key in set(pkey):
        rows = [r for r, p in zip(perm, pkey) if p == key]
        vals = v[rows]
        exp[rows] = [vals[max(0, i - 1000):i + 1].max() for i in range(len(rows))]
    assert np.array_equal(got["m"].to_numpy(), exp)


def test_specials_in_keys_and_values(c):
    k = [0.0, -0.0, np.nan, np.nan, 1.0, INF, -INF, 0.0, None, 1.0]
    v = [1.0, INF, -INF, 2.0, np.nan, -0.0, 0.0, INF, 3.0, -INF]
    df = pd.DataFrame({"k": np.array(k, dtype=float), "u": np.arange(10), "v": np.array(v, dtype=float)})
    c.create_table("wx", df)
    rel = Q.table(df)
    calls = []
    items = []
    for j, fn in enumerate(["SUM", "MIN", "MAX", "COUNT", "FIRST_VALUE", "AVG"]):
        items.append(f"{fn}(v) OVER (PARTITION BY k ORDER BY u) AS o{j}")
        calls.append((f"o{j}", fn, "v", ["k"], [("u", True, False)], (True, -INF, 0)))
    _check(c, f"SELECT u, {', '.join(items)} FROM wx", rel, ["u"], calls)


def test_sources_filter_join_groupby_parquet(c, tmp_path):
    rng = np.random.default_rng(3)
    df = _table(rng, 400)
    df["u"] = np.arange(len(df))
    dim = pd.DataFrame({"t": np.arange(20), "w": rng.integers(0, 5, 20)})
    c.create_table("wf", df, npartitions=4)
    c.create_table("wd", dim)
    rel = Q.table(df)
    order = [("t", True, False), ("u", True, False)]
    # a filter
    sub = Q.where(rel, ~np.isnan(rel["v"].values) & (rel["v"].values > 0))
    _check(c, "SELECT u, SUM(v) OVER (PARTITION BY k ORDER BY t, u ROWS 3 PRECEDING) AS s FROM wf WHERE v > 0", sub,
           ["u"], [("s", "SUM", "v", ["k"], order, (False, -3, 0))])
    # a join
    joined = df.merge(dim, on="t")
    jrel = Q.table(joined[["u", "t", "w", "v"]])
    _check(c, "SELECT u, MAX(v) OVER (PARTITION BY w ORDER BY wf.t, u) AS m FROM wf JOIN wd ON wf.t = wd.t", jrel,
           ["u"], [("m", "MAX", "v", ["w"], order, (True, -INF, 0))])
    # a GROUP BY output, ranked by an aggregate
    g = df.groupby("t", as_index=False).agg(s=("iv", "sum"))
    grel = Q.table(g)
    _check(c, "SELECT t, SUM(iv) AS s, RANK() OVER (ORDER BY SUM(iv) DESC) AS r FROM wf GROUP BY t", grel, ["t", "s"],
           [("r", "RANK", None, [], [("s", False, True)], None)])
    # a lazy Parquet table
    path = str(tmp_path / "w.parquet")
    df.to_parquet(path, row_group_size=100)
    c.create_table("wp", path, format="parquet")
    _check(c, "SELECT u, COUNT(iv) OVER (PARTITION BY k ORDER BY t, u ROWS BETWEEN 2 PRECEDING AND 2 FOLLOWING) AS n "
           "FROM wp", rel, ["u"], [("n", "COUNT", "iv", ["k"], order, (False, -2, 2))])


def test_varchar_and_date(c):
    rng = np.random.default_rng(4)
    n = 200
    words = np.array(["pear", "apple", "fig", None, "kiwi"], dtype=object)
    s = words[rng.integers(0, 5, n)]
    d = pd.to_datetime("2020-01-01") + pd.to_timedelta(rng.integers(0, 400, n), unit="D")
    df = pd.DataFrame({"s": pd.Series(s, dtype="category"), "d": d.values.astype("datetime64[D]").astype("datetime64[s]"),
                       "u": np.arange(n)})
    c.create_table("wv", df)
    got = c.sql("SELECT u, MIN(s) OVER (PARTITION BY CAST(d AS DATE) ORDER BY u) AS ms, "
                "LAST_VALUE(s) OVER (ORDER BY u ROWS BETWEEN 1 PRECEDING AND CURRENT ROW) AS ls, "
                "MAX(d) OVER (PARTITION BY s ORDER BY u) AS md FROM wv").compute()
    days = df["d"].to_numpy().astype("datetime64[D]").view(np.int64)
    rel = {"s": Q.Column(np.array(s, dtype=object), np.array([x is None for x in s]), Q.STR),
           "dd": Q.Column(days, None, Q.I64), "u": Q.Column(np.arange(n), None, Q.I64)}
    _, ms = W.window(rel, ["dd"], [("u", True, False)], "MIN", "s", (True, -INF, 0))
    _, ls = W.window(rel, [], [("u", True, False)], "LAST_VALUE", "s", (False, -1, 0))
    _, md = W.window(rel, ["s"], [("u", True, False)], "MAX", "dd", (True, -INF, 0))
    g = _got(got, {"u": "int", "ms": "str", "ls": "str", "md": "int"})
    assert g["ms"] == ms and g["ls"] == ls and g["md"] == md


def test_top_n_and_order_limit(c):
    rng = np.random.default_rng(6)
    df = _table(rng, 300)
    df["u"] = np.arange(len(df))
    c.create_table("wn", df)
    got = c.sql("SELECT * FROM (SELECT k, u, ROW_NUMBER() OVER (PARTITION BY k ORDER BY u DESC) AS r FROM wn) s "
                "WHERE r <= 3").compute()
    exp = df.assign(kk=df["k"].fillna(-1)).sort_values("u", ascending=False).groupby("kk").head(3)
    assert sorted(got["u"].tolist()) == sorted(exp["u"].tolist())
    assert got["r"].max() == 3
    got = c.sql("SELECT u, SUM(t) OVER (ORDER BY u) AS s FROM wn ORDER BY s DESC LIMIT 5").compute()
    assert got["u"].tolist() == [299, 298, 297, 296, 295]
    assert got["s"].tolist() == [int(df["t"][:i + 1].sum()) for i in (299, 298, 297, 296, 295)]
    # a window call in ORDER BY that the SELECT list does not output, and one it outputs under an alias
    got = c.sql("SELECT u FROM wn ORDER BY SUM(t) OVER (ORDER BY u) DESC LIMIT 5").compute()
    assert list(got.columns) == ["u"] and got["u"].tolist() == [299, 298, 297, 296, 295]
    got = c.sql("SELECT u, ROW_NUMBER() OVER (ORDER BY u DESC) AS r FROM wn "
                "ORDER BY ROW_NUMBER() OVER (ORDER BY u DESC) LIMIT 3").compute()
    assert got["u"].tolist() == [299, 298, 297] and got["r"].tolist() == [1, 2, 3]


@pytest.mark.parametrize("case", list(GW.CASES))
def test_reference_known_answers(c, case):
    table, rows, sql, expected = GW.CASES[case]
    c.create_table(table, pd.DataFrame(rows))
    got = c.sql(sql).compute()
    for name, want in expected.items():
        have = [None if pd.isna(x) else x for x in got[name]]
        assert have == want, f"{case}: {name} = {have}, expected {want}"
