"""Subqueries end to end on the GPU: Context.sql() against sqlite3 running the same SQL on the same rows, for
[NOT] IN, [NOT] EXISTS and scalar subqueries in WHERE, HAVING and the SELECT list, under NOT / OR / CASE,
nested, over multi-partition tables, with VARCHAR keys of two dictionaries and DATE keys, small Q4-, Q16-, Q18-
Q17-, Q20- and Q21-shaped queries, correlated scalar subqueries (COUNT of an empty group
is 0), two subqueries in one SELECT list, a correlated [NOT] IN on a float column whose NULLs are NaN, the reference's EXISTS answer, the more-than-one-row error, stats["marks"], and the
star path declining a query with a mark."""
import sqlite3

import numpy as np
import pandas as pd
import pytest

from tests.golden import reference_subquery as GS

pytestmark = pytest.mark.gpu


def _frames(seed=0, n=4000, m=900):
    rng = np.random.default_rng(seed)

    def nullable(v, p):
        s = pd.Series(v).astype("Int64")
        s[rng.random(len(v)) < p] = pd.NA
        return s

    def floats(k):                       # a NULL float is a NaN
        v = rng.integers(0, 6, k).astype(np.float64)
        v[rng.random(k) < 0.1] = np.nan
        return v

    o = pd.DataFrame({"a": nullable(rng.integers(0, 60, n), 0.05), "b": rng.integers(0, 100, n),
                      "c": nullable(rng.integers(0, 10, n), 0.05), "v": rng.random(n), "f": floats(n)})
    i = pd.DataFrame({"x": nullable(rng.integers(0, 50, m), 0.05), "y": rng.integers(0, 100, m),
                      "z": nullable(rng.integers(0, 10, m), 0.05), "g": floats(m)})
    return o, i


@pytest.fixture(scope="module")
def env():
    import torch
    torch.cuda.set_device(0)
    from dask_sql_b200 import Context
    o, i = _frames()
    c = Context()
    c.create_table("o", o, npartitions=3)
    c.create_table("i", i)
    db = sqlite3.connect(":memory:")
    o.astype(object).where(o.notna(), None).to_sql("o", db, index=False)
    i.astype(object).where(i.notna(), None).to_sql("i", db, index=False)
    return c, db


def _norm(v):
    if v is None or (isinstance(v, float) and np.isnan(v)) or v is pd.NA:
        return None
    if isinstance(v, (bool, np.bool_)):
        return int(v)
    if isinstance(v, (float, np.floating)):
        return round(float(v), 9)
    return int(v) if isinstance(v, (int, np.integer)) else v


def _same(c, db, sql):
    got = c.sql(sql, return_futures=False)
    want = db.execute(sql).fetchall()
    g = sorted((tuple(_norm(x) for x in r) for r in got.itertuples(index=False)), key=repr)
    w = sorted((tuple(_norm(x) for x in r) for r in want), key=repr)
    assert g == w, sql
    return got


QUERIES = [
    "SELECT a, b FROM o WHERE a IN (SELECT x FROM i)",
    "SELECT a, b FROM o WHERE a NOT IN (SELECT x FROM i WHERE y > 20)",
    "SELECT a, b FROM o WHERE a NOT IN (SELECT y FROM i)",
    "SELECT a, b FROM o WHERE b > 50 AND EXISTS (SELECT 1 FROM i WHERE i.x = o.a)",
    "SELECT a, b FROM o WHERE NOT EXISTS (SELECT 1 FROM i WHERE i.x = o.a AND i.y < o.b)",
    "SELECT a, b FROM o WHERE EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.z <> o.c)",
    "SELECT a, b FROM o WHERE c IN (SELECT z FROM i WHERE i.x = o.a)",
    "SELECT a, b FROM o WHERE c NOT IN (SELECT z FROM i WHERE i.x = o.a AND i.y >= o.b)",
    "SELECT a, b FROM o WHERE a IN (SELECT x FROM i) OR b < 10",
    "SELECT a, b FROM o WHERE NOT (a IN (SELECT x FROM i WHERE z = 3))",
    "SELECT a, CASE WHEN a IN (SELECT x FROM i) THEN 1 ELSE 0 END AS k FROM o",
    "SELECT a, a IN (SELECT x FROM i WHERE y < 30) AS m FROM o",
    "SELECT a, EXISTS (SELECT 1 FROM i WHERE i.x = o.a AND i.y > o.b) AS e FROM o",
    "SELECT a, b FROM o WHERE EXISTS (SELECT 1 FROM i WHERE y > 1000)",
    "SELECT a, b FROM o WHERE NOT EXISTS (SELECT 1 FROM i WHERE y > 1000)",
    "SELECT a, b FROM o WHERE b > (SELECT AVG(y) FROM i)",
    "SELECT a, b, (SELECT MAX(y) FROM i) AS top FROM o WHERE c = 1",
    "SELECT a, b FROM o WHERE b > (SELECT MAX(y) FROM i WHERE y > 1000)",
    "SELECT c, COUNT(*) AS n FROM o GROUP BY c HAVING c IN (SELECT z FROM i WHERE y < 50)",
    "SELECT c, SUM(b) AS s FROM o GROUP BY c HAVING SUM(b) > (SELECT SUM(y) FROM i) / 20",
    # nesting
    "SELECT a, b FROM o WHERE a IN (SELECT x FROM i WHERE z IN (SELECT c FROM o WHERE b < 5))",
    # Q18: IN over a grouped subquery with HAVING
    "SELECT a, SUM(b) AS s FROM o WHERE a IN (SELECT x FROM i GROUP BY x HAVING SUM(y) > 800) GROUP BY a",
    # Q4: EXISTS with a correlated pair term, then a GROUP BY
    "SELECT c, COUNT(*) AS n FROM o WHERE b < 80 AND EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.y < o.b) "
    "GROUP BY c",
    # Q16: NOT IN of a filtered subquery, then COUNT(DISTINCT)
    "SELECT c, COUNT(DISTINCT a) AS n FROM o WHERE a NOT IN (SELECT x FROM i WHERE y > 90 AND x IS NOT NULL) "
    "GROUP BY c",
    # Q21: EXISTS with <> and NOT EXISTS with <> and >
    "SELECT a, COUNT(*) AS n FROM o WHERE EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.z <> o.c) "
    "AND NOT EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.z <> o.c AND i.y > o.b) GROUP BY a",
    # two subqueries in one SELECT list
    "SELECT a, a IN (SELECT x FROM i) AS m, EXISTS (SELECT 1 FROM i WHERE i.x = o.a AND i.y > o.b) AS e FROM o",
    # correlated [NOT] IN on a float column whose NULLs are NaN
    "SELECT a, b FROM o WHERE f IN (SELECT g FROM i WHERE i.x = o.a)",
    "SELECT a, b FROM o WHERE f NOT IN (SELECT g FROM i WHERE i.x = o.a)",
    "SELECT a, b FROM o WHERE f NOT IN (SELECT g FROM i WHERE y < 40)",
    # a grouped correlated body
    "SELECT a, b FROM o WHERE EXISTS (SELECT z FROM i WHERE i.x = o.a GROUP BY z HAVING COUNT(*) > 1)",
    # Q17: correlated scalar AVG, decorrelated into a LEFT JOIN on the grouped body
    "SELECT SUM(v) AS s, COUNT(*) AS n FROM o WHERE b < (SELECT 0.6 * AVG(y) FROM i WHERE i.x = o.a)",
    # COUNT over an empty correlation group is 0, in the SELECT list and in WHERE
    "SELECT a, b, (SELECT COUNT(*) FROM i WHERE i.x = o.a AND i.y > 50) AS n FROM o",
    "SELECT a, b FROM o WHERE (SELECT COUNT(y) FROM i WHERE i.x = o.a AND i.y > 90) = 0",
    "SELECT a, b, (SELECT MAX(y) FROM i WHERE i.x = o.a) AS top FROM o WHERE c = 2",
    # Q20: IN whose body filters by a correlated scalar SUM of a third block
    "SELECT a, b FROM o WHERE a IN (SELECT x FROM i WHERE y > (SELECT SUM(b) FROM o WHERE o.a = i.x) / 100)",
    # CTE reference inside the body
    "WITH big AS (SELECT x FROM i WHERE y > 60) SELECT a FROM o WHERE a IN (SELECT x FROM big)",
]


@pytest.mark.parametrize("sql", QUERIES)
def test_matches_sqlite(env, sql):
    c, db = env
    _same(c, db, sql)


def test_marks_counted_and_star_path_declines():
    """the Q3 shape fuses into the star path; the same query with an IN subquery over its fact rows does not"""
    from dask_sql_b200 import Context, executor
    rng = np.random.default_rng(0)
    nd, nf = 5000, 200_000
    dim = pd.DataFrame({"pk": rng.permutation(nd).astype(np.int64), "flag": rng.integers(0, 10, nd),
                        "grp": rng.integers(0, 100, nd)})
    fact = pd.DataFrame({"fk": rng.integers(0, nd, nf), "x": rng.integers(-100, 100, nf), "val": rng.random(nf)})
    keep = pd.DataFrame({"k": np.arange(0, 100, 3, dtype=np.int64)})
    c = Context()
    c.create_table("fact", fact, npartitions=4)
    c.create_table("dim", dim)
    c.create_table("keep", keep)
    q3 = ("SELECT d.grp, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fk = d.pk WHERE f.x > 0 AND d.flag < 5 {} "
          "GROUP BY d.grp")
    marks, star = executor.stats["marks"], executor.stats["star_fused"]
    c.sql(q3.format(""), return_futures=False)
    assert executor.stats["star_fused"] > star and executor.stats["marks"] == marks
    star = executor.stats["star_fused"]
    got = c.sql(q3.format("AND f.x IN (SELECT k FROM keep)"), return_futures=False)
    assert executor.stats["star_fused"] == star and executor.stats["marks"] > marks
    j = fact[(fact.x > 0) & fact.x.isin(keep.k)].merge(dim[dim.flag < 5], left_on="fk", right_on="pk")
    want = j.groupby("grp").val.sum()
    got = got.set_index("grp").rev.sort_index()
    assert got.index.tolist() == want.index.tolist()
    np.testing.assert_allclose(got.to_numpy(), want.to_numpy(), rtol=1e-9)


def test_more_than_one_row_is_an_error(env):
    c, _ = env
    with pytest.raises(ValueError, match="more than one row"):
        c.sql("SELECT a FROM o WHERE b > (SELECT y FROM i)", return_futures=False)


def test_varchar_keys_of_two_dictionaries_and_date_keys():
    from dask_sql_b200 import Context
    rng = np.random.default_rng(4)
    words = np.array(["ant", "bee", "cat", "dog", "eel", "fox"])
    o = pd.DataFrame({"s": pd.Series(words[rng.integers(0, 6, 500)]).astype("category"), "d": pd.to_datetime("2024-01-01") +
                      pd.to_timedelta(rng.integers(0, 40, 500), unit="D"), "k": rng.integers(0, 9, 500)})
    i = pd.DataFrame({"t": pd.Series(words[rng.integers(2, 6, 60)].tolist() + ["zebra"]).astype("category"), "e": (
        pd.to_datetime("2024-01-10") + pd.to_timedelta(rng.integers(0, 40, 61), unit="D")).values.astype("datetime64[s]")})
    c = Context()
    c.create_table("o", o, npartitions=2)
    c.create_table("i", i)
    got = c.sql("SELECT s, k FROM o WHERE s IN (SELECT t FROM i)", return_futures=False)
    want = o[o.s.isin(set(i.t))]
    assert sorted(zip(got.s.astype(str), got.k)) == sorted(zip(want.s.astype(str), want.k))
    got = c.sql("SELECT k FROM o WHERE NOT EXISTS (SELECT 1 FROM i WHERE i.e = o.d)", return_futures=False)
    keep = ~o.d.isin(set(pd.to_datetime(i.e)))
    assert sorted(got.k.tolist()) == sorted(o.k[keep].tolist())


def test_lazy_parquet_table(tmp_path, env):
    from dask_sql_b200 import Context
    _, db = env
    o, i = _frames()
    path = tmp_path / "o.parquet"
    o.to_parquet(path, row_group_size=700)
    c = Context()
    c.create_table("o", str(path), format="parquet")
    c.create_table("i", i)
    _same(c, db, "SELECT a, b FROM o WHERE a NOT IN (SELECT x FROM i WHERE y > 20) AND b > 10")
    _same(c, db, "SELECT a, b FROM o WHERE EXISTS (SELECT 1 FROM i WHERE i.x = o.a AND i.y < o.b)")


def test_reference_exists_answer():
    from dask_sql_b200 import Context
    c = Context()
    c.create_table("user_table_1", pd.DataFrame(GS.USER_TABLE_1))
    c.create_table("user_table_2", pd.DataFrame(GS.USER_TABLE_2))
    got = c.sql(GS.EXISTS_SQL, return_futures=False)
    assert list(got.columns) == ["user_id", "c"]
    assert sorted(map(tuple, got.values.tolist())) == GS.EXISTS_ANSWER
