"""SQL-level GPU parity: the reference's known-answer tests (tests/golden/reference_vectors.py)
and a sqlite3 differential on seeded random data (the reference's own differential oracle,
tests/integration/test_compatibility.py:25-83), both through Context.sql() -> plugins ->
libb200sql.so.  Row order is not part of the contract (frames are compared as multisets)."""
import sqlite3

import numpy as np
import pandas as pd
import pytest

from tests.golden import reference_vectors as G

pytestmark = pytest.mark.gpu


def _norm(df):
    out = pd.DataFrame({str(c): df[c].to_numpy(dtype=float, na_value=np.nan) for c in df.columns})
    if len(out):
        out = out.sort_values(list(out.columns), na_position="last").reset_index(drop=True)
    return out


def assert_same(got, exp, float_cols=(), rtol=1e-9, check_names=True):
    assert len(got.columns) == len(exp.columns), f"{list(got.columns)} vs {list(exp.columns)}"
    if check_names:
        assert [str(c) for c in got.columns] == [str(c) for c in exp.columns]
    g, e = _norm(got), _norm(exp)
    e.columns = g.columns
    assert len(g) == len(e), f"{len(g)} rows vs {len(e)}"
    for c, ce in zip(g.columns, exp.columns):
        if str(ce) in float_cols or str(c) in float_cols:
            np.testing.assert_allclose(g[c].to_numpy(), e[c].to_numpy(), rtol=rtol, equal_nan=True)
        else:
            np.testing.assert_array_equal(g[c].to_numpy(), e[c].to_numpy())


@pytest.fixture()
def c():
    from dask_sql_b200 import Context
    return Context()


@pytest.mark.parametrize("case", G.CASES, ids=[c["name"] for c in G.CASES])
@pytest.mark.parametrize("npartitions", [1, 3])
def test_reference_known_answers(c, case, npartitions):
    tables = G.tables_of(case)
    for name, df in tables.items():
        c.create_table(name, df, npartitions=npartitions)   # the reference registers with npartitions=3
    got = c.sql(case["sql"]).compute()
    exp = G.expected_of(case, tables)
    assert_same(got, exp, case.get("float_cols", ()))


def make_rand_df(size, seed=0, **kwargs):
    """Same generator shape as the reference's make_rand_df (test_compatibility.py:50-83):
    kwargs: column -> (type, null_ct)."""
    np.random.seed(seed)
    data = {}
    for k, v in kwargs.items():
        dt, null_ct = v if isinstance(v, tuple) else (v, 0)
        if dt is int:
            s = np.random.randint(10, size=size).astype(float if null_ct else int)
        elif dt is float:
            s = np.random.rand(size)
        elif dt is bool:
            s = np.where(np.random.randint(2, size=size), True, False).astype(object if null_ct else bool)
        else:
            raise NotImplementedError
        s = pd.Series(s)
        if null_ct:
            idx = np.random.choice(size, null_ct, replace=False).tolist()
            s[idx] = np.nan
        data[k] = s
    return pd.DataFrame(data)


def eq_sqlite(c, sql, float_cols=(), **dfs):
    con = sqlite3.connect(":memory:")
    for name, df in dfs.items():
        c.create_table(name, df, npartitions=2)
        df.to_sql(name, con, index=False)
    got = c.sql(sql).compute()
    exp = pd.read_sql(sql, con)
    assert_same(got, exp, float_cols or [str(x) for x in exp.columns if exp[x].dtype.kind == "f"], check_names=False)


def test_where(c):
    # tests/integration/test_compatibility.py:177-196 (int columns; float columns carry NaN whose
    # comparison semantics differ between numpy and sqlite, see DESIGN.md)
    df = make_rand_df(100, a=(int, 30), b=(int, 30), c=(float, 0))
    eq_sqlite(c, "SELECT * FROM a WHERE TRUE OR TRUE", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE FALSE AND FALSE", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a<2 OR c>0.8", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a<2 AND c>0.3", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a IS NULL OR (b>=5 AND c<0.5)", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE c IS NOT NULL OR (a<5 AND b IS NOT NULL)", a=df)
    eq_sqlite(c, "SELECT a + b AS s, a * 2 - b AS t, c / 2 AS h FROM a WHERE a = b OR a > 3", a=df)
    # the reference's float block (test_compatibility.py:191-196), NaN as NULL in all three columns
    df = make_rand_df(100, a=(float, 30), b=(float, 30), c=(float, 30))
    eq_sqlite(c, "SELECT * FROM a WHERE a<0.5 AND b<0.5 AND c<0.5", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a<0.5 OR b<0.5 AND c<0.5", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a IS NULL OR (b<0.5 AND c<0.5)", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a*b IS NULL OR (b*c<0.5 AND c*a<0.5)", a=df)
    # NOT / <> over a nullable INTEGER column follow SQL three-valued logic (validity bitmap)
    df = pd.DataFrame({"a": pd.array(np.where(np.arange(100) % 7 == 0, None, np.arange(100) % 10), dtype="Int64"),
                       "b": np.arange(100) % 4})
    eq_sqlite(c, "SELECT * FROM a WHERE NOT (a<5) AND b <> 1", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a <> 3 OR b = 0", a=df)


def test_in_between(c):
    # test_compatibility.py:198-207
    df = make_rand_df(100, a=(int, 30), b=(int, 0))
    eq_sqlite(c, "SELECT * FROM a WHERE a IN (2,4,6)", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a BETWEEN 2 AND 4+1", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a NOT IN (2,4,6) AND a IS NOT NULL", a=df)
    eq_sqlite(c, "SELECT * FROM a WHERE a NOT BETWEEN 2 AND 4+1 AND a IS NOT NULL", a=df)


def test_join_inner_and_left(c):
    # test_compatibility.py:210-238
    a = make_rand_df(100, a=(int, 40), b=(int, 0), c=int)
    b = make_rand_df(80, seed=1, d=(float, 10), a=(int, 10), b=(int, 0))
    eq_sqlite(c, "SELECT a.*, d, d*c AS x FROM a INNER JOIN b ON a.a=b.a AND a.b=b.b", a=a, b=b)
    eq_sqlite(c, "SELECT a.*, d, d*c AS x FROM a LEFT JOIN b ON a.a=b.a AND a.b=b.b", a=a, b=b)
    eq_sqlite(c, "SELECT a.a, a.c, b.d FROM a JOIN b ON a.a = b.a WHERE a.c > 3 AND b.d < 0.7", a=a, b=b)


def test_agg_count_sum_avg_min_max(c):
    # test_compatibility.py:379-451, 490-522
    a = make_rand_df(100, a=(int, 50), b=(int, 50), c=(int, 30), d=(float, 30), e=(float, 40))
    eq_sqlite(c, """SELECT a, b, COUNT(c) AS c_c, COUNT(d) AS c_d, COUNT(*) AS n, SUM(c) AS s_c, AVG(c) AS a_c,
                    SUM(d) AS s_d, AVG(e) AS a_e, MIN(c) AS mn, MAX(d) AS mx
                    FROM a GROUP BY a, b""", a=a)
    eq_sqlite(c, "SELECT SUM(c) AS s, AVG(d) AS av, COUNT(*) AS n, MIN(e) AS mn, MAX(c) AS mx FROM a", a=a)
    eq_sqlite(c, "SELECT a, SUM(c+d) AS s, AVG(c*2) AS av FROM a WHERE b IS NOT NULL GROUP BY a", a=a)
    eq_sqlite(c, "SELECT a, COUNT(DISTINCT b) AS cd FROM a GROUP BY a", a=a)
    eq_sqlite(c, "SELECT DISTINCT a, b FROM a", a=a)
    eq_sqlite(c, "SELECT a, SUM(c) AS s FROM a GROUP BY a HAVING SUM(c) > 20", a=a)


def test_stddev_variance(c):
    # moment aggregates (aggregate.py:129-231): sample = ddof 1 like pandas std()/var(), pop = ddof 0
    rng = np.random.default_rng(3)
    df = pd.DataFrame({"k": rng.integers(0, 6, 500), "v": rng.normal(5, 2, 500), "i": rng.integers(-9, 9, 500)})
    df.loc[rng.integers(0, 500, 40), "v"] = np.nan
    c.create_table("t", df, npartitions=3)
    got = c.sql("""SELECT k, STDDEV(v) AS sd, STDDEV_POP(v) AS sdp, VAR_SAMP(v) AS vs, VAR_POP(i) AS vp, AVG(v) AS m
                   FROM t GROUP BY k""", return_futures=False)
    g = df.groupby("k")
    exp = pd.DataFrame({"k": sorted(df.k.unique()), "sd": g.v.std().values, "sdp": g.v.std(ddof=0).values,
                        "vs": g.v.var().values, "vp": g.i.var(ddof=0).values, "m": g.v.mean().values})
    assert_same(got, exp, ["sd", "sdp", "vs", "vp", "m"], rtol=1e-9)
    got = c.sql("SELECT STDDEV_SAMP(i) AS sd, VARIANCE(v) AS vs FROM t WHERE k < 3", return_futures=False)
    e = df[df.k < 3]
    np.testing.assert_allclose([got.sd[0], got.vs[0]], [e.i.std(), e.v.var()], rtol=1e-9)


def test_variance_is_stable_for_large_means(c):
    """sum-of-squares around zero loses every digit of VAR when mean >> spread (1e9 +- 1 in float64:
    S2/n - mean^2 cancels ~18 of 16 digits); the shifted moments must agree with pandas (Welford)."""
    rng = np.random.default_rng(8)
    n = 200_000
    df = pd.DataFrame({"k": rng.integers(0, 50, n), "v": 1e9 + rng.normal(0, 1, n),
                       "w": rng.integers(10**12, 10**12 + 1000, n)})
    c.create_table("t", df, npartitions=4)
    got = c.sql("SELECT k, VAR_SAMP(v) AS vs, STDDEV_POP(v) AS sp, VAR_POP(w) AS vw FROM t GROUP BY k",
                return_futures=False)
    # expected values from CENTRED data (v - 1e9 and w - 1e12 are exact in float64): pandas' own running
    # update on the raw values is itself only good to ~1e-7 here
    cen = pd.DataFrame({"k": df.k, "v": df.v - 1e9, "w": (df.w - 10**12).astype(float)})
    g = cen.groupby("k")
    exp = pd.DataFrame({"k": sorted(df.k.unique()), "vs": g.v.var().values, "sp": g.v.std(ddof=0).values,
                        "vw": g.w.var(ddof=0).values})
    assert_same(got, exp, ["vs", "sp", "vw"], rtol=1e-9)
    g_raw = df.groupby("k")                                      # and pandas on the raw values agrees to its own precision
    np.testing.assert_allclose(got.sort_values("k").vs.to_numpy(), g_raw.v.var().values, rtol=1e-5)
    got = c.sql("SELECT VARIANCE(v) AS vs, STDDEV(w) AS sw FROM t", return_futures=False)
    np.testing.assert_allclose([got.vs[0], got.sw[0]], [cen.v.var(), cen.w.std()], rtol=1e-9)
    # a constant group has variance exactly 0 (not NaN from sqrt of -1e-17); one row: sample variance NULL
    c.create_table("u", pd.DataFrame({"k": [1, 1, 1, 2], "v": [3.3e8 + 0.1] * 3 + [7.0]}))
    got = c.sql("SELECT k, STDDEV_POP(v) AS sp, VAR_SAMP(v) AS vs FROM u GROUP BY k", return_futures=False)
    got = got.sort_values("k").reset_index(drop=True)
    assert got.sp.tolist() == [0.0, 0.0] and got.vs[0] == 0.0 and pd.isna(got.vs[1])


def test_distinct_and_plain_aggregates_together(c):
    """COUNT(DISTINCT x) next to ordinary aggregates: one pass per distinct input, stitched on the keys
    (a literal key when there is no GROUP BY)."""
    rng = np.random.default_rng(21)
    n = 20_000
    df = pd.DataFrame({"k": rng.integers(0, 30, n), "a": rng.integers(0, 100, n), "b": rng.integers(0, 7, n),
                       "v": rng.random(n)})
    c.create_table("t", df, npartitions=3)
    got = c.sql("""SELECT k, COUNT(DISTINCT a) AS da, COUNT(DISTINCT b) AS db, SUM(v) AS s, COUNT(*) AS n
                   FROM t GROUP BY k""", return_futures=False)
    g = df.groupby("k")
    exp = pd.DataFrame({"k": sorted(df.k.unique()), "da": g.a.nunique().values, "db": g.b.nunique().values,
                        "s": g.v.sum().values, "n": g.size().values})
    assert_same(got, exp, ["s"])
    got = c.sql("SELECT COUNT(DISTINCT a) AS da, SUM(v) AS s, COUNT(DISTINCT b) AS db FROM t WHERE k < 10",
                return_futures=False)
    e = df[df.k < 10]
    assert len(got) == 1 and int(got.da[0]) == e.a.nunique() and int(got.db[0]) == e.b.nunique()
    np.testing.assert_allclose(float(got.s[0]), e.v.sum(), rtol=1e-9)
    got = c.sql("SELECT k, SUM(v) FILTER (WHERE a > 50) AS s, COUNT(*) FILTER (WHERE b = 3) AS n3, COUNT(*) AS n "
                "FROM t GROUP BY k", return_futures=False)
    exp = pd.DataFrame({"k": sorted(df.k.unique()),
                        "s": df[df.a > 50].groupby("k").v.sum().reindex(sorted(df.k.unique())).values,
                        "n3": df[df.b == 3].groupby("k").size().reindex(sorted(df.k.unique()), fill_value=0).values,
                        "n": g.size().values})
    assert_same(got, exp, ["s"])


@pytest.mark.parametrize("split_out", [1, 2, 4])
def test_groupby_split_out(c, split_out):
    """sql.aggregate.split_out (tests/integration/test_groupby.py:491-523): the result has that many
    partitions, every group in exactly one of them; also for DISTINCT and with a NULL-able key."""
    from dask_sql_b200 import executor
    rng = np.random.default_rng(split_out)
    n = 3_000
    df = pd.DataFrame({"user_id": pd.array(np.where(rng.random(n) < 0.05, None, rng.integers(0, 300, n)), dtype="Int64"),
                       "b": rng.integers(0, 50, n)})
    c.create_table("user_table_1", df, npartitions=3)
    lazy = c.sql('SELECT user_id, SUM(b) AS "S" FROM user_table_1 GROUP BY user_id',
                 config_options={"sql.aggregate.split_out": split_out})
    assert lazy.npartitions == split_out
    parts = executor.execute(lazy)
    assert len(parts) == split_out
    seen = [set(executor.D.column_to_host(p["user_id"]).tolist() if p.n else []) for p in parts]
    for i in range(len(seen)):
        for j in range(i + 1, len(seen)):
            assert not ({x for x in seen[i] if x is not pd.NA} & {x for x in seen[j] if x is not pd.NA})
    exp = df.groupby("user_id", dropna=False).agg(S=("b", "sum")).reset_index()
    assert_same(lazy.compute(), exp)
    lazy = c.sql("SELECT DISTINCT(user_id) FROM user_table_1", config_options={"sql.aggregate.split_out": split_out})
    assert lazy.npartitions == split_out
    assert_same(lazy.compute(), df[["user_id"]].drop_duplicates())


def test_order_by_limit(c):
    # ORDER BY / LIMIT (tests/integration/test_sort.py: results compared in order)
    rng = np.random.default_rng(5)
    n = 50_000
    df = pd.DataFrame({"a": rng.integers(-20, 20, n), "b": rng.random(n), "c": rng.integers(0, 1000, n)})
    df.loc[rng.integers(0, n, 300), "b"] = np.nan
    df["k"] = pd.array(np.where(rng.random(n) < 0.02, None, rng.integers(-3, 4, n)), dtype="Int64")
    c.create_table("t", df, npartitions=3)

    def check(sql, exp, float_cols=("b",)):
        got = c.sql(sql, return_futures=False).reset_index(drop=True)
        exp = exp.reset_index(drop=True)
        assert len(got) == len(exp)
        for col in exp.columns:
            g = got[col].to_numpy(dtype=float, na_value=np.nan)
            e = exp[col].to_numpy(dtype=float, na_value=np.nan)
            np.testing.assert_array_equal(g, e)

    check("SELECT a, c FROM t ORDER BY a, c", df.sort_values(["a", "c"], kind="stable")[["a", "c"]])
    check("SELECT a, c FROM t ORDER BY a DESC, c ASC", df.sort_values(["a", "c"], ascending=[False, True], kind="stable")[["a", "c"]])
    # floats with NaN: ASC defaults to NULLS LAST, DESC to NULLS FIRST (postgres / DataFusion defaults)
    check("SELECT b FROM t ORDER BY b", df.sort_values("b", na_position="last")[["b"]])
    check("SELECT b FROM t ORDER BY b DESC", df.sort_values("b", ascending=False, na_position="first")[["b"]])
    check("SELECT b FROM t ORDER BY b DESC NULLS LAST", df.sort_values("b", ascending=False, na_position="last")[["b"]])
    check("SELECT k, c FROM t ORDER BY k NULLS FIRST, c DESC",
          df.sort_values("c", ascending=False, kind="stable").sort_values("k", na_position="first", kind="stable")[["k", "c"]])
    check("SELECT a, c FROM t ORDER BY a, c LIMIT 17", df.sort_values(["a", "c"], kind="stable")[["a", "c"]].head(17))
    check("SELECT a, c FROM t ORDER BY a, c LIMIT 10 OFFSET 33",
          df.sort_values(["a", "c"], kind="stable")[["a", "c"]].iloc[33:43])
    check("SELECT a, c FROM t ORDER BY a + c DESC, c LIMIT 50",
          df.assign(s=df.a + df.c).sort_values(["s", "c"], ascending=[False, True], kind="stable")[["a", "c"]].head(50))
    # the real TPC-H Q3 tail: top groups by revenue
    got = c.sql("SELECT a, SUM(c) AS rev FROM t WHERE c > 10 GROUP BY a ORDER BY rev DESC, a LIMIT 5",
                return_futures=False)
    e = df[df.c > 10].groupby("a", as_index=False).agg(rev=("c", "sum")).sort_values(
        ["rev", "a"], ascending=[False, True], kind="stable").head(5)
    assert got["a"].tolist() == e["a"].tolist() and got["rev"].tolist() == e["rev"].tolist()


def test_integration_filter_join_groupby(c):
    # shape of test_compatibility.py:1015-1036 (CTEs: filter + agg + inner + left join)
    a = make_rand_df(200, a=int, b=(int, 20), c=(float, 0))
    b = make_rand_df(60, seed=2, a=int, d=(float, 0))
    eq_sqlite(c, """
        WITH t1 AS (SELECT a, SUM(c) AS sc FROM a WHERE b > 2 GROUP BY a),
             t2 AS (SELECT a, AVG(d) AS ad FROM b GROUP BY a)
        SELECT t1.a, t1.sc, t2.ad FROM t1 INNER JOIN t2 ON t1.a = t2.a
        """, a=a, b=b)
    eq_sqlite(c, """
        SELECT x.a, x.sc, b.d FROM (SELECT a, SUM(c) AS sc FROM a GROUP BY a) AS x
        LEFT JOIN b ON x.a = b.a WHERE x.sc > 5
        """, a=a, b=b)


def test_q3_shape_uses_fused_pipeline(c):
    from dask_sql_b200 import executor
    from oracle import pandas_oracle as O
    rng = np.random.default_rng(4)
    nd, nf = 20_000, 500_000
    dim = pd.DataFrame({"pk": rng.permutation(nd), "flag": rng.integers(0, 10, nd), "grp": rng.integers(0, 500, nd)})
    fact = pd.DataFrame({"fk": rng.integers(0, nd, nf), "x": rng.integers(-2**31, 2**31, nf), "val": rng.random(nf)})
    c.create_table("fact", fact, npartitions=8, persist=True)
    c.create_table("dim", dim, persist=True)
    before = executor.stats["star_fused"]
    got = c.sql("""SELECT d.grp, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fk = d.pk
                   WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp""", return_futures=False)
    assert executor.stats["star_fused"] == before + 1
    assert_same(got, O.c4_q3(O.split(fact, 8), dim), ["rev"])
    # C1 / C2 / C3 shapes
    got = c.sql("SELECT SUM(x) FROM fact WHERE x > 0", return_futures=False)
    assert int(got.iloc[0, 0]) == int(fact.x[fact.x > 0].sum())
    assert list(got.columns) == ["SUM(fact.x)"]
    got = c.sql("SELECT fk, SUM(val) AS s, AVG(val) AS a FROM fact GROUP BY fk", return_futures=False)
    exp = O.c5_groupby_sum_avg(O.split(fact.rename(columns={"fk": "key"})[["key", "val"]], 8))
    assert_same(got, exp, ["s", "a"], check_names=False)
    got = c.sql("SELECT f.fk, f.val, d.grp FROM fact f JOIN dim d ON f.fk = d.pk", return_futures=False)
    exp = fact.merge(dim, left_on="fk", right_on="pk")[["fk", "val", "grp"]]
    assert_same(got, exp, ["val"])


def test_plumbing(c):
    # tests/unit/test_context.py:51-69: lazy vs computed, dataframes= kwarg, explain
    df = pd.DataFrame({"a": [1, 2, 3], "b": [1.1, 2.2, 3.3]})
    c.create_table("df", df)
    lazy = c.sql("SELECT a FROM df")
    assert not isinstance(lazy, pd.DataFrame) and lazy.columns == ["a"]
    assert lazy.compute()["a"].tolist() == [1, 2, 3]
    res = c.sql("SELECT a FROM other", return_futures=False, dataframes={"other": df})
    assert isinstance(res, pd.DataFrame) and res["a"].tolist() == [1, 2, 3]
    assert "TableScan: df projection=[a]" in c.explain("SELECT a FROM df")
    c.drop_table("df")
    with pytest.raises(Exception):
        c.sql("SELECT a FROM df")
    # per-query config (context.py:519) and split_out/split_every keys are accepted
    res = c.sql("SELECT a, SUM(b) AS s FROM other GROUP BY a", return_futures=False,
                config_options={"sql.aggregate.split_out": 2, "sql.aggregate.split_every": 3})
    assert len(res) == 3


def test_no_cpu_fallback_errors_are_loud(c):
    df = pd.DataFrame({"a": [1, 2, 3], "s": ["x", "y", "z"]})
    with pytest.raises(NotImplementedError):
        c.create_table("t", df)          # strings are outside the int64/float64 hot path


def _ingest_frame(n=10_007, seed=3):
    rng = np.random.default_rng(seed)
    return pd.DataFrame({
        "k": rng.integers(0, 50, n).astype(np.int32),
        "v": rng.random(n),
        "ni": pd.array(np.where(rng.random(n) < 0.1, None, rng.integers(-5, 5, n)), dtype="Int64"),
        "nf": np.where(rng.random(n) < 0.1, np.nan, rng.random(n)),
        "b": rng.integers(0, 2, n).astype(bool),
    })


@pytest.mark.parametrize("persist", [True, False])
def test_create_table_from_arrow_buffers(c, persist):
    """pyarrow.Table -> device columns without a pandas detour: int32 widened, Arrow validity
    bitmaps used as they are (nullable ints stay ints instead of turning into float64 + NaN),
    NULL floats = NaN, multi-chunk and offset (sliced) inputs."""
    import pyarrow as pa
    df = _ingest_frame()
    t = pa.Table.from_pandas(df, preserve_index=False)
    chunked = pa.concat_tables([t.slice(0, 4001), t.slice(4001, 3), t.slice(4004)])      # 3 chunks per column
    c.create_table("t", chunked, persist=persist, npartitions=3)
    got = c.sql("SELECT k, SUM(v) AS sv, SUM(ni) AS sn, COUNT(ni) AS cn, AVG(nf) AS af, COUNT(*) AS n FROM t "
                "WHERE b GROUP BY k", return_futures=False)
    d = df[df["b"]]
    exp = d.groupby("k").agg(sv=("v", "sum"), sn=("ni", lambda s: s.sum(min_count=1)), cn=("ni", "count"),
                             af=("nf", "mean"), n=("k", "size")).reset_index()
    assert_same(got, exp, float_cols=("sv", "af"))
    # a slice with a non-byte-aligned offset
    c.create_table("s", t.slice(13, 5000), persist=persist)
    got = c.sql("SELECT SUM(ni) AS sn, COUNT(ni) AS cn, COUNT(*) AS n FROM s", return_futures=False)
    sl = df.iloc[13:5013]
    assert got["sn"].iloc[0] == sl["ni"].sum() and got["cn"].iloc[0] == sl["ni"].count() and got["n"].iloc[0] == 5000
    out = c.sql("SELECT ni, k FROM s WHERE ni IS NULL OR ni > 3", return_futures=False)
    assert str(out["ni"].dtype) == "Int64" and str(out["k"].dtype) == "int32"
    assert int(out["ni"].isna().sum()) == int(sl["ni"].isna().sum())


def test_parquet_and_csv_locations_and_ddl(c, tmp_path):
    """CREATE TABLE ... WITH (location=...), CREATE TABLE|VIEW ... AS, DROP TABLE
    (physical/rel/custom/create_table.py, create_memory_table.py, drop_table.py)."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    df = _ingest_frame(5_003, seed=4)
    pq_path, csv_path = str(tmp_path / "t.parquet"), str(tmp_path / "t.csv")
    pq.write_table(pa.Table.from_pandas(df, preserve_index=False), pq_path, row_group_size=1000)
    df[["k", "v"]].to_csv(csv_path, index=False)

    c.create_table("p", pq_path, persist=True, npartitions=2, columns=["k", "v", "ni"])
    assert c.sql("SELECT * FROM p").columns == ["k", "v", "ni"]
    c.sql(f"CREATE TABLE q WITH (location = '{pq_path}', format = 'parquet', persist = True)")
    c.sql(f"CREATE TABLE cs WITH (location = '{csv_path}')")
    exp = df.groupby("k").agg(s=("v", "sum")).reset_index()
    for name in ("p", "q", "cs"):
        got = c.sql(f"SELECT k, SUM(v) AS s FROM {name} GROUP BY k", return_futures=False)
        assert_same(got, exp, float_cols=("s",))

    with pytest.raises(RuntimeError):
        c.sql(f"CREATE TABLE q WITH (location = '{pq_path}')")                 # already present
    c.sql(f"CREATE TABLE IF NOT EXISTS q WITH (location = '{csv_path}')")       # silently kept
    assert "ni" in c.sql("SELECT * FROM q").columns

    # CREATE TABLE AS persists the result on the device; CREATE VIEW keeps the lazy frame
    c.sql("CREATE TABLE agg AS (SELECT k, SUM(v) AS s, COUNT(*) AS n FROM q WHERE v > 0.25 GROUP BY k)")
    c.sql("CREATE VIEW big AS SELECT k, v FROM q WHERE v > 0.25")
    from dask_sql_b200.frame import TableSource
    assert isinstance(c.schema["root"].tables["agg"].df.source, TableSource)
    assert not isinstance(c.schema["root"].tables["big"].df.source, TableSource) or c.schema["root"].tables["big"].df.pred
    d = df[df["v"] > 0.25]
    exp = d.groupby("k").agg(s=("v", "sum"), n=("k", "size")).reset_index()
    assert_same(c.sql("SELECT * FROM agg", return_futures=False), exp, float_cols=("s",))
    got = c.sql("SELECT a.k, a.n, SUM(b.v) AS s2 FROM agg a JOIN big b ON a.k = b.k GROUP BY a.k, a.n",
                return_futures=False)
    exp2 = exp.merge(d, on="k").groupby(["k", "n"]).agg(s2=("v", "sum")).reset_index()
    assert_same(got, exp2, float_cols=("s2",))
    c.sql("CREATE OR REPLACE TABLE agg AS SELECT k FROM q WHERE k < 3 GROUP BY k")
    assert sorted(c.sql("SELECT k FROM agg", return_futures=False)["k"].tolist()) == [0, 1, 2]

    c.sql("DROP TABLE agg")
    with pytest.raises(RuntimeError):
        c.sql("DROP TABLE agg")
    c.sql("DROP TABLE IF EXISTS agg")
    with pytest.raises(Exception):
        c.sql("SELECT * FROM agg")
    with pytest.raises(AttributeError):
        c.sql("CREATE TABLE nope WITH (format = 'parquet')")                    # location is mandatory


def test_lazy_parquet_pushdown_end_to_end(c, tmp_path):
    """Queries over a persist=False Parquet table read only the surviving row groups and still return
    exactly what pandas returns on the whole file (filter, group-by, join build side)."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    from dask_sql_b200 import executor
    n = 40_000
    rng = np.random.default_rng(17)
    df = pd.DataFrame({"a": np.arange(n), "k": rng.integers(0, 40, n), "v": rng.random(n),
                       "m": pd.array(np.where(rng.random(n) < 0.1, None, rng.integers(0, 9, n)), dtype="Int64")})
    path = str(tmp_path / "t.parquet")
    pq.write_table(pa.Table.from_pandas(df), path, row_group_size=4096)
    c.create_table("t", path)
    table = c.schema[c.schema_name].tables["t"].df.source.table
    before = executor.stats.get("rowgroups_skipped", 0)
    got = c.sql("SELECT k, SUM(v) AS s, COUNT(m) AS cm FROM t WHERE a >= 30000 AND a < 36000 GROUP BY k",
                return_futures=False)
    e = df[(df.a >= 30000) & (df.a < 36000)]
    exp = e.groupby("k").agg(s=("v", "sum"), cm=("m", "count")).reset_index()
    assert_same(got, exp, ["s"])
    assert executor.stats.get("rowgroups_skipped", 0) - before >= 7           # 10 row groups, at most 3 overlap
    assert not any(k[1] == "a" and k[0] < 7 for k in table._cache)            # early row groups never decoded
    got = c.sql("SELECT a, v FROM t WHERE a = 12345 OR a = 5", return_futures=False)   # OR: no pruning, same answer
    assert_same(got, df[(df.a == 12345) | (df.a == 5)][["a", "v"]], ["v"])
    c.create_table("d", pd.DataFrame({"k": np.arange(40), "w": np.arange(40) * 2.0}), persist=True)
    got = c.sql("SELECT d.w, SUM(t.v) AS s FROM t JOIN d ON t.k = d.k WHERE t.a < 5000 GROUP BY d.w",
                return_futures=False)
    e = df[df.a < 5000].merge(pd.DataFrame({"k": np.arange(40), "w": np.arange(40) * 2.0}), on="k")
    assert_same(got, e.groupby("w").agg(s=("v", "sum")).reset_index(), ["s"])


def test_modulo_is_floored_for_columns_and_constants(c):
    """SQL '%' is floored (the reference's da.mod, NumPy): the kernel on a column and the host's constant
    fold agree, -7 % 3 = 2; a zero divisor is NULL on both (DESIGN.md section 6).  Not sqlite: its % truncates."""
    a = np.array([-7, 7, -6, 5, 0, -1, 1, 2 ** 62 + 1, -(2 ** 63), 2 ** 63 - 1, 0], np.int64)
    null = np.zeros(len(a), bool)
    null[[4, 10]] = True
    df = pd.DataFrame({"a": pd.arrays.IntegerArray(a, null)})
    c.create_table("t", df, npartitions=2)
    got = c.sql("SELECT a, a % 3 AS m3, a % -3 AS mm3, -7 % a AS r, -7 % 3 AS k, 7 % -3 AS k2, a % 0 AS z, "
                "7 % 0 AS z2 FROM t", return_futures=False)
    av = np.where(null, 0, a)

    def col(v, null=null):
        return pd.array(np.where(null, None, v).tolist(), dtype="Int64")

    r = col(np.mod(-7, np.where(av == 0, 1, av)), null | (av == 0))
    exp = pd.DataFrame({"a": df["a"], "m3": col(np.mod(av, 3)), "mm3": col(np.mod(av, -3)), "r": r, "k": 2, "k2": -2,
                        "z": pd.array([None] * len(a), dtype="Int64"), "z2": pd.array([None] * len(a), dtype="Int64")})
    assert_same(got, exp)
    got = c.sql("SELECT a FROM t WHERE a % 3 = -7 % 3", return_futures=False)
    assert sorted(got["a"].tolist()) == sorted(int(x) for x, n in zip(a, null) if not n and x % 3 == 2)


def test_int_column_against_float_literal_at_2_53(c):
    """x = 9007199254740992.0 (2^53) compares in float64, where 2^53 + 1 rounds to 2^53, both as a lone
    conjunct (a kernel term) and inside an OR (the expression interpreter)"""
    x = np.array([2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, -(2 ** 53) - 1, 5, 2 ** 53 + 2], np.int64)
    y = pd.array([1, None, 2, 3, 4, 5], dtype="Int64")
    c.create_table("t", pd.DataFrame({"x": x, "y": y}))
    for lit, op in (("9007199254740992.0", "="), ("-9007199254740992.0", "="), ("9007199254740992.0", "<>"),
                    ("9007199254740992.0", "<"), ("9007199254740992.0", ">="), ("9007199254740993.0", ">")):
        hit = {"=": np.equal, "<>": np.not_equal, "<": np.less, ">=": np.greater_equal,
               ">": np.greater}[op](x.astype(np.float64), float(lit))
        alone = c.sql(f"SELECT x FROM t WHERE x {op} {lit}", return_futures=False)
        inside = c.sql(f"SELECT x FROM t WHERE x {op} {lit} OR y IS NULL", return_futures=False)
        assert sorted(alone["x"].tolist()) == sorted(x[hit].tolist()), (op, lit)
        assert sorted(inside["x"].tolist()) == sorted(x[hit | y.isna()].tolist()), (op, lit)


def test_order_by_float_edges(c):
    """ORDER BY over ±inf, ±0.0, subnormals, NaN and NULL: NaN sorts with the NULLs, -0.0 ties with 0.0"""
    rng = np.random.default_rng(12)
    n = 20_003
    f = rng.choice(np.array([np.inf, -np.inf, 0.0, -0.0, np.nan, 5e-324, -5e-324, 1.5, -1.5]), n)
    df = pd.DataFrame({"i": np.arange(n), "f": f})
    c.create_table("t", df, npartitions=3)
    for sql, asc, na in (("ORDER BY f", True, "last"), ("ORDER BY f DESC", False, "first"),
                         ("ORDER BY f NULLS FIRST", True, "first"), ("ORDER BY f DESC NULLS LAST", False, "last")):
        got = c.sql(f"SELECT i, f FROM t {sql}", return_futures=False)
        exp = df.sort_values("f", ascending=asc, na_position=na, kind="stable")
        np.testing.assert_array_equal(got["f"].to_numpy(), exp["f"].to_numpy(), err_msg=sql)   # -0.0 == 0.0 here
        assert sorted(got["i"].tolist()) == list(range(n)), sql
    got = c.sql("SELECT i, f FROM t ORDER BY f, i DESC", return_futures=False)
    exp = df.assign(z=df.f + 0.0).sort_values(["z", "i"], ascending=[True, False], na_position="last", kind="stable")
    np.testing.assert_array_equal(got["i"].to_numpy(), exp["i"].to_numpy())                 # ±0.0 tie: i decides


# ---- group-by edges: expected values from NumPy / fractions, not from pandas' summation ----------------------
def _groups(got, key):
    """{key (NaN -> None): row} of a GROUP BY result"""
    out = {}
    for r in got.to_dict("records"):            # per-column types: an int64 key stays an int
        k = r[key]
        out[None if pd.isna(k) else k] = r
    return out


def test_groupby_double_key_edges(c):
    """-0.0 and +0.0 are one group, NaN (any payload) and NULL are the NULL group, +-inf are groups of their own"""
    nan2 = np.array([0x7FF8000000000001], np.int64).view(np.float64)[0]
    keys = np.array([0.0, -0.0, np.nan, nan2, np.inf, -np.inf, 1.5, -0.0, np.inf, 2.5])
    null = np.zeros(len(keys), bool)
    null[9] = True                                  # a NULL next to the two NaN payloads
    rng = np.random.default_rng(1)
    reps = 3001
    df = pd.DataFrame({"f": np.tile(keys, reps), "v": rng.integers(-100, 100, len(keys) * reps)})
    df.loc[np.tile(null, reps), "f"] = None
    c.create_table("t", df, npartitions=3)
    got = _groups(c.sql("SELECT f, COUNT(*) AS n, SUM(v) AS s FROM t GROUP BY f", return_futures=False), "f")
    kk = np.tile(keys, reps)
    ident = np.where(np.isnan(kk) | np.tile(null, reps), np.nan, kk + 0.0)
    exp = {}
    for k in (0.0, np.inf, -np.inf, 1.5, None):
        sel = np.isnan(ident) if k is None else ident == k
        exp[k] = (int(sel.sum()), int(df.v.to_numpy()[sel].sum()))
    assert set(got) == set(exp), sorted(map(str, got))
    for k, (n, s) in exp.items():
        assert (got[k]["n"], got[k]["s"]) == (n, s), k


def test_groupby_boolean_key_with_nulls(c):
    rng = np.random.default_rng(2)
    n = 50_003
    b = rng.integers(0, 2, n).astype(bool)
    null = rng.random(n) < 0.1
    df = pd.DataFrame({"b": pd.array(np.where(null, None, b).tolist(), dtype="boolean"), "v": rng.integers(-9, 9, n)})
    c.create_table("t", df, npartitions=2)
    got = _groups(c.sql("SELECT b, COUNT(*) AS n, SUM(v) AS s FROM t GROUP BY b", return_futures=False), "b")
    v = df.v.to_numpy()
    exp = {True: ~null & b, False: ~null & ~b, None: null}
    assert set(got) == set(exp)
    for k, sel in exp.items():
        assert (got[k]["n"], got[k]["s"]) == (sel.sum(), v[sel].sum()), k


def test_groupby_bigint_extreme_keys_sum_wraps_and_avg_near_2_62(c):
    """keys INT64_MIN and INT64_MAX; per-group SUM wraps (two's complement), AVG near 2^62 is within the
    float-sum bound of the exact mean"""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    n = 30_001
    k = rng.choice(np.array([-(2 ** 63), 2 ** 63 - 1, 0, 5], np.int64), n)
    v = (2 ** 62 + rng.integers(-2 ** 40, 2 ** 40, n)).astype(np.int64)
    c.create_table("t", pd.DataFrame({"k": k, "v": v}), npartitions=3)
    got = _groups(c.sql("SELECT k, SUM(v) AS s, AVG(v) AS m, COUNT(*) AS n FROM t GROUP BY k", return_futures=False), "k")
    assert set(got) == {-(2 ** 63), 2 ** 63 - 1, 0, 5}
    for key, r in got.items():
        vs = [int(x) for x in v[k == key]]
        wrapped = (sum(vs) + 2 ** 63) % 2 ** 64 - 2 ** 63
        assert int(r["s"]) == wrapped and int(r["n"]) == len(vs), key
        exact = Fraction(sum(vs), len(vs))
        assert abs(Fraction(float(r["m"])) - exact) <= (len(vs) + 2) * 2.0 ** -53 * exact, key


def test_groupby_min_max_of_signed_zeros_infinities_and_subnormals(c):
    """MIN / MAX compare the order-preserving image: MIN{-0.0, +0.0} = -0.0 and MAX = +0.0, whatever came first"""
    groups = {1: [0.0, -0.0], 2: [-0.0, 0.0], 3: [5e-324, -5e-324, 0.0], 4: [np.inf, -np.inf, 1.0],
              5: [np.nan, -0.0, None], 6: [None, None]}
    rows = [(k, x) for k, xs in groups.items() for x in xs]
    df = pd.DataFrame({"k": [r[0] for r in rows], "x": pd.array([r[1] for r in rows], dtype="Float64")})
    df["x"] = df["x"].astype("float64")
    c.create_table("t", df, npartitions=2)
    got = _groups(c.sql("SELECT k, MIN(x) AS lo, MAX(x) AS hi FROM t GROUP BY k", return_futures=False), "k")
    exp = {1: (-0.0, 0.0), 2: (-0.0, 0.0), 3: (-5e-324, 5e-324), 4: (-np.inf, np.inf), 5: (-0.0, -0.0), 6: (None, None)}
    for k, (lo, hi) in exp.items():
        for name, e in (("lo", lo), ("hi", hi)):
            g = got[k][name]
            if e is None:
                assert pd.isna(g), (k, name, g)
            else:
                assert g == e and np.signbit(g) == np.signbit(e), (k, name, g, e)


def test_groupby_variance_against_the_exact_two_pass_value(c):
    """VAR_SAMP / STDDEV on N(1e9, 1) with groups of one and two rows and NULLs, against the exact variance"""
    from fractions import Fraction
    rng = np.random.default_rng(4)
    n = 20_000
    k = rng.integers(0, 20, n)
    k[:3] = [100, 101, 101]                       # a group of one row and one of two
    x = 1e9 + rng.normal(0, 1, n)
    x[rng.random(n) < 0.05] = np.nan
    x[:3] = [1e9 + 0.5, 1e9 + 0.25, 1e9 - 0.75]
    df = pd.DataFrame({"k": k, "x": x})
    c.create_table("t", df, npartitions=3)
    got = _groups(c.sql("SELECT k, VAR_SAMP(x) AS v, STDDEV(x) AS s FROM t GROUP BY k", return_futures=False), "k")
    for key, r in got.items():
        xs = [Fraction(float(a)) for a in x[(k == key) & ~np.isnan(x)]]
        if len(xs) < 2:
            assert pd.isna(r["v"]) and pd.isna(r["s"]), key
            continue
        mean = sum(xs) / len(xs)
        var = float(sum((a - mean) ** 2 for a in xs) / (len(xs) - 1))
        np.testing.assert_allclose([r["v"], r["s"]], [var, np.sqrt(var)], rtol=1e-9, err_msg=str(key))


def test_groupby_skewed_key_whose_hottest_key_is_filtered_out(c, monkeypatch):
    """Zipf keys under the heavy-hitter kernel: the hottest key is sampled (from the unfiltered column) but every
    one of its rows fails the WHERE clause, and the never-NULL float SUM is the group's only existence mark:
    the group must not appear"""
    from dask_sql_b200 import executor
    monkeypatch.setenv("B200SQL_SKEW", "hot")
    rng = np.random.default_rng(5)
    n = 400_003
    k = np.minimum(rng.zipf(1.2, n), 5000).astype(np.int64)
    f = rng.integers(-1, 2 ** 10, n) * 2.0 ** -4
    f[k == 1] = -1.0                               # key 1 holds ~1/3 of the rows, all filtered
    v = rng.integers(-2 ** 10, 2 ** 10, n) * 2.0 ** -8
    c.create_table("t", pd.DataFrame({"k": k, "f": f, "v": v}), npartitions=2)
    before = executor.stats.get("grouped_groupby", 0)
    got = _groups(c.sql("SELECT k, SUM(v) AS s FROM t WHERE f >= 0 GROUP BY k", return_futures=False), "k")
    assert executor.stats.get("grouped_groupby", 0) > before, "the skew path did not run"
    keep = f >= 0
    assert 1 not in got
    assert set(got) == set(np.unique(k[keep]).tolist())
    sums = {}
    for key, val in zip(k[keep].tolist(), v[keep].tolist()):
        sums[key] = sums.get(key, 0.0) + val       # dyadic values: every order gives the same sum
    for key, r in got.items():
        assert r["s"] == sums[key], key
