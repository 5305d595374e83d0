"""ANALYZE TABLE ... COMPUTE STATISTICS end to end on the GPU, against pandas describe() of the same data: the
reference's test_analyze (dask_sql tests/integration/test_analyze.py) restated, then seeded tables that mix
BIGINT, DOUBLE with NaN and NULL, BOOLEAN, DATE, TIMESTAMP and VARCHAR over 1 and 8 partitions and as a lazy
Parquet table, empty and all-NULL columns, n = 1, and the select's pass count.

count, min, max and the quantiles must equal describe()'s exactly.  mean and std are bounded against the exact
values the way the aggregate tests bound AVG / STDDEV_SAMP (tests/groupagg_ref.py, tests/query_ref.py)."""
import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from tests import groupagg_ref as G
from tests import query_ref as Q
from tests import select_ref as R

pytestmark = pytest.mark.gpu

INDEX = ["count", "mean", "std", "min", "25%", "50%", "75%", "max", "data_type", "col_name"]
U = 2.0 ** -53


def _ctx():
    import torch
    torch.cuda.set_device(0)
    from dask_sql_b200 import Context
    return Context()


def _expected(c, table, cols=None):
    """the reference's frame: describe() of the table's rows, then the data_type and col_name rows"""
    from dask_sql_b200.mappings import python_to_sql_type
    host = c.sql(f"SELECT * FROM {table}").compute()
    cols = list(host.columns) if cols is None else cols
    dtypes = c.schema["root"].tables[table].df.dtypes
    exp = pd.concat([host[cols].describe(),
                     pd.DataFrame({k: str(python_to_sql_type(dtypes[k])).lower() for k in cols}, index=["data_type"]),
                     pd.DataFrame({k: k for k in cols}, index=["col_name"])])
    return exp, host


def _sql_type(dtype):
    from dask_sql_b200.mappings import python_to_sql_type
    return str(python_to_sql_type(dtype)).lower()


def _mean_bound(x):
    e, b = G.exact_sum(x), G.sum_bound(x)
    return e / len(x), b / len(x) + U * abs(e / len(x))


def _std_bound(x):
    xs = [Fraction(float(v)) for v in x]
    m = len(xs)
    mean = sum(xs) / m
    ss = sum((v - mean) ** 2 for v in xs)
    sd = math.sqrt(float(ss / (m - 1)))
    b = Q.moment_bound(ss, m, float(np.max(x) - np.min(x)), m - 1)
    return sd, (b / sd if sd > 0 else math.sqrt(b)) + 2 * U * sd


def _compare(got, exp, host):
    assert isinstance(got, pd.DataFrame)
    assert list(got.index) == INDEX
    assert list(got.columns) == list(exp.columns)
    for col in got.columns:
        for row in ("count", "min", "25%", "50%", "75%", "max", "data_type", "col_name"):
            g = got.at[row, col]
            e = exp.at[row, col] if row in exp.index else np.nan
            if pd.isna(e):
                assert pd.isna(g), (col, row, g)
            else:
                assert g == e, (col, row, g, e)
        g_mean, g_std = got.at["mean", col], got.at["std", col]
        s = host[col]
        if pd.isna(exp.at["count", col]) or not exp.at["count", col]:
            assert pd.isna(g_mean) and pd.isna(g_std), col
            continue
        if isinstance(g_mean, pd.Timestamp):
            unit = np.datetime_data(s.dropna().to_numpy().dtype)[0]
            ticks = s.dropna().to_numpy().astype(f"M8[{unit}]").astype(np.int64).astype(np.float64)
            e, b = _mean_bound(ticks)
            g = np.datetime64(g_mean, unit).astype(np.int64)
            assert abs(g - e) <= b + 1, (col, g_mean, e, b)          # + 1: the mean truncates to a tick
            assert pd.isna(g_std)
            continue
        x = s.dropna().to_numpy(dtype=np.float64)
        e, b = _mean_bound(x)
        assert abs(g_mean - e) <= b, (col, g_mean, e, b)
        if len(x) < 2:
            assert pd.isna(g_std)
        else:
            e, b = _std_bound(x)
            assert abs(g_std - e) <= b, (col, g_std, e, b)


def test_reference_analyze():
    """test_analyze of the reference on its `df` fixture, for ALL COLUMNS and for COLUMNS a"""
    np.random.seed(42)
    df = pd.DataFrame({"a": [1.0] * 100 + [2.0] * 200 + [3.0] * 400, "b": 10 * np.random.rand(700)})
    c = _ctx()
    c.create_table("df", df)
    got = c.sql("ANALYZE TABLE df COMPUTE STATISTICS FOR ALL COLUMNS")
    exp, host = _expected(c, "df")
    _compare(got, exp, host)
    assert got.loc["data_type"].tolist() == [_sql_type("float64")] * 2 and got.loc["col_name"].tolist() == ["a", "b"]
    got = c.sql("ANALYZE TABLE df COMPUTE STATISTICS FOR COLUMNS a", return_futures=False)
    _compare(got, exp[["a"]], host)


def _mixed_table(n, seed):
    rng = np.random.default_rng(seed)
    null = rng.random(n) < 0.1
    f = rng.standard_normal(n) * 100
    f[rng.random(n) < 0.05] = np.nan
    day0 = np.datetime64("1990-01-01", "D").astype(np.int64)
    return pa.table({
        "i": pa.array(rng.integers(-10 ** 6, 10 ** 6, n), mask=null),
        "big": pa.array(rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64)),
        "f": pa.array(f, from_pandas=True),
        "fn": pa.array(rng.random(n), mask=rng.random(n) < 0.2),
        "flag": pa.array(rng.random(n) < 0.5),
        "d": pa.array((day0 + rng.integers(0, 20_000, n)).astype("datetime64[D]"), pa.date32()),
        "ts": pa.array(rng.integers(0, 2 * 10 ** 18, n).astype("datetime64[ns]"), mask=rng.random(n) < 0.1),
        "s": pa.array(rng.choice(["x", "yy", "zzz"], n)).dictionary_encode(),
        "dup": pa.array(np.repeat(np.arange(4, dtype=np.int64), -(-n // 4))[:n]),
    })


@pytest.mark.parametrize("nparts", [1, 8])
def test_mixed_types(nparts):
    c = _ctx()
    c.create_table("t", _mixed_table(3001, nparts), npartitions=nparts)
    got = c.sql("ANALYZE TABLE t COMPUTE STATISTICS FOR ALL COLUMNS")
    exp, host = _expected(c, "t")
    _compare(got, exp, host)
    # described columns first, BOOLEAN / VARCHAR after them, in table order
    assert list(got.columns) == ["i", "big", "f", "fn", "d", "ts", "dup", "flag", "s"]
    assert got.at["data_type", "d"] == _sql_type("datetime64[D]")
    assert got.at["data_type", "ts"] == _sql_type("datetime64[ns]")
    assert all(pd.isna(got.at[r, "flag"]) and pd.isna(got.at[r, "s"]) for r in INDEX[:8])
    cols = ["s", "ts", "f", "flag", "i"]
    got = c.sql("ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS s, ts, f, flag, i")
    exp, host = _expected(c, "t", cols)
    _compare(got, exp, host)
    assert list(got.columns) == ["ts", "f", "i", "s", "flag"]


def test_lazy_parquet_table(tmp_path):
    import pyarrow.parquet as pq
    path = str(tmp_path / "t.parquet")
    pq.write_table(_mixed_table(2500, 3), path, row_group_size=700)
    c = _ctx()
    c.create_table("p", path, persist=False)
    got = c.sql("ANALYZE TABLE p COMPUTE STATISTICS FOR ALL COLUMNS")
    exp, host = _expected(c, "p")
    _compare(got, exp, host)


def test_empty_all_null_and_single_row():
    c = _ctx()
    c.create_table("e", pd.DataFrame({"x": np.array([], np.float64), "k": np.array([], np.int64)}))
    got = c.sql("ANALYZE TABLE e COMPUTE STATISTICS FOR ALL COLUMNS")
    exp, host = _expected(c, "e")
    _compare(got, exp, host)
    assert got.at["count", "x"] == 0 and all(pd.isna(got.at[r, "x"]) for r in INDEX[1:8])
    c.create_table("z", pd.DataFrame({"x": [np.nan] * 40, "k": pd.array([None] * 40, dtype="Int64"),
                                      "v": np.arange(40.0)}), npartitions=2)
    got = c.sql("ANALYZE TABLE z COMPUTE STATISTICS FOR ALL COLUMNS")
    exp, host = _expected(c, "z")
    _compare(got, exp, host)
    c.create_table("one", pd.DataFrame({"x": [2.5], "k": [-7], "t": pd.to_datetime(["2001-02-03 04:05:06"])}))
    got = c.sql("ANALYZE TABLE one COMPUTE STATISTICS FOR ALL COLUMNS")
    exp, host = _expected(c, "one")
    _compare(got, exp, host)


def test_all_boolean_or_varchar_keeps_the_shape():
    c = _ctx()
    c.create_table("bv", pa.table({"flag": pa.array([True, False, True]),
                                   "s": pa.array(["a", "b", "a"]).dictionary_encode()}))
    got = c.sql("ANALYZE TABLE bv COMPUTE STATISTICS FOR ALL COLUMNS")
    assert list(got.index) == INDEX and list(got.columns) == ["flag", "s"]
    assert all(pd.isna(got.at[r, k]) for r in INDEX[:8] for k in ("flag", "s"))
    assert got.loc["data_type"].tolist() == [_sql_type("bool"), _sql_type("category")]


def test_pass_count_follows_the_min_max_images():
    from dask_sql_b200 import executor as X
    from dask_sql_b200._lib import F64, I64
    rng = np.random.default_rng(8)
    n = 200_000
    key = rng.integers(0, 1 << 20, n)
    val = rng.random(n)
    const = np.full(n, 5, np.int64)
    c = _ctx()
    c.create_table("c2", pd.DataFrame({"key": key, "val": val, "const": const}), npartitions=8)
    want = sum(R.passes(X.select_image(lo, dt), X.select_image(hi, dt))
               for lo, hi, dt in ((key.min(), key.max(), I64), (val.min(), val.max(), F64), (5, 5, I64)))
    assert R.passes(X.select_image(key.min(), I64), X.select_image(key.max(), I64)) == 2
    before = X.stats.get("select_passes", 0)
    got = c.sql("ANALYZE TABLE c2 COMPUTE STATISTICS FOR ALL COLUMNS")
    assert X.stats["select_passes"] - before == want
    exp, host = _expected(c, "c2")
    _compare(got, exp, host)
