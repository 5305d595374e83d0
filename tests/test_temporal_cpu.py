"""DATE / TIMESTAMP on the host: parsing, binding, literal rounding onto a column's unit, fused-scan terms,
the YEAR / CAST AS DATE rewrite, Parquet statistics and constant folding.  No kernel is launched."""
import datetime

import numpy as np
import pandas as pd
import pytest

from tests import temporal_ref as R


def _ctx():
    import pyarrow as pa
    from dask_sql_b200 import Context
    c = Context()
    c.create_table("t", pa.table({
        "ts": pa.array(np.array([0, 10 ** 6, -1], dtype="datetime64[us]")),
        "tn": pa.array(np.array([0, 5, 7], dtype="datetime64[ns]")),
        "d": pa.array(np.array(["1995-03-14", "1995-03-15", "1996-01-01"], dtype="datetime64[D]"), pa.date32()),
        "v": [1.0, 2.0, 3.0]}))
    return c


def test_parse_literals():
    from dask_sql_b200 import temporal as T
    assert T.parse_date("1995-03-15").ticks == int(np.datetime64("1995-03-15", "D").astype(np.int64))
    ts = T.parse_timestamp("2021-10-03 15:53:42.000047")
    assert (ts.unit, ts.ticks) == ("us", int(np.datetime64("2021-10-03T15:53:42.000047", "us").astype(np.int64)))
    assert T.parse_timestamp("2000-01-01 00:00:00.123456789").unit == "ns"
    iv = T.parse_interval("1 year 2 months 3 days")
    assert (iv.months, iv.ns) == (14, 3 * T.NS_PER_DAY)
    assert T.parse_interval("4", "DAY").ns == 4 * T.NS_PER_DAY
    for bad in ("1995-02-30", "1995-13-01", "yesterday"):
        with pytest.raises(ValueError):
            T.parse_date(bad)


def test_sql_reaches_lazy_frames_with_date_columns():
    from dask_sql_b200.frame import LazyFrame
    c = _ctx()
    for q in ["SELECT ts, d FROM t WHERE d > DATE '1995-03-14'",
              "SELECT y, SUM(v) AS s FROM (SELECT EXTRACT(YEAR FROM ts) AS y, v FROM t) AS q GROUP BY y",
              "SELECT d + INTERVAL '1' MONTH AS m, ts - INTERVAL '2 hours' AS h, LAST_DAY(d) AS l FROM t",
              "SELECT TIMESTAMPADD(DAY, 3, ts) AS a, TIMESTAMPDIFF(MONTH, d, ts) AS b FROM t",
              "SELECT FLOOR(ts TO HOUR) AS f, CEIL(tn TO SECOND) AS c, CAST(ts AS DATE) AS cd FROM t",
              "SELECT MIN(d) AS lo, MAX(ts) AS hi, COUNT(DISTINCT d) AS n FROM t",
              "SELECT * FROM t WHERE d BETWEEN '1995-01-01' AND '1995-12-31' AND ts IN ('1970-01-01 00:00:01')",
              "SELECT d, DATE_PART('dow', d) AS w, YEAR(d) AS y FROM t ORDER BY d DESC NULLS FIRST"]:
        assert isinstance(c.sql(q), LazyFrame), q
    lf = c.sql("SELECT d, ts FROM t")
    assert str(lf.dtypes["d"]) == "datetime64[D]" and str(lf.dtypes["ts"]) == "datetime64[us]"


def test_unsupported_temporal_forms_raise():
    c = _ctx()
    with pytest.raises(NotImplementedError):
        c.sql("SELECT SUM(d) FROM t")
    with pytest.raises(NotImplementedError):
        c.sql("SELECT AVG(ts) FROM t")
    with pytest.raises(NotImplementedError, match="TIMESTAMPDIFF"):
        c.sql("SELECT ts - tn FROM t")
    with pytest.raises(NotImplementedError):
        c.sql("SELECT FLOOR(ts TO YEAR) FROM t")
    from dask_sql_b200.utils import ParsingException
    with pytest.raises(ParsingException):
        c.sql("SELECT * FROM t WHERE d > DATE '1995-02-30'")
    with pytest.raises(ParsingException):
        c.sql("SELECT * FROM t WHERE d > 'not a date'")
    from dask_sql_b200 import Context
    with pytest.raises(NotImplementedError):
        Context().create_table("z", pd.DataFrame({"t": pd.date_range("2020-01-01", periods=3, tz="UTC")}))
    with pytest.raises(NotImplementedError):
        Context().create_table("z", pd.DataFrame({"t": pd.to_timedelta([1, 2], unit="s")}))


def _terms(c, q):
    from dask_sql_b200 import expr as E
    lf = c.sql(q)
    return [E.as_term(p) for p in lf.pred]


def test_date_comparisons_are_fused_terms_on_the_columns_own_unit():
    from dask_sql_b200 import _lib as L
    c = _ctx()
    day = int(np.datetime64("1995-03-15", "D").astype(np.int64))
    assert _terms(c, "SELECT v FROM t WHERE d < DATE '1995-03-15'") == [("d", L.LT, day)]
    assert _terms(c, "SELECT v FROM t WHERE ts >= DATE '1995-03-15'") == [("ts", L.GE, day * 86400 * 10 ** 6)]
    assert _terms(c, "SELECT v FROM t WHERE '1995-03-15' > d") == [("d", L.LT, day)]


def test_literal_rounding_onto_a_coarser_column():
    """d (days) > TIMESTAMP '1995-03-15 12:00' keeps d >= 1995-03-16: a fused term on the DATE bytes."""
    from dask_sql_b200 import _lib as L
    c = _ctx()
    day = int(np.datetime64("1995-03-15", "D").astype(np.int64))
    assert _terms(c, "SELECT v FROM t WHERE d > TIMESTAMP '1995-03-15 12:00:00'") == [("d", L.GT, day)]
    assert _terms(c, "SELECT v FROM t WHERE d >= TIMESTAMP '1995-03-15 12:00:00'") == [("d", L.GE, day + 1)]
    assert _terms(c, "SELECT v FROM t WHERE d < TIMESTAMP '1995-03-15 12:00:00'") == [("d", L.LT, day + 1)]
    assert _terms(c, "SELECT v FROM t WHERE d <= TIMESTAMP '1995-03-15 12:00:00'") == [("d", L.LE, day)]
    assert _terms(c, "SELECT v FROM t WHERE d >= TIMESTAMP '1995-03-15 00:00:00'") == [("d", L.GE, day)]
    # '=' with an inexact literal scales the column instead: no fused term, and no row can match
    assert _terms(c, "SELECT v FROM t WHERE d = TIMESTAMP '1995-03-15 12:00:00'") == [None]


def test_year_and_cast_as_date_become_ranges():
    from dask_sql_b200 import _lib as L
    c = _ctx()
    y95 = int(np.datetime64("1995-01-01", "D").astype(np.int64))
    y96 = int(np.datetime64("1996-01-01", "D").astype(np.int64))
    us = 86400 * 10 ** 6
    assert _terms(c, "SELECT v FROM t WHERE YEAR(ts) = 1995") == [("ts", L.GE, y95 * us), ("ts", L.LT, y96 * us)]
    assert _terms(c, "SELECT v FROM t WHERE EXTRACT(YEAR FROM d) < 1996") == [("d", L.LT, y96)]
    assert _terms(c, "SELECT v FROM t WHERE EXTRACT(YEAR FROM d) BETWEEN 1995 AND 1995") == \
        [("d", L.GE, y95), ("d", L.LT, y96)]
    day = int(np.datetime64("1995-03-15", "D").astype(np.int64))
    assert _terms(c, "SELECT v FROM t WHERE CAST(ts AS DATE) = DATE '1995-03-15'") == \
        [("ts", L.GE, day * us), ("ts", L.LT, (day + 1) * us)]
    assert _terms(c, "SELECT v FROM t WHERE CAST(tn AS DATE) > '1995-03-15'") == \
        [("tn", L.GE, (day + 1) * 86400 * 10 ** 9)]
    assert _terms(c, "SELECT v FROM t WHERE YEAR(ts) <> 1995") == [None]      # <> stays in the interpreter


def test_constant_folding_uses_the_calendar_rules():
    c = _ctx()
    from dask_sql_b200 import temporal as T
    lf = c.sql("SELECT DATE '1998-08-18' - INTERVAL '4 days' AS b, DATE '2000-01-31' + INTERVAL '1' MONTH AS m, "
               "TIMESTAMPDIFF(DAY, DATE '2000-01-01', DATE '2000-03-01') AS n, "
               "LAST_DAY(DATE '2000-02-10') AS l, EXTRACT(WEEK FROM DATE '2021-01-03') AS w FROM t")
    got = {n: lf.exprs[n] for n in lf.columns}
    day = lambda s: int(np.datetime64(s, "D").astype(np.int64))  # noqa: E731
    assert got["b"].value == day("1998-08-14") and got["b"].logical == T.DATE_LOGICAL
    assert got["m"].value == day("2000-02-29")
    assert got["n"].value == 60
    assert got["l"].value == day("2000-02-29")
    assert got["w"].value == 53


def test_host_fold_matches_reference():
    from dask_sql_b200 import temporal as T
    rng = np.random.default_rng(3)
    for unit in ("D", "s", "ms", "us", "ns"):
        lim = 3_000_000 if unit == "D" else 10 ** 17 // max(1, 10 ** 9 // T.TPS[unit])
        for x in rng.integers(-lim, lim, 200).tolist():
            for f in T.FIELDS:
                assert T.datepart(x, f, unit) == int(R.datepart(np.array([x]), f, unit)[0]), (x, f, unit)
            n = int(rng.integers(-30, 30))
            assert T.add_months(x, n, unit) == int(R.add_months(np.array([x]), n, unit)[0])
            assert T.add_months(x, n, unit, True) == int(R.add_months(np.array([x]), n, unit, True)[0])


def test_parquet_statistics_of_temporal_columns(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq
    from dask_sql_b200 import _lib as L
    from dask_sql_b200.table import ParquetTable
    days = np.arange(np.datetime64("1995-01-01"), np.datetime64("1995-01-01") + 400).astype("datetime64[D]")
    t = pa.table({"d": pa.array(days, pa.date32()),
                  "ts": pa.array(days.astype("datetime64[ms]"), pa.timestamp("ms")),
                  "v": np.arange(400, dtype=np.float64)})
    path = str(tmp_path / "dates.parquet")
    pq.write_table(t, path, row_group_size=100)
    pt = ParquetTable(path)
    d0 = int(days[0].astype(np.int64))
    st = pt.column_stats("d")
    assert (st.vmin, st.vmax) == (d0, d0 + 399)
    assert pt.column_stats("ts").vmax == (d0 + 399) * 86400 * 1000
    assert pt.surviving_groups([("d", L.GE, d0 + 350)]) == [3]
    assert pt.surviving_groups([("ts", L.LT, (d0 + 150) * 86400 * 1000)]) == [0, 1]
    assert [s for n, _, s in pt.schema()] == ["date32[day]", "datetime64[ms]", "float64"]


def test_arrow_temporal_inputs():
    import pyarrow as pa
    from dask_sql_b200.table import arrow_columns
    cols = arrow_columns(pa.table({
        "a": pa.array([0, None, -1], pa.date32()),
        "b": pa.array([86_400_000, 0, None], pa.date64()),
        "c": pa.array([1, 2, None], pa.timestamp("ns"))}))
    assert cols["a"].logical == "date32[day]" and cols["a"].values.tolist()[::2] == [0, -1]
    assert cols["b"].logical == "date32[day]" and cols["b"].values.tolist()[:2] == [1, 0]
    assert cols["c"].logical == "datetime64[ns]" and cols["c"].valid_words() is not None
    for bad in (pa.array([1], pa.timestamp("us", tz="UTC")), pa.array([1], pa.time64("us")),
                pa.array([1], pa.duration("s"))):
        with pytest.raises(NotImplementedError):
            arrow_columns(pa.table({"x": bad}))


def test_calendar_program_compiles_to_the_new_opcodes():
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import expr as E
    from dask_sql_b200 import temporal as T
    x = E.ColRef("x", E.I64, "datetime64[ms]")
    p = E.compile_expr(T.extract("QUARTER", x), ["x"])
    assert [(p.code[i].op, p.code[i].a, p.code[i].imm_i) for i in range(p.n)] == \
        [(L.OP_LOAD, 0, 0), (L.OP_DATEPART, L.DP_QUARTER, 1000)]
    p = E.compile_expr(T.add_months_expr(x, 0, to_last=True), ["x"])
    assert [(p.code[i].op, p.code[i].a) for i in range(p.n)] == [(L.OP_LOAD, 0), (L.OP_CONST_I, 0), (L.OP_ADDMONTHS, 1)]
    assert datetime.date(2000, 2, 29) == (datetime.date(1970, 1, 1) +
                                          datetime.timedelta(days=T.add_months(T.parse_date("2000-02-03").ticks, 0, "D", True)))


def test_literal_beyond_the_columns_int64_range_keeps_the_comparison():
    """DATE '9999-12-31' in nanoseconds is past INT64_MAX (and 0001-01-01 before INT64_MIN): the comparison
    is then the same for every non-NULL row of a datetime64[ns] column, a term against INT64_MAX / MIN."""
    from dask_sql_b200 import _lib as L
    c = _ctx()
    hi, lo = (1 << 63) - 1, -(1 << 63)
    for q, want in [("tn < DATE '9999-12-31'", ("tn", L.LE, hi)), ("tn <= DATE '9999-12-31'", ("tn", L.LE, hi)),
                    ("tn <> DATE '9999-12-31'", ("tn", L.LE, hi)), ("tn > DATE '9999-12-31'", ("tn", L.GT, hi)),
                    ("tn >= DATE '9999-12-31'", ("tn", L.GT, hi)), ("tn = DATE '9999-12-31'", ("tn", L.GT, hi)),
                    ("DATE '9999-12-31' > tn", ("tn", L.LE, hi)),
                    ("tn > DATE '0001-01-01'", ("tn", L.GE, lo)), ("tn >= DATE '0001-01-01'", ("tn", L.GE, lo)),
                    ("tn <> DATE '0001-01-01'", ("tn", L.GE, lo)), ("tn < DATE '0001-01-01'", ("tn", L.LT, lo)),
                    ("tn <= DATE '0001-01-01'", ("tn", L.LT, lo)), ("tn = DATE '0001-01-01'", ("tn", L.LT, lo)),
                    ("tn BETWEEN DATE '0001-01-01' AND DATE '9999-12-31'", None)]:
        got = _terms(c, f"SELECT v FROM t WHERE {q}")
        if want is None:
            assert got == [("tn", L.GE, lo), ("tn", L.LE, hi)], q
        else:
            assert got == [want], q
    # the same literals on a microsecond column fit and stay exact
    us = int(np.datetime64("9999-12-31", "D").astype(np.int64)) * 86400 * 10 ** 6
    assert _terms(c, "SELECT v FROM t WHERE ts < DATE '9999-12-31'") == [("ts", L.LT, us)]


def test_cast_of_a_date_to_bigint_is_its_ticks():
    c = _ctx()
    lf = c.sql("SELECT CAST(d AS BIGINT) AS x, CAST(ts AS BIGINT) AS y, CAST(DATE '1970-01-11' AS BIGINT) AS z FROM t")
    assert [lf.exprs[n].logical for n in ("x", "y")] == ["int64", "int64"]
    assert str(lf.dtypes["x"]) == "int64" and lf.exprs["z"].value == 10
    assert len(_terms(c, "SELECT v FROM t WHERE CAST(d AS BIGINT) = 9204")) == 1     # an int64 comparison
