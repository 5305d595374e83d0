"""DATE / TIMESTAMP end to end through Context.sql() on the GPU: known answers of the reference's temporal
tests (dask_sql tests/integration/test_rex.py), round trips of every unit, GROUP BY / JOIN / ORDER BY on
dates, the Q3 shape on DATE columns (fused star join, no interpreter launch for its predicates) and
Parquet row-group pruning on a date-sorted file."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from tests.golden import reference_temporal as G

pytestmark = pytest.mark.gpu


def _ctx():
    import torch
    torch.cuda.set_device(0)
    from dask_sql_b200 import Context
    return Context()



@pytest.mark.parametrize("case", G.CASES, ids=[c["where"] for c in G.CASES])
def test_reference_golden_case(case):
    """Every DATE / TIMESTAMP known answer transcribed in tests/golden/reference_temporal.py."""
    c = _ctx()
    for name, cols in case["tables"].items():
        c.create_table(name, pd.DataFrame({k: pd.Series(np.array(v, dtype=dt)) for k, (v, dt) in cols.items()}))
    if "raises" in case:
        with pytest.raises({"NotImplementedError": NotImplementedError}[case["raises"]]):
            c.sql(case["sql"]).compute()
        return
    got = c.sql(case["sql"]).compute()
    for col, want in case["expected"].items():
        vals = got[col].tolist()
        assert len(vals) == len(want), (col, vals)
        for g, w in zip(vals, want):
            if isinstance(w, str):
                assert pd.Timestamp(g) == pd.Timestamp(w), (col, g, w)
            else:
                assert int(g) == w, (col, g, w)


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
def test_pandas_round_trip_with_nat(unit):
    c = _ctx()
    s = pd.Series(np.array(["1969-12-31T23:59:59", "NaT", "2262-01-01", "1677-12-31", "2000-02-29T12:00:00"],
                           dtype=f"datetime64[{unit}]"))
    c.create_table("t", pd.DataFrame({"x": s, "k": np.arange(5)}))
    got = c.sql("SELECT x, k FROM t").compute()
    assert got["x"].dtype == np.dtype(f"datetime64[{unit}]")
    np.testing.assert_array_equal(got["x"].to_numpy(), s.to_numpy())
    got = c.sql("SELECT k FROM t WHERE x IS NULL").compute()
    assert got["k"].tolist() == [1]


def test_arrow_date_round_trip_and_group_by():
    from dask_sql_b200 import executor
    c = _ctx()
    rng = np.random.default_rng(0)
    days = rng.integers(9000, 9400, 50_000)
    c.create_table("t", pa.table({"d": pa.array(days.astype("datetime64[D]"), pa.date32()),
                                  "v": rng.random(50_000)}), persist=True)
    before = executor.stats["dense_groupby"]
    got = c.sql("SELECT d, SUM(v) AS s, COUNT(*) AS n FROM t GROUP BY d").compute().sort_values("d")
    assert executor.stats["dense_groupby"] > before
    want = pd.DataFrame({"d": days, "v": 0}).groupby("d").size()
    assert got["n"].tolist() == want.tolist()
    assert got["d"].dtype == np.dtype("datetime64[s]")
    assert got["d"].to_numpy().astype("datetime64[D]").astype(np.int64).tolist() == want.index.tolist()
    y = c.sql("SELECT y, COUNT(*) AS n FROM (SELECT EXTRACT(YEAR FROM d) AS y FROM t) AS q GROUP BY y").compute()
    yy = pd.Series(days.astype("datetime64[D]")).dt.year.value_counts()
    assert dict(zip(y["y"].tolist(), y["n"].tolist())) == yy.to_dict()
    mm = c.sql("SELECT MIN(d) AS lo, MAX(d) AS hi, COUNT(DISTINCT d) AS nd FROM t").compute()
    assert mm["lo"].iloc[0] == np.datetime64(int(days.min()), "D") and int(mm["nd"].iloc[0]) == len(set(days.tolist()))
    o = c.sql("SELECT d FROM t ORDER BY d DESC LIMIT 3").compute()
    assert o["d"].to_numpy().astype("datetime64[D]").astype(np.int64).tolist() == sorted(days.tolist())[::-1][:3]


def test_join_on_dates_of_two_units_and_ctas():
    c = _ctx()
    days = np.array(["2000-01-01", "2000-01-02", "2000-01-03", "NaT"], dtype="datetime64[D]")
    c.create_table("a", pa.table({"d": pa.array(days, pa.date32()), "x": [1, 2, 3, 4]}))
    c.create_table("b", pd.DataFrame({"t": pd.Series(days.astype("datetime64[ms]")), "y": [10, 20, 30, 40]}))
    got = c.sql("SELECT x, y FROM a JOIN b ON a.d = b.t").compute().sort_values("x")
    assert got["x"].tolist() == [1, 2, 3] and got["y"].tolist() == [10, 20, 30]
    c.sql("CREATE TABLE c AS SELECT d, x FROM a WHERE d >= DATE '2000-01-02'")
    r = c.sql("SELECT d, x FROM c ORDER BY d NULLS FIRST").compute()
    assert r["x"].tolist() == [2, 3]
    assert c.sql("SELECT d FROM c").dtypes["d"] == np.dtype("datetime64[D]")


def _q3_tables(n_dim=20_000, n_fact=400_000, seed=4):
    rng = np.random.default_rng(seed)
    base = int(np.datetime64("1992-01-01", "D").astype(np.int64))
    odate = base + rng.integers(0, 2400, n_dim)
    otime = odate * 86_400_000_000 + rng.integers(0, 86_400_000_000, n_dim)      # the same orders, in us
    ship = base + rng.integers(0, 2400, n_fact)
    dim = {"pk": rng.permutation(n_dim).astype(np.int64), "odate": odate, "otime": otime}
    fact = {"fk": rng.integers(0, n_dim, n_fact), "ship": ship, "price": rng.random(n_fact)}
    return dim, fact


def test_q3_on_date_columns_runs_the_fused_star_join(tmp_path, monkeypatch):
    """The Q3 shape on Parquet files with real date32 / timestamp[us] columns: the fused star join runs, the
    groups equal those of the same ticks typed int64, and no interpreter pass evaluates a date predicate --
    plain (`ship > DATE ...`), `YEAR(ship) = 1995` or `CAST(otime AS DATE) < DATE ...`.  The interpreter
    programs the query does launch are the bookkeeping of the group-by (its NULL-group check), the same
    programs the int64 query launches, and none holds a calendar opcode or a predicate literal."""
    import pyarrow.parquet as pq
    from dask_sql_b200 import _lib, executor
    dim, fact = _q3_tables()
    as_date = lambda v: pa.array(v.astype("datetime64[D]"), pa.date32())  # noqa: E731
    pq.write_table(pa.table({"ok": dim["pk"], "odate": as_date(dim["odate"]),
                             "otime": pa.array(dim["otime"].astype("datetime64[us]"), pa.timestamp("us"))}),
                   str(tmp_path / "orders.parquet"))
    pq.write_table(pa.table({"ok": fact["fk"], "ship": as_date(fact["ship"]), "price": fact["price"]}),
                   str(tmp_path / "lineitem.parquet"))
    pq.write_table(pa.table({"ok": dim["pk"], "odate": dim["odate"], "otime": dim["otime"]}),
                   str(tmp_path / "orders_i.parquet"))
    pq.write_table(pa.table({"ok": fact["fk"], "ship": fact["ship"], "price": fact["price"]}),
                   str(tmp_path / "lineitem_i.parquet"))
    c = _ctx()
    for name in ("orders", "lineitem", "orders_i", "lineitem_i"):
        c.create_table(name, str(tmp_path / f"{name}.parquet"))
    lit = int(np.datetime64("1995-03-15", "D").astype(np.int64))
    y95, y96 = (int(np.datetime64(s, "D").astype(np.int64)) for s in ("1995-01-01", "1996-01-01"))
    lit_us = lit * 86_400_000_000
    programs = []
    real = _lib.expr_eval

    def spy(prog_ref, *rest):
        prog = prog_ref._obj
        programs.append(tuple((prog.code[i].op, prog.code[i].a, prog.code[i].imm_i) for i in range(prog.n)))
        return real(prog_ref, *rest)

    monkeypatch.setattr(_lib, "expr_eval", spy)

    def run(q):
        programs.clear()
        before = executor.stats["star_fused"]
        out = c.sql(q).compute().sort_values("odate")
        assert executor.stats["star_fused"] > before
        return out, list(programs)

    q = "SELECT o.odate, SUM(l.price) AS rev FROM lineitem{t} l JOIN orders{t} o ON l.ok = o.ok WHERE {w} GROUP BY o.odate"
    for w_date, w_int in [
            ("l.ship > DATE '1995-03-15' AND o.odate < DATE '1995-03-15'", f"l.ship > {lit} AND o.odate < {lit}"),
            ("YEAR(l.ship) = 1995 AND CAST(o.otime AS DATE) < DATE '1995-03-15'",
             f"l.ship >= {y95} AND l.ship < {y96} AND o.otime < {lit_us}")]:
        got, p_date = run(q.format(t="", w=w_date))
        want, p_int = run(q.format(t="_i", w=w_int))
        assert p_date == p_int, (w_date, p_date, p_int)
        for prog in p_date:
            assert not any(op in (_lib.OP_DATEPART, _lib.OP_ADDMONTHS) for op, _, _ in prog), prog
            assert not any(op == _lib.OP_CONST_I and imm in (lit, lit_us, y95, y96) for op, _, imm in prog), prog
        assert got["odate"].dtype == np.dtype("datetime64[s]")
        assert got["odate"].to_numpy().astype("datetime64[D]").astype(np.int64).tolist() == want["odate"].tolist()
        np.testing.assert_allclose(got["rev"].to_numpy(), want["rev"].to_numpy(), rtol=1e-12)


def test_order_by_nulls_first_and_last_on_dates():
    c = _ctx()
    days = np.array(["2000-01-02", "NaT", "1999-12-31", "2000-01-01"], dtype="datetime64[D]")
    c.create_table("a", pa.table({"d": pa.array(days, pa.date32()), "x": [1, 2, 3, 4]}))
    assert c.sql("SELECT d, x FROM a ORDER BY d NULLS FIRST").compute()["x"].tolist() == [2, 3, 4, 1]
    assert c.sql("SELECT d, x FROM a ORDER BY d NULLS LAST").compute()["x"].tolist() == [3, 4, 1, 2]
    assert c.sql("SELECT d, x FROM a ORDER BY d DESC NULLS FIRST").compute()["x"].tolist() == [2, 1, 4, 3]
    got = c.sql("SELECT d FROM a ORDER BY d NULLS FIRST").compute()["d"]
    assert pd.isna(got.iloc[0]) and got.dtype == np.dtype("datetime64[s]")


def test_csv_location_round_trip(tmp_path):
    path = tmp_path / "t.csv"
    path.write_text("d,ts,v\n2000-01-01,2000-01-01 12:30:00,1\n1969-12-31,1969-12-31 23:59:59,2\n,,3\n")
    c = _ctx()
    c.create_table("t", str(path))
    got = c.sql("SELECT d, ts, v FROM t WHERE d < DATE '2000-01-01' OR d IS NULL").compute()
    assert got["v"].tolist() == [2, 3]
    assert pd.Timestamp(got["d"].iloc[0]) == pd.Timestamp("1969-12-31") and pd.isna(got["d"].iloc[1])
    assert pd.Timestamp(got["ts"].iloc[0]) == pd.Timestamp("1969-12-31 23:59:59") and pd.isna(got["ts"].iloc[1])
    assert c.sql("SELECT d, ts FROM t").dtypes.tolist() == [np.dtype("datetime64[D]"), np.dtype("datetime64[s]")]


def test_parquet_row_groups_pruned_on_sorted_dates(tmp_path):
    import pyarrow.parquet as pq
    days = np.sort(np.random.default_rng(1).integers(8000, 12000, 100_000)).astype("datetime64[D]")
    path = str(tmp_path / "d.parquet")
    pq.write_table(pa.table({"d": pa.array(days, pa.date32()), "v": np.ones(100_000)}), path, row_group_size=10_000)
    c = _ctx()
    c.create_table("p", path)
    got = c.sql("SELECT COUNT(*) AS n FROM p WHERE d >= DATE '2000-01-01' AND YEAR(d) < 2002").compute()
    lo, hi = np.datetime64("2000-01-01"), np.datetime64("2002-01-01")
    assert int(got["n"].iloc[0]) == int(((days >= lo) & (days < hi)).sum())
    pt = c.schema[c.schema_name].tables["p"].df.source.table
    assert pt.stats["row_groups_skipped"] >= 5
