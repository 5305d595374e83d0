"""RAND / RANDOM / RAND_INTEGER and TABLESAMPLE on the CPU side: the grammar, the errors, call-site numbering,
unseeded keys, the refusals, and the first row number of partitions, pruned Parquet row groups and shards."""
import numpy as np
import pandas as pd
import pytest

from dask_sql_b200 import Context
from dask_sql_b200.utils import ParsingException


@pytest.fixture()
def c():
    c = Context()
    c.create_table("t", pd.DataFrame({"a": np.arange(100), "system": np.arange(100) * 2.0}), npartitions=3)
    return c


def _scan(rel):
    while rel.get_current_node_type() != "TableScan":
        rel = rel.getInputs()[0] if hasattr(rel, "getInputs") else rel.inputs[0]
    return rel


def _exprs(rel):
    return [e for e in rel.expressions() if e.kind == "scalarfn" or (e.kind == "alias" and e.args[0].kind == "scalarfn")]


@pytest.mark.parametrize("sql", [
    "SELECT a FROM t TABLESAMPLE BERNOULLI (10)",
    "SELECT a FROM t AS x TABLESAMPLE BERNOULLI (10.5) REPEATABLE (4)",
    "SELECT a FROM t x TABLESAMPLE SYSTEM (0)",
    "SELECT system FROM t system TABLESAMPLE SYSTEM (100) REPEATABLE (-3)",
])
def test_tablesample_grammar(c, sql):
    rel, _ = c._get_ral(sql)
    s = _scan(rel).sample
    assert s is not None and s.method in ("bernoulli", "system") and 0 <= s.p <= 100 and s.site == 1


def test_columns_named_like_the_contextual_words(c):
    c.create_table("u", pd.DataFrame({"tablesample": [1], "bernoulli": [2], "repeatable": [3]}))
    rel, _ = c._get_ral("SELECT tablesample, bernoulli, repeatable FROM u")
    assert _scan(rel).sample is None
    rel, _ = c._get_ral("SELECT system FROM t")
    assert _scan(rel).sample is None


@pytest.mark.parametrize("sql,match", [
    ("SELECT a FROM t TABLESAMPLE BERNOULLI (101)", "outside"),
    ("SELECT a FROM t TABLESAMPLE BERNOULLI (-1)", "outside"),
    ("SELECT a FROM t TABLESAMPLE SYSTEM (a)", "numeric literal"),
    ("SELECT a FROM t TABLESAMPLE SYSTEM ('5')", "numeric literal"),
    ("SELECT a FROM t TABLESAMPLE BERNOULLI (5) REPEATABLE (1.5)", "integer literal"),
    ("SELECT RAND(1, 2) FROM t", "RAND takes 0 or 1"),
    ("SELECT RANDOM(a) FROM t", "RANDOM takes its seed"),
    ("SELECT RAND(0.5) FROM t", "RAND takes its seed"),
    ("SELECT RAND_INTEGER() FROM t", "RAND_INTEGER takes 1 or 2"),
    ("SELECT RAND_INTEGER(1, 2, 3) FROM t", "RAND_INTEGER takes 1 or 2"),
    ("SELECT RAND_INTEGER(0) FROM t", "RAND_INTEGER takes its bound"),
    ("SELECT RAND_INTEGER(1, -5) FROM t", "RAND_INTEGER takes its bound"),
    ("SELECT RAND_INTEGER(a) FROM t", "RAND_INTEGER takes its bound"),
    ("SELECT RAND_INTEGER(a, 10) FROM t", "RAND_INTEGER takes its seed"),
])
def test_errors_name_the_function(c, sql, match):
    with pytest.raises(ParsingException, match=match):
        c._get_ral(sql)


def test_call_sites_are_numbered_in_textual_order(c):
    rel, text = c._get_ral("SELECT RAND(1) AS r, RAND_INTEGER(2, 5) AS i FROM t TABLESAMPLE BERNOULLI (5) "
                           "REPEATABLE (3) WHERE RANDOM(4) < 0.5")
    assert "rand(Int64(1), Int64(1))" in text and "rand_integer(Int64(2), Int64(2), Int64(5))" in text
    assert "rand(Int64(4), Int64(4))" in text
    assert _scan(rel).sample.site == 3 and _scan(rel).sample.key == 3


def test_negative_seed_is_twos_complement(c):
    _, text = c._get_ral("SELECT RAND(-1) AS r FROM t")
    assert "rand(Int64(-1), Int64(1))" in text          # key 2^64 - 1 as a signed int64


def test_unseeded_key_differs_between_statements(c):
    from dask_sql_b200.planner import plan_sql
    keys = set()
    for _ in range(3):
        rel = plan_sql("SELECT RAND() AS r, RAND_INTEGER(9) AS i FROM t", c._catalog)
        assert rel.volatile
        texts = [e.args[0].args[0].value for e in rel.exprs]
        assert texts[0] == texts[1]                    # one key per statement, the sites tell the calls apart
        keys.add(texts[0])
    assert len(keys) == 3
    assert not plan_sql("SELECT RAND(3) AS r FROM t", c._catalog).volatile
    # a statement with an unseeded key is not served from the plan cache
    a, b = c.sql("SELECT RAND() AS r FROM t"), c.sql("SELECT RAND() AS r FROM t")
    assert a is not b
    a, b = c.sql("SELECT RAND(1) AS r FROM t"), c.sql("SELECT RAND(1) AS r FROM t")
    assert a is b


def test_refusals(c):
    c.create_table("u", pd.DataFrame({"b": np.arange(10)}))
    c.sql("CREATE VIEW v AS SELECT a FROM t WHERE a > 3")
    with pytest.raises(NotImplementedError, match="TABLESAMPLE of the view"):
        c.sql("SELECT a FROM v TABLESAMPLE BERNOULLI (5)")
    with pytest.raises(NotImplementedError, match="TABLESAMPLE of the common table expression"):
        c.sql("WITH w AS (SELECT a FROM t) SELECT a FROM w TABLESAMPLE SYSTEM (5)")
    with pytest.raises(NotImplementedError, match="TABLESAMPLE of a subquery"):
        c.sql("SELECT a FROM (SELECT a FROM t) s TABLESAMPLE SYSTEM (5)")
    rule = "defined on the rows of one base table"
    with pytest.raises(NotImplementedError, match=rule):
        c.sql("SELECT RAND(1) AS r FROM t JOIN u ON t.a = u.b")
    with pytest.raises(NotImplementedError, match=rule):
        c.sql("SELECT COUNT(*) AS n, RAND(1) AS r FROM t")
    with pytest.raises(NotImplementedError, match=rule):
        c.sql("SELECT RAND(1) AS r FROM (SELECT a FROM t ORDER BY a LIMIT 5) s")


def test_row_base_of_partitions():
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import TableSource
    from dask_sql_b200.table import DeviceTable
    t = DeviceTable.from_columns({"a": np.arange(1000)}, npartitions=7, persist=False)
    assert all(rb is None for _, rb in executor.table_parts(TableSource(t), {"a"}))     # nothing draws: no numbers
    src = TableSource(t)
    src.numbered = True
    got = [(p["a"].n, rb) for p, rb in executor.table_parts(src, {"a"})]
    sizes = [n for n, _ in got]
    assert sum(sizes) == 1000 and [rb for _, rb in got] == list(np.cumsum([0] + sizes[:-1]))
    for p, rb in executor.table_parts(src, {"a"}):
        assert p["a"].data[0].item() == rb                    # the value of column a is the row's number


def test_row_base_of_pruned_parquet_groups(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import TableSource
    from dask_sql_b200.table import ParquetTable
    path = str(tmp_path / "p.parquet")
    pq.write_table(pa.table({"a": np.arange(1000, dtype=np.int64)}), path, row_group_size=130)
    t = ParquetTable(path)
    pred_terms = [("a", L.GE, 500)]
    from dask_sql_b200.expr import ColRef, Lit, binop
    pred = [binop("ge", ColRef("a", L.I64), Lit(500))]
    src = TableSource(t)
    src.numbered = True
    got = executor.table_parts(src, {"a"}, pred)
    assert t.surviving_groups(pred_terms) == [3, 4, 5, 6, 7]
    assert [rb for _, rb in got] == [390, 520, 650, 780, 910]
    for p, rb in got:
        assert int(p["a"].data[0]) == rb


def _sharded_ranks(monkeypatch, bounds):
    """one table per rank holding rows bounds[r] .. bounds[r + 1] - 1 of a column a = row number, with
    parallel.world / all_gather_ints answering as rank r of len(bounds) - 1 ranks would hear them"""
    from dask_sql_b200 import executor
    from dask_sql_b200 import parallel as P
    from dask_sql_b200.table import DeviceTable
    world = len(bounds) - 1
    gathered = []
    monkeypatch.setattr(executor, "_dev", lambda: "cpu")
    monkeypatch.setattr(P, "all_gather_ints",
                        lambda vals, dev: gathered.append(1) or [[bounds[r + 1] - bounds[r]] for r in range(world)])
    for rank in range(world):
        lo, hi = bounds[rank], bounds[rank + 1]
        t = DeviceTable.from_columns({"a": np.arange(lo, hi)}, npartitions=2, persist=False, distribution="sharded")
        monkeypatch.setattr(P, "world", lambda rank=rank: (rank, world))
        yield rank, t, gathered


@pytest.mark.parametrize("uneven", [False, True], ids=["shard_bounds", "uneven"])
def test_row_base_of_sharded_ranks(monkeypatch, uneven):
    """rank r numbers its rows from the rows of the ranks before it: shard_bounds' lower bound when the
    shards were cut by it, and 0 ... N-1 once each whatever the shards' sizes"""
    from dask_sql_b200 import executor
    from dask_sql_b200 import parallel as P
    from dask_sql_b200.frame import TableSource
    n, world = 10_000, 3
    bounds = [0, 6_000, 6_100, n] if uneven else [P.shard_bounds(n, r, world)[0] for r in range(world)] + [n]
    seen = []
    for rank, t, _ in _sharded_ranks(monkeypatch, bounds):
        src = TableSource(t)
        src.numbered = True
        for p, rb in executor.table_parts(src, {"a"}):
            assert int(p["a"].data[0]) == rb
            seen += list(range(rb, rb + p["a"].n))
        assert executor.table_row_start(t) == bounds[rank]
        if not uneven:
            assert bounds[rank] == P.shard_bounds(n, rank, world)[0]
    assert seen == list(range(n))


def test_unnumbered_sharded_scan_asks_the_other_ranks_nothing(monkeypatch):
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import TableSource
    for rank, t, gathered in _sharded_ranks(monkeypatch, [0, 500, 1000]):
        assert all(rb is None for _, rb in executor.table_parts(TableSource(t), {"a"}))
        assert not gathered
