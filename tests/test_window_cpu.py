"""Window functions without a GPU: parsing and binding of every OVER form, the Window plan node and its EXPLAIN
text, the default frames, and each construct that is refused."""
import pytest

from dask_sql_b200.planner import plan as P
from dask_sql_b200.planner.builder import Binder
from dask_sql_b200.planner.sqlparse import parse_sql
from dask_sql_b200.utils import ParsingException

INF = float("inf")
COLS = [("k", "BIGINT"), ("t", "BIGINT"), ("v", "DOUBLE"), ("s", "VARCHAR"), ("d", "DATE")]


def _plan(sql):
    return Binder(sql, lambda schema, name: ("root", COLS) if name == "t" else None).bind_statement(parse_sql(sql))


def _window(plan):
    return next(p for p in P.walk(plan) if isinstance(p, P.Window))


@pytest.mark.parametrize("text,frame", [
    ("", (True, -INF, 0)),
    ("ROWS 3 PRECEDING", (False, -3, 0)),
    ("ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING", (False, -2, 3)),
    ("ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING", (False, 0, INF)),
    ("ROWS BETWEEN 3 FOLLOWING AND 1 PRECEDING", (False, 3, -1)),
    ("RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW", (True, -INF, 0)),
    ("RANGE BETWEEN CURRENT ROW AND CURRENT ROW", (True, 0, 0)),
    ("RANGE UNBOUNDED PRECEDING", (True, -INF, 0)),
])
def test_frames_bind(text, frame):
    w = _window(_plan(f"SELECT SUM(v) OVER (PARTITION BY k ORDER BY t DESC NULLS LAST {text}) FROM t"))
    (e,) = w.window_exprs
    assert e.frame == frame and e.name == "SUM" and e.sql_type == "DOUBLE"
    assert [(o.display(), a, nf) for o, a, nf in e.order] == [("t.t", False, False)]
    assert [p.display() for p in e.partition] == ["t.k"]


def test_default_frame_without_order_is_the_partition():
    (e,) = _window(_plan("SELECT COUNT(*) OVER (PARTITION BY k) FROM t")).window_exprs
    assert e.frame == (False, -INF, INF) and e.sql_type == "BIGINT" and not e.args


@pytest.mark.parametrize("fn,arg,ty", [("ROW_NUMBER", "", "BIGINT"), ("RANK", "", "BIGINT"), ("DENSE_RANK", "", "BIGINT"),
                                       ("COUNT", "s", "BIGINT"), ("SUM", "k", "BIGINT"), ("AVG", "k", "DOUBLE"),
                                       ("MIN", "s", "VARCHAR"), ("MAX", "d", "DATE"), ("FIRST_VALUE", "v", "DOUBLE"),
                                       ("LAST_VALUE", "s", "VARCHAR")])
def test_result_types(fn, arg, ty):
    (e,) = _window(_plan(f"SELECT {fn}({arg}) OVER (ORDER BY t) FROM t")).window_exprs
    assert e.sql_type == ty


def test_plan_shape_specs_and_explain():
    plan = _plan("SELECT k, ROW_NUMBER() OVER (PARTITION BY k ORDER BY t) AS r, "
                 "SUM(v) OVER (PARTITION BY k ORDER BY t ROWS 2 PRECEDING) AS s, MAX(v) OVER () AS m FROM t "
                 "WHERE v > 0 ORDER BY r LIMIT 3")
    kinds = [p.node_type for p in P.walk(plan)]
    assert kinds == ["Limit", "Sort", "Projection", "Window", "Filter", "TableScan"]
    w = _window(plan)
    groups = w.getGroups()
    assert len(groups) == 2 and [len(calls) for _, calls in groups] == [2, 1]
    assert [f.getName() for f in w.schema][-3:] == [e.display() for e in w.window_exprs]
    text = w.explain()
    assert text.startswith("Window: [PARTITION BY [t.k] ORDER BY [t.t ASC NULLS LAST]]: ROW_NUMBER()")
    assert "[whole input]: MAX(t.v) ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING" in text


def test_window_over_group_by_binds_aggregates():
    plan = _plan("SELECT k, SUM(v), RANK() OVER (ORDER BY SUM(v) DESC) FROM t GROUP BY k HAVING COUNT(*) > 1")
    assert [p.node_type for p in P.walk(plan)][:4] == ["Projection", "Window", "Filter", "Aggregate"]
    (e,) = _window(plan).window_exprs
    assert e.order[0][0].kind == "column" and e.order[0][0].name == "SUM(t.v)"


def test_top_n_through_subquery_filters_above_the_window():
    from dask_sql_b200.planner.optimizer import optimize
    plan = optimize(_plan("SELECT * FROM (SELECT k, ROW_NUMBER() OVER (PARTITION BY k ORDER BY t) AS r FROM t) s "
                          "WHERE r <= 3"))
    kinds = [p.node_type for p in P.walk(plan)]
    assert kinds.index("Filter") < kinds.index("Window")


def test_order_by_a_window_call_of_the_select_list():
    plan = _plan("SELECT k, ROW_NUMBER() OVER (ORDER BY t) FROM t ORDER BY ROW_NUMBER() OVER (ORDER BY t) DESC")
    assert plan.node_type == "Sort" and plan.keys[0][0].name.startswith("ROW_NUMBER()")
    # aliased in the SELECT list: the sort reads the alias, nothing is computed twice
    plan = _plan("SELECT k, ROW_NUMBER() OVER (ORDER BY t) AS r FROM t ORDER BY ROW_NUMBER() OVER (ORDER BY t)")
    assert plan.node_type == "Sort" and plan.keys[0][0].name == "r"
    assert len(_window(plan).window_exprs) == 1


def test_order_by_a_window_call_outside_the_select_list():
    plan = _plan("SELECT k FROM t ORDER BY RANK() OVER (PARTITION BY k ORDER BY v DESC), k LIMIT 5")
    assert [p.node_type for p in P.walk(plan)] == ["Projection", "Limit", "Sort", "Projection", "Window", "TableScan"]
    assert [f.getName() for f in plan.schema] == ["k"]
    sort = plan.inputs[0].inputs[0]
    assert sort.keys[0][0].name.startswith("RANK()") and sort.keys[1][0].name == "k"
    # over a GROUP BY output, reading an aggregate only ORDER BY names
    plan = _plan("SELECT k FROM t GROUP BY k ORDER BY RANK() OVER (ORDER BY SUM(v) DESC)")
    assert "SUM(t.v)" in [a.display() for a in next(p for p in P.walk(plan) if p.node_type == "Aggregate").agg_exprs]
    with pytest.raises(NotImplementedError, match="DISTINCT"):
        _plan("SELECT DISTINCT k FROM t ORDER BY ROW_NUMBER() OVER (ORDER BY t)")


@pytest.mark.parametrize("sql,match", [
    ("SELECT LAG(v) OVER (ORDER BY t) FROM t", "LAG"),
    ("SELECT LEAD(v, 1) OVER (ORDER BY t) FROM t", "LEAD"),
    ("SELECT NTILE(4) OVER (ORDER BY t) FROM t", "NTILE"),
    ("SELECT NTH_VALUE(v, 2) OVER (ORDER BY t) FROM t", "NTH_VALUE"),
    ("SELECT PERCENT_RANK() OVER (ORDER BY t) FROM t", "PERCENT_RANK"),
    ("SELECT CUME_DIST() OVER (ORDER BY t) FROM t", "CUME_DIST"),
    ("SELECT SINGLE_VALUE(v) OVER (ORDER BY t) FROM t", "SINGLE_VALUE"),
    ("SELECT SUM(v) OVER (ORDER BY t RANGE BETWEEN 2 PRECEDING AND CURRENT ROW) FROM t", "RANGE"),
    ("SELECT SUM(v) OVER (ORDER BY t GROUPS 2 PRECEDING) FROM t", "GROUPS"),
    ("SELECT SUM(v) OVER (ORDER BY t ROWS 2 PRECEDING EXCLUDE CURRENT ROW) FROM t", "EXCLUDE"),
    ("SELECT SUM(v) OVER w FROM t", "named window"),
    ("SELECT SUM(v) OVER (ORDER BY t) FROM t WINDOW w AS (ORDER BY t)", "WINDOW clause"),
    ("SELECT COUNT(DISTINCT v) OVER (ORDER BY t) FROM t", "DISTINCT"),
    ("SELECT SUM(v) FILTER (WHERE v > 0) OVER (ORDER BY t) FROM t", "FILTER"),
    ("SELECT STDDEV(v) OVER (ORDER BY t) FROM t", "STDDEV"),
    ("SELECT SUM(s) OVER (ORDER BY t) FROM t", "VARCHAR"),
])
def test_refusals(sql, match):
    with pytest.raises(NotImplementedError, match=match):
        _plan(sql)


@pytest.mark.parametrize("sql", [
    "SELECT k FROM t WHERE ROW_NUMBER() OVER (ORDER BY t) = 1",
    "SELECT COUNT(*) FROM t GROUP BY ROW_NUMBER() OVER (ORDER BY t)",
    "SELECT k, COUNT(*) FROM t GROUP BY k HAVING RANK() OVER (ORDER BY k) = 1",
    "SELECT SUM(v) OVER (ORDER BY t ROWS BETWEEN UNBOUNDED FOLLOWING AND CURRENT ROW) FROM t",
    "SELECT SUM(v) OVER (ORDER BY t ROWS BETWEEN CURRENT ROW AND UNBOUNDED PRECEDING) FROM t",
    "SELECT SUM(v) OVER (ORDER BY t ROWS 1.5 PRECEDING) FROM t",
    "SELECT SUM(SUM(v) OVER ()) OVER () FROM t",
    "SELECT ROW_NUMBER(k) OVER () FROM t",
    "SELECT SUM(ROW_NUMBER() OVER ()) FROM t",
    "SELECT COUNT(*) FILTER (WHERE RANK() OVER (ORDER BY t) = 1) FROM t",
])
def test_errors(sql):
    with pytest.raises(ParsingException):
        _plan(sql)


def test_window_only_function_needs_over():
    with pytest.raises(NotImplementedError, match="OVER"):
        _plan("SELECT ROW_NUMBER() FROM t")


def test_plugin_is_registered_as_window_only():
    from dask_sql_b200.physical.rel.logical import DaskWindowPlugin
    assert DaskWindowPlugin.class_name == "Window"


def test_columns_named_like_window_words_still_parse():
    cols = [("over", "BIGINT"), ("rows", "BIGINT"), ("range", "BIGINT"), ("partition", "BIGINT")]
    sql = "SELECT over, rows, range, partition FROM t"
    plan = Binder(sql, lambda s, n: ("root", cols)).bind_statement(parse_sql(sql))
    assert [f.getName() for f in plan.schema] == ["over", "rows", "range", "partition"]


def test_bench_window_runs_to_the_first_device_call(tmp_path):
    """scripts/bench_window.py builds its table and checks the reference before touching a device; without one it
    stops at the first device call (there is no CPU fallback)."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the script would run for real")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.join(root, "scripts", "bench_window.py"), "--rows", "3000", "--keys",
                          "30", "--check-rows", "1000", "--out", str(tmp_path / "o.json")],
                         capture_output=True, text=True, timeout=600, cwd=str(tmp_path))
    assert res.returncode != 0
    assert "Traceback" in res.stderr and ("CUDA" in res.stderr or "NVIDIA" in res.stderr), res.stderr[-2000:]
    assert "torch.cuda.set_device" in res.stderr or "_lazy_init" in res.stderr
    assert not (tmp_path / "o.json").exists()
