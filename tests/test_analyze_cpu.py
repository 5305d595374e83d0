"""ANALYZE TABLE ... COMPUTE STATISTICS on the host: the grammar, schema-qualified names, contextual words as
column names, the planner's errors, and the AnalyzeTable node that Context.sql hands to its plugin.  No
kernel is launched: the plugin is swapped for one that returns the plan node."""
import numpy as np
import pandas as pd
import pytest


def _ctx():
    from dask_sql_b200 import Context
    c = Context()
    c.create_table("t", pd.DataFrame({"a": [1.0, 2.0], "columns": [1, 2], "statistics": [3, 4], "B": [5, 6]}))
    c.create_schema("other")
    c.create_table("u", pd.DataFrame({"x": [1, 2]}), schema_name="other")
    return c


@pytest.fixture
def plan_of():
    """Context.sql with the AnalyzeTable plugin replaced by one that returns the plan node it is given"""
    from dask_sql_b200.physical.rel import RelConverter
    from dask_sql_b200.physical.rel.custom import AnalyzeTablePlugin

    class Capture:
        class_name = "AnalyzeTable"

        def convert(self, rel, context):
            return rel

    RelConverter.add_plugin_class(Capture, replace=True)
    try:
        c = _ctx()
        yield lambda sql: c.sql(sql)
    finally:
        RelConverter.add_plugin_class(AnalyzeTablePlugin, replace=True)


def _parse(sql):
    from dask_sql_b200.planner.sqlparse import parse_sql
    return parse_sql(sql)


def test_parser_forms():
    n = _parse("ANALYZE TABLE t COMPUTE STATISTICS FOR ALL COLUMNS")
    assert (n.kind, n.name, n.columns) == ("analyze_table", "t", [])
    n = _parse("analyze table s.t compute statistics for columns a, columns , statistics;")
    assert (n.name, n.columns) == ("s.t", ["a", "columns", "statistics"])
    n = _parse('ANALYZE TABLE "My Table" COMPUTE STATISTICS FOR COLUMNS "all", "for"')
    assert (n.name, n.columns) == ("My Table", ["all", "for"])
    from dask_sql_b200.utils import ParsingException
    for bad in ("ANALYZE TABLE t COMPUTE STATISTICS", "ANALYZE TABLE t COMPUTE STATISTICS FOR ALL",
                "ANALYZE TABLE t STATISTICS FOR ALL COLUMNS", "ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS",
                "ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS a,", "ANALYZE t COMPUTE STATISTICS FOR ALL COLUMNS",
                "ANALYZE TABLE t COMPUTE STATISTICS FOR ALL COLUMNS x"):
        with pytest.raises(ParsingException):
            _parse(bad)


def test_contextual_words_stay_column_names():
    from dask_sql_b200.planner.sqlparse import KEYWORDS
    assert not {"ANALYZE", "COMPUTE", "STATISTICS", "FOR", "COLUMNS"} & KEYWORDS
    c = _ctx()
    rel, _ = c._get_ral("SELECT columns, statistics FROM t WHERE columns > 1")
    assert [f.getName() for f in rel.getRowType().getFieldList()] == ["columns", "statistics"]


def test_sql_produces_the_analyze_node(plan_of):
    rel = plan_of("ANALYZE TABLE t COMPUTE STATISTICS FOR ALL COLUMNS")
    assert rel.get_current_node_type() == "AnalyzeTable"
    stmt = rel.analyze_table()
    assert (stmt.getSchemaName(), stmt.getTableName(), stmt.getColumns()) == ("root", "t", [])
    rel = plan_of("ANALYZE TABLE T COMPUTE STATISTICS FOR COLUMNS columns, a")
    assert rel.analyze_table().getColumns() == ["columns", "a"]
    assert rel.analyze_table().getTableName() == "t"
    rel = plan_of("ANALYZE TABLE other.u COMPUTE STATISTICS FOR COLUMNS x")
    stmt = rel.analyze_table()
    assert (stmt.getSchemaName(), stmt.getTableName(), stmt.getColumns()) == ("other", "u", ["x"])


def test_errors_follow_the_planner():
    from dask_sql_b200.utils import ParsingException
    c = _ctx()
    with pytest.raises(ParsingException) as select_err:
        c.sql("SELECT * FROM missing")
    with pytest.raises(ParsingException) as analyze_err:
        c.sql("ANALYZE TABLE missing COMPUTE STATISTICS FOR ALL COLUMNS")
    assert "table 'missing' not found" in str(select_err.value)
    assert "table 'missing' not found" in str(analyze_err.value)
    with pytest.raises(ParsingException, match="other.t"):
        c.sql("ANALYZE TABLE other.t COMPUTE STATISTICS FOR ALL COLUMNS")
    with pytest.raises(ParsingException, match="nope"):
        c.sql("ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS a, nope")
    with pytest.raises(ParsingException, match="'a'.*more than once"):
        c.sql("ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS a, columns, a")
    with pytest.raises(ParsingException, match="'b'"):      # identifiers are case sensitive by default
        c.sql("ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS b")


def test_case_insensitive_columns(plan_of):
    from dask_sql_b200 import config
    with config.set({"sql.identifier.case_sensitive": False}):
        rel = plan_of("ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS b, A")
    assert rel.analyze_table().getColumns() == ["B", "a"]


def test_select_image_round_trips():
    from dask_sql_b200 import executor as X
    from dask_sql_b200._lib import F64, I64
    from tests import select_ref as R
    xs = np.array([-np.inf, -1e300, -1.0, -5e-324, -0.0, 0.0, 5e-324, 2.5, np.inf])
    imgs = [X.select_image(x, F64) for x in xs]
    assert imgs == sorted(imgs) and imgs == [int(u) for u in R.images(xs)]
    assert all(X.select_value(u, F64) == x and np.signbit(X.select_value(u, F64)) == np.signbit(x)
               for u, x in zip(imgs, xs))
    ks = [-(1 << 63), -1, 0, 1, (1 << 63) - 1]
    imgs = [X.select_image(k, I64) for k in ks]
    assert imgs == [0, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, (1 << 64) - 1]
    assert [X.select_value(u, I64) for u in imgs] == ks
