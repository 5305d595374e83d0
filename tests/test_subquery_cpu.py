"""Subqueries in the planner, without a GPU: parse and bind of every form, the split of correlated conjuncts into
equality keys and pair terms, the EXPLAIN text, each refusal and its message, and the plan cache skipping a
statement with an uncorrelated scalar subquery."""
import pytest

from dask_sql_b200.planner import plan_sql
from dask_sql_b200.planner.sqlparse import parse_sql
from dask_sql_b200.utils import ParsingException

CAT = {"t": [("a", "BIGINT"), ("b", "DOUBLE"), ("c", "BIGINT")], "u": [("x", "BIGINT"), ("y", "DOUBLE"), ("z", "BIGINT")],
       "w": [("p", "BIGINT")]}


def _catalog(schema, table):
    return ("root", CAT[table]) if table in CAT else None


def _plan(sql):
    return plan_sql(sql, _catalog)


def _calls(plan):
    from dask_sql_b200.planner import plan as P
    out = []
    for node in P.walk(plan):
        for e in node.expressions():
            out += e.subqueries()
    return out


def test_parse_every_form():
    w = parse_sql("SELECT a FROM t WHERE a NOT IN (SELECT x FROM u) AND NOT EXISTS (SELECT 1 FROM u) "
                  "AND b > (SELECT MAX(y) FROM u)").where
    assert w.l.l.kind == "insubquery" and w.l.l.negated
    assert w.l.r.kind == "not" and w.l.r.e.kind == "exists"
    assert w.r.r.kind == "scalarsubquery"
    assert parse_sql("SELECT a FROM t WHERE a IN (WITH q AS (SELECT x FROM u) SELECT x FROM q)").where.kind == \
        "insubquery"


def test_uncorrelated_in_keys_on_its_operand():
    (call,) = _calls(_plan("SELECT a FROM t WHERE a IN (SELECT x FROM u WHERE z > 1)"))
    sq = call.value
    assert sq.kind == "in" and sq.null_aware and sq.keys == [0] and sq.terms == []
    assert [a.display() for a in call.args] == ["t.a"]


def test_correlated_split_into_keys_and_pair_terms():
    (call,) = _calls(_plan("SELECT a FROM t WHERE c IN (SELECT z FROM u WHERE u.x = t.a AND u.y < t.b AND "
                           "t.c <> u.z AND z > 0)"))
    sq = call.value
    assert sq.kind == "in" and not sq.null_aware
    names = [f.getName() for f in sq.plan.schema]
    assert [names[k] for k in sq.keys] == ["__corr0"]
    # outer <cmp> inner: u.y < t.b is t.b > y; the IN's own t.c = z is three-valued (where=False)
    assert [(names[k], op, where) for k, op, where in sq.terms] == [("__corr1", ">", True), ("__corr2", "!=", True),
                                                                    ("z", "=", False)]
    assert [a.display() for a in call.args] == ["t.a", "t.b", "t.c", "t.c"]
    assert "u.z > Int64(0)" in sq.plan.explain()         # the local conjunct stays a filter of the body


def test_exists_and_not_exists_and_select_list():
    plan = _plan("SELECT a, EXISTS (SELECT 1 FROM u WHERE u.x = t.a) AS e FROM t "
                 "WHERE NOT EXISTS (SELECT 1 FROM u WHERE x = a AND t.b >= u.y)")
    calls = _calls(plan)
    assert sorted(c.value.kind for c in calls) == ["exists", "exists"]
    assert all(c.sql_type == "BOOLEAN" for c in calls)


def test_explain_prints_subqueries_with_keys_and_terms():
    text = _plan("EXPLAIN SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.x = t.a AND u.y < t.b) "
                 "AND a NOT IN (SELECT p FROM w)").explain()
    assert "Subquery: EXISTS keys=[t.a = __corr0] pair terms=[t.b > __corr1]" in text
    assert "Subquery: IN keys=[t.a = p]" in text
    assert "TableScan: w" in text and "TableScan: u" in text


def test_nested_subquery_and_cte():
    plan = _plan("WITH q AS (SELECT x FROM u WHERE y > 1) SELECT a FROM t WHERE a IN (SELECT x FROM q WHERE x IN "
                 "(SELECT p FROM w))")
    (outer,) = _calls(plan)
    assert len(_calls(outer.value.plan)) == 1


@pytest.mark.parametrize("sql, msg", [
    ("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.y < t.b)", "needs an equality key"),
    ("SELECT a FROM t WHERE c IN (SELECT z FROM u WHERE u.y < t.b)", "needs an equality key"),
    ("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.x = t.a AND u.z IN (SELECT p FROM w WHERE w.p = t.c))",
     "immediately enclosing block"),
    ("SELECT a FROM t WHERE EXISTS (SELECT t.a FROM u WHERE u.x = t.a)", "immediately enclosing block"),
    ("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.x + t.a = t.c)", "must compare"),
    ("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.x = t.a OR u.y = t.b)", "must compare"),
    ("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.x = t.a AND u.y < t.b AND u.y > t.b AND u.z <> t.c "
     "AND u.z < t.a AND u.x <> t.c)", "at most 4"),
    ("SELECT a FROM t WHERE (a, c) IN (SELECT x, z FROM u)", "row values"),
    ("SELECT a FROM t WHERE a = ANY (SELECT x FROM u)", "ANY / ALL / SOME"),
    ("SELECT a FROM t WHERE a > ALL (SELECT x FROM u)", "ANY / ALL / SOME"),
    ("SELECT a FROM t JOIN w ON t.a = w.p AND w.p IN (SELECT x FROM u)", "ON clause"),
    ("SELECT c, COUNT(*) FROM t GROUP BY c IN (SELECT z FROM u)", "GROUP BY"),
    ("SELECT a FROM t ORDER BY a IN (SELECT x FROM u)", "ORDER BY"),
    ("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM u WHERE u.x = t.a LIMIT 1)", "LIMIT, ORDER BY, DISTINCT"),
    ("SELECT a FROM t WHERE EXISTS (SELECT DISTINCT y FROM u WHERE u.x = t.a)", "LIMIT, ORDER BY, DISTINCT"),
    ("SELECT a FROM t WHERE EXISTS (SELECT COUNT(*) FROM u WHERE u.x = t.a)", "needs a GROUP BY"),
    ("SELECT a FROM t WHERE EXISTS (SELECT z FROM u WHERE u.x = t.a AND u.y < t.b GROUP BY z)",
     "equality keys only"),
    ("SELECT a FROM t WHERE b > (SELECT y FROM u WHERE u.x = t.a)", "must be one aggregate"),
    ("SELECT a FROM t WHERE b > (SELECT AVG(y) FROM u WHERE u.x = t.a GROUP BY z)", "must be one aggregate"),
    ("SELECT a FROM t WHERE b > (SELECT COUNT(*) + 1 FROM u WHERE u.x = t.a)", "COUNT inside an expression"),
    ("SELECT a FROM t WHERE b > (SELECT AVG(y) FROM u WHERE u.x = t.a + 1)", "on columns of the enclosing block"),
    ("SELECT c, COUNT(*) FROM t GROUP BY c HAVING c > (SELECT AVG(y) FROM u WHERE u.x = t.c)", "in HAVING"),
])
def test_refusals_name_the_rule(sql, msg):
    with pytest.raises(NotImplementedError, match=msg):
        _plan(sql)


def test_in_subquery_of_two_columns_is_a_parsing_error():
    with pytest.raises(ParsingException, match="one column"):
        _plan("SELECT a FROM t WHERE a IN (SELECT x, z FROM u)")
    with pytest.raises(ParsingException, match="one column"):
        _plan("SELECT a FROM t WHERE b > (SELECT x, z FROM u)")


def test_uncorrelated_scalar_subquery_is_not_cached():
    assert _plan("SELECT a FROM t WHERE b > (SELECT AVG(y) FROM u)").volatile
    assert not _plan("SELECT a FROM t WHERE a IN (SELECT x FROM u)").volatile


def test_subquery_predicate_stays_above_the_scan():
    plan = _plan("SELECT a FROM t WHERE c > 0 AND a IN (SELECT x FROM u)")
    text = plan.explain()
    assert "Filter: t.a IN (<subquery>)" in text
    assert "TableScan: t projection=[a, c], full_filters=[t.c > Int64(0)]" in text


def test_correlated_scalar_becomes_a_left_join_on_the_grouped_body():
    """DataFusion's scalar-subquery-to-join rule: LEFT JOIN (SELECT keys, agg FROM ... GROUP BY keys) ON keys"""
    plan = _plan("SELECT a FROM t WHERE b < (SELECT 0.2 * AVG(y) FROM u WHERE u.x = t.a AND u.z > 0)")
    text = plan.explain()
    assert "Left Join: t.a = __sq1.__corr0" in text
    assert "Aggregate: groupBy=[[u.x]], aggr=[[AVG(u.y)]]" in text
    assert "Filter: t.b < __sq1.__sv" in text
    assert not plan.volatile and _calls(plan) == []
    # COUNT over an empty correlation group is 0, not NULL; SELECT * does not show the joined columns
    plan = _plan("SELECT *, (SELECT COUNT(*) FROM u WHERE u.x = t.a) AS n FROM t")
    assert "CASE WHEN __sq1.__sv IS NULL THEN Int64(0) ELSE __sq1.__sv END AS n" in plan.explain()
    assert [f.getName() for f in plan.schema] == ["a", "b", "c", "n"]


def test_grouped_correlated_body_groups_by_its_keys():
    (call,) = _calls(_plan("SELECT a FROM t WHERE EXISTS (SELECT z FROM u WHERE u.x = t.a GROUP BY z "
                           "HAVING COUNT(*) > 1)"))
    assert "Aggregate: groupBy=[[u.z, u.x]]" in call.value.plan.explain()


def test_varchar_pair_terms_are_refused_at_plan_time():
    cat = dict(CAT, s=[("k", "BIGINT"), ("name", "VARCHAR")])
    with pytest.raises(NotImplementedError, match="VARCHAR expressions by equality keys only"):
        plan_sql("SELECT a FROM t WHERE EXISTS (SELECT 1 FROM s WHERE s.k = t.a AND s.name <> t.c)",
                 lambda schema, table: ("root", cat[table]) if table in cat else None)


@pytest.mark.parametrize("dist, refused", [("sharded", True), ("root", True), ("replicated", False)])
def test_marks_over_sharded_or_root_rows_are_refused_on_more_than_one_gpu(monkeypatch, dist, refused):
    """both the outer rows and the subquery's rows: a rank holding part of either would mark wrongly"""
    from dask_sql_b200 import executor as X
    from dask_sql_b200.frame import LazyFrame, TableSource

    class Table:
        distribution = dist

    src = TableSource.__new__(TableSource)
    src.table = Table()
    frame = LazyFrame.__new__(LazyFrame)
    frame.source = src
    monkeypatch.setattr(X.P, "world", lambda: (0, 2))
    why = X.mark_refusal(frame)
    assert (why is not None) == refused
    if refused:
        assert "sharded or root table on more than one GPU" in why
    monkeypatch.setattr(X.P, "world", lambda: (0, 1))
    assert X.mark_refusal(frame) is None
