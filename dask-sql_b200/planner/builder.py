"""Syntax tree -> logical plan (the job of DataFusion's SqlToRel in the reference,
src/sql.rs:586-596), for the hot-path grammar.  Produces the same plan SHAPES the reference's
plugins expect: Projection / Aggregate / Filter / Join / SubqueryAlias / TableScan."""
from typing import Callable, Dict, List, Optional, Tuple

from .. import rand as R
from .. import temporal as T
from ..utils import ParsingException
from . import plan as P
from .plan import PyExpr, RelDataTypeField
from .sqlparse import Node

_NUMERIC = ("BIGINT", "DOUBLE", "INTEGER", "FLOAT", "SMALLINT", "TINYINT", "REAL", "DECIMAL")
_CAST_TYPES = {"BIGINT": "BIGINT", "INT": "BIGINT", "INTEGER": "BIGINT", "SMALLINT": "BIGINT", "TINYINT": "BIGINT",
               "DOUBLE": "DOUBLE", "FLOAT": "DOUBLE", "REAL": "DOUBLE", "DECIMAL": "DOUBLE", "NUMERIC": "DOUBLE",
               "BOOLEAN": "BOOLEAN", "BOOL": "BOOLEAN", "VARCHAR": "VARCHAR", "STRING": "VARCHAR", "TEXT": "VARCHAR",
               "DATE": "DATE", "TIMESTAMP": "TIMESTAMP"}
_TEMPORAL = ("DATE", "TIMESTAMP")


def _norm_type(t: str) -> str:
    """Physical family of a SQL type: ints -> BIGINT, floats -> DOUBLE."""
    if t in ("INTEGER", "SMALLINT", "TINYINT", "BIGINT"):
        return "BIGINT"
    if t in ("FLOAT", "REAL", "DECIMAL", "DOUBLE"):
        return "DOUBLE"
    return t


def _arith_type(a: str, b: str) -> str:
    a, b = _norm_type(a), _norm_type(b)
    if "DOUBLE" in (a, b):
        return "DOUBLE"
    if a == "NULL":
        return b
    if b == "NULL":
        return a
    return "BIGINT"


class Binder:
    def __init__(self, sql: str, catalog: Callable[[Optional[str], str], Optional[Tuple[str, List[Tuple[str, str]]]]],
                 case_sensitive: bool = True):
        """catalog(schema_or_None, table) -> (schema_name, [(column, sql_type), ...]) or None."""
        self.sql, self.catalog, self.case_sensitive = sql, catalog, case_sensitive
        self._key = None          # the statement's key for RAND / TABLESAMPLE without a seed
        self.volatile = False     # the statement drew that key: re-planning it must draw a new one
        # subqueries: the scope of the block enclosing the one being bound (None: a derived table, CTE, ON,
        # GROUP BY ... where no correlation is allowed), the correlated conjuncts of each subquery's WHERE, and
        # the common table expressions each block sees
        self._outer: List[Optional[list]] = []
        self._corr: List[list] = []
        self._kind: List[str] = []          # "in" | "exists" | "scalar": the subquery each _corr entry is for
        self._ctes: List[dict] = []
        self._joins: List[list] = []        # per block: correlated scalar subqueries to LEFT JOIN onto its rows
        self._nsq = 0

    def err(self, msg):
        raise ParsingException(self.sql, msg)

    # -- queries ------------------------------------------------------------------------------
    def bind_statement(self, node: Node) -> P.LogicalPlan:
        if node.kind == "explain":
            return P.Explain(self.bind_query(node.query, {}))
        if node.kind == "create_memory_table":
            return P.CreateMemoryTable(self.bind_query(node.query, {}), node.name, node.or_replace,
                                       node.if_not_exists, node.is_table)
        if node.kind == "create_table":
            return P.CreateTable(node.name, node.kwargs, node.or_replace, node.if_not_exists)
        if node.kind == "drop_table":
            return P.DropTable(node.name, node.if_exists)
        if node.kind == "analyze_table":
            return self.bind_analyze(node)
        return self.bind_query(node, {})

    def bind_analyze(self, node: Node) -> P.LogicalPlan:
        parts = node.name.split(".")
        schema_name, table_name = (parts[-2], parts[-1]) if len(parts) >= 2 else (None, parts[0])
        found = self.catalog(schema_name, table_name)
        if found is None:
            self.err(f"Error during planning: table '{node.name}' not found")
        schema_name, cols = found
        names = [c for c, _ in cols]
        columns = []
        for c in node.columns:
            hits = [n for n in names if n == c]
            if not hits and not self.case_sensitive:
                hits = [n for n in names if n.lower() == c.lower()]
            if len(hits) != 1:
                self.err(f"Column '{c}' not found in table '{node.name}'" if not hits else
                         f"Column '{c}' is ambiguous in table '{node.name}'")
            if hits[0] in columns:
                self.err(f"Column '{c}' is listed more than once in ANALYZE TABLE")
            columns.append(hits[0])
        return P.AnalyzeTable(schema_name, table_name.lower(), columns, columns or names)

    def bind_query(self, q: Node, ctes: Dict[str, P.LogicalPlan]) -> P.LogicalPlan:
        # a subquery body binds its WHERE with the enclosing block's scope on top of self._outer; everything
        # else of it, and any block it reads from, sees no outer scope
        correlated = bool(self._outer) and self._outer[-1] is not None
        self._outer.append(None)
        try:
            ctes = dict(ctes)
            for name, sub in q.ctes or []:
                ctes[name] = self.bind_query(sub, ctes)
            plan = self.bind_from(q.source, ctes) if q.source is not None else self._empty_relation()
        finally:
            self._outer.pop()
        self._ctes.append(ctes)
        try:
            return self._bind_block(q, plan, correlated)
        finally:
            self._ctes.pop()

    def _bind_block(self, q: Node, plan: P.LogicalPlan, correlated: bool) -> P.LogicalPlan:
        self._joins.append([])
        try:
            return self._bind_where(q, plan, correlated)
        finally:
            self._joins.pop()

    def _apply_joins(self, plan: P.LogicalPlan) -> P.LogicalPlan:
        """LEFT JOIN the grouped bodies of the correlated scalar subqueries bound so far onto `plan`"""
        for alias, body, pairs in self._joins[-1]:
            plan = P.Join(plan, P.SubqueryAlias(body, alias), "LEFT", pairs, None)
        self._joins[-1].clear()
        return plan

    def _bind_where(self, q: Node, plan: P.LogicalPlan, correlated: bool) -> P.LogicalPlan:
        corr = []
        if q.where is not None:
            pred = self.bind_expr(q.where, plan.schema)
            if pred.contains_agg():
                self.err("Aggregate functions are not allowed in WHERE")
            if pred.contains_window():
                self.err("Window functions are not allowed in WHERE")
            if correlated:
                local = []
                for c in P.conjuncts(pred):
                    (corr if _outer_columns(c) else local).append(c)
                pred = P.conjunction(local)
                corr = [self._split_correlated(c) for c in corr]
            plan = self._apply_joins(plan)
            if pred is not None:
                plan = P.Filter(plan, pred)
        self._outer.append(None)
        try:
            return self._bind_rest(q, plan, corr)
        finally:
            self._outer.pop()

    def _split_correlated(self, c: PyExpr):
        """a correlated conjunct -> (inner expression, op, outer expression): `inner op outer`"""
        if c.kind == "binary" and c.op in _FLIP and not c.contains_subquery():
            a, b = c.args
            oa, ob = _outer_columns(a), _outer_columns(b)
            ia, ib = len(a.columns()) > len(oa), len(b.columns()) > len(ob)
            if ob and not oa and not ib:
                return a, c.op, _strip_outer(b)
            if oa and not ob and not ia:
                return b, _FLIP[c.op], _strip_outer(a)
        raise NotImplementedError(f"the correlated predicate {c.display()} must compare an expression of the "
                                  "subquery's rows with an expression of the enclosing block's rows (= <> < <= > >=)")

    def _bind_rest(self, q: Node, plan: P.LogicalPlan, corr) -> P.LogicalPlan:

        # select list
        items: List[Tuple[PyExpr, Optional[str]]] = []
        for e, alias in q["items"]:
            if e.kind == "star":
                fields = [f for f in plan.schema if (e.qualifier is None or f.qualifier == e.qualifier) and
                          not (f.qualifier or "").startswith(_SQ_ALIAS)]
                if not fields:
                    self.err(f"Invalid qualifier {e.qualifier}")
                for f in fields:
                    items.append((P.col(f.qualifier, f.getName(), f.sql_type), None))
            else:
                items.append((self.bind_expr(e, plan.schema), alias))
        plan = self._apply_joins(plan)
        extra_groups = []
        if corr:
            # a correlated body outputs its select list, then the inner side of each correlated conjunct; a grouped
            # body also groups by those (equality keys only), so each group lies within one correlation group
            kind = self._kind[-1]
            aggregated = any(e.contains_agg() for e, _ in items)
            if kind == "scalar":
                if q.group_by or q.having is not None or not aggregated or len(items) != 1:
                    raise NotImplementedError("a correlated scalar subquery must be one aggregate over the correlated "
                                              "rows, without GROUP BY or HAVING")
                self._corr[-1].append(_count_kind(items[0][0]))
                items[0] = (items[0][0], "__sv")
            elif (q.group_by or q.having is not None or aggregated) and not q.group_by:
                raise NotImplementedError("a correlated IN / EXISTS subquery with an aggregate needs a GROUP BY: "
                                          "without one it is a single row even for an empty correlation group")
            if (q.group_by or aggregated) and any(op != "=" for _, op, _ in corr):
                raise NotImplementedError("a correlated subquery with GROUP BY or an aggregate is correlated by "
                                          "equality keys only")
            if q.group_by or aggregated:
                extra_groups = [inner for inner, _, _ in corr]
            if q.distinct or q.order_by or q.limit is not None or q.offset is not None or \
                    any(e.contains_window() for e, _ in items):
                raise NotImplementedError("LIMIT, ORDER BY, DISTINCT and window functions are not supported in a "
                                          "correlated subquery")
            self._corr[-1][:0] = [(inner, op, outer, len(items) + k) for k, (inner, op, outer) in enumerate(corr)]
            items = items + [(inner, f"__corr{k}") for k, (inner, _, _) in enumerate(corr)]
        aliases = {a: e for e, a in items if a}
        # window calls of ORDER BY, bound where the SELECT list's are (they may read aggregates too)
        order_windows = {j: self.bind_expr(e, plan.schema) for j, (e, _, _) in enumerate(q.order_by or [])
                         if e.kind == "window"}
        having = self.bind_expr(q.having, plan.schema, aliases) if q.having is not None else None
        if having is not None and having.contains_window():
            self.err("Window functions are not allowed in HAVING")
        if self._joins[-1]:
            raise NotImplementedError("a correlated scalar subquery in HAVING is not supported; use it in WHERE or "
                                      "the SELECT list")
        is_agg = bool(q.group_by) or any(e.contains_agg() for e, _ in items) or \
            (having is not None and having.contains_agg()) or any(w.contains_agg() for w in order_windows.values())

        if is_agg:
            group_exprs = []
            for g in q.group_by:
                if g.kind == "lit" and isinstance(g.value, int) and not isinstance(g.value, bool):
                    if not 1 <= g.value <= len(items):
                        self.err(f"GROUP BY position {g.value} is not in select list")
                    group_exprs.append(items[g.value - 1][0])
                elif g.kind == "col" and len(g.parts) == 1 and g.parts[0] in aliases and \
                        not self._resolves(g.parts[0], plan.schema):
                    group_exprs.append(aliases[g.parts[0]])
                else:
                    group_exprs.append(self.bind_expr(g, plan.schema))
            group_exprs += [x for x in extra_groups if all(x.display() != g.display() for g in group_exprs)]
            if any(g.contains_window() for g in group_exprs):
                self.err("Window functions are not allowed in GROUP BY")
            if any(g.contains_subquery() for g in group_exprs):
                raise NotImplementedError("a subquery in GROUP BY is not supported")
            agg_calls: List[PyExpr] = []

            def collect(e: PyExpr):
                if e.kind == "agg":
                    if not any(a.display() == e.display() for a in agg_calls):
                        agg_calls.append(e)
                    return
                for c in (e.window_exprs() if e.kind == "window" else e.args):
                    collect(c)

            for e, _ in items:
                collect(e)
            if having is not None:
                collect(having)
            for w in order_windows.values():
                collect(w)
            agg_plan = P.Aggregate(plan, group_exprs, agg_calls)

            def rewrite(e: PyExpr) -> PyExpr:
                for g in group_exprs:
                    if g.display() == e.display():
                        q_, n_ = g.output_field()
                        return P.col(q_, n_, g.sql_type)
                if e.kind == "agg":
                    return P.col(None, e.display(), e.sql_type)
                if e.kind == "column":
                    self.err(f"Column {e.display()} must appear in the GROUP BY clause or be used in an "
                             "aggregate function")
                out = e.clone()
                out.args = [rewrite(a) for a in e.args]
                if e.kind == "window":
                    out.partition = [rewrite(x) for x in e.partition]
                    out.order = [(rewrite(x), a, nf) for x, a, nf in e.order]
                return out

            plan = agg_plan
            if having is not None:
                plan = P.Filter(plan, rewrite(having))
            items = [(rewrite(e), alias) for e, alias in items]
            order_windows = {j: rewrite(w) for j, w in order_windows.items()}

        # window calls: computed by a Window node between the rows they read and the projection
        windows: List[PyExpr] = []

        def collect_windows(e: PyExpr):
            if e.kind == "window":
                if not any(w.display() == e.display() for w in windows):
                    windows.append(e)
                return
            for c in e.children():
                collect_windows(c)

        def window_columns(e: PyExpr) -> PyExpr:
            if e.kind == "window":
                return P.col(None, e.display(), e.sql_type)
            out = e.clone()
            out.args = [window_columns(a) for a in e.args]
            return out

        for e, _ in items:
            collect_windows(e)
        for w in order_windows.values():
            collect_windows(w)
        if windows:
            plan = P.Window(plan, windows)
            items = [(window_columns(e), a) for e, a in items]
        proj = [PyExpr("alias", e.sql_type, name=a, args=[e]) if a else e for e, a in items]
        # an ORDER BY window call that the SELECT list does not output rides along as a hidden column, dropped
        # again after the sort
        def passes(e):       # the Window column a projection item outputs unchanged, or None
            inner = e.args[0] if e.kind == "alias" else e
            return inner.name if inner.kind == "column" and inner.qualifier is None else None

        hidden = []
        for w in order_windows.values():
            if all(passes(e) != w.display() for e in proj + hidden):
                hidden.append(P.col(None, w.display(), w.sql_type))
        if hidden and q.distinct:
            raise NotImplementedError("with SELECT DISTINCT, a window function in ORDER BY must also be in the "
                                      "SELECT list")
        plan = P.Projection(plan, proj + hidden)
        visible = plan.schema[:len(proj)]

        if q.distinct:
            plan = P.Distinct(plan)
        if q.order_by:
            keys = []
            for e, asc, nulls_first in q.order_by:
                if e.kind == "lit" and isinstance(e.value, int) and not isinstance(e.value, bool):
                    f = plan.schema[e.value - 1]
                    b = P.col(f.qualifier, f.getName(), f.sql_type)
                elif e.kind == "window":
                    # by the Window node's output column, which the projection passes on
                    w = order_windows[len(keys)]
                    f = plan.schema[next(i for i, x in enumerate(proj + hidden) if passes(x) == w.display())]
                    b = P.col(f.qualifier, f.getName(), f.sql_type)
                else:
                    b = self.bind_expr(e, plan.schema, order_by_fallback=items)
                if b.contains_subquery():
                    raise NotImplementedError("a subquery in ORDER BY is not supported")
                keys.append((b, asc, (not asc) if nulls_first is None else nulls_first))
            plan = P.Sort(plan, keys)
        if q.limit is not None or q.offset is not None:
            fetch = q.limit.value if q.limit is not None else None
            skip = q.offset.value if q.offset is not None else 0
            plan = P.Limit(plan, skip, fetch)
        if hidden:
            plan = P.Projection(plan, [P.col(f.qualifier, f.getName(), f.sql_type) for f in visible])
        return plan

    def _empty_relation(self):
        p = P.LogicalPlan()
        p.node_type = "EmptyRelation"
        return p

    def _resolves(self, name, scope) -> bool:
        return any(f.getName() == name for f in scope)

    # -- FROM ---------------------------------------------------------------------------------
    def bind_from(self, src: Node, ctes) -> P.LogicalPlan:
        if src.kind == "table":
            parts = src.name
            if len(parts) == 1 and parts[0] in ctes:
                if src.sample is not None:
                    self._no_sample(f"the common table expression {parts[0]}")
                return P.SubqueryAlias(ctes[parts[0]], src.alias or parts[0])
            schema_name, table_name = (parts[-2], parts[-1]) if len(parts) >= 2 else (None, parts[0])
            found = self.catalog(schema_name, table_name)
            if found is None:
                self.err(f"Error during planning: table '{'.'.join(parts)}' not found")
            schema_name, cols = found
            fields = [RelDataTypeField(None, c, t, i) for i, (c, t) in enumerate(cols)]
            scan = P.TableScan(schema_name, table_name.lower(), table_name if not src.alias else table_name, fields)
            if src.sample is not None:
                scan.sample = self._bind_sample(src.sample)
            return P.SubqueryAlias(scan, src.alias) if src.alias else scan
        if src.kind == "subquery":
            if src.sample is not None:
                self._no_sample("a subquery")
            return P.SubqueryAlias(self.bind_query(src.query, ctes), src.alias)
        if src.kind == "join":
            left, right = self.bind_from(src.left, ctes), self.bind_from(src.right, ctes)
            if src.how == "CROSS" or src.on is None:
                return P.CrossJoin(left, right)
            scope = left.schema + right.schema
            nleft = len(left.schema)
            if src.on.kind == "using":
                pairs = []
                for c in src.on.cols:
                    lf = [f for f in left.schema if f.getName() == c]
                    rf = [f for f in right.schema if f.getName() == c]
                    if len(lf) != 1 or len(rf) != 1:
                        self.err(f"USING column {c} must exist exactly once on both sides")
                    pairs.append((P.col(lf[0].qualifier, c, lf[0].sql_type), P.col(rf[0].qualifier, c, rf[0].sql_type)))
                return P.Join(left, right, src.how, pairs, None)
            cond = self.bind_expr(src.on, scope)
            if cond.contains_subquery():
                raise NotImplementedError("a subquery in a JOIN's ON clause is not supported")
            pairs, residual = [], []
            holder = P.LogicalPlan()
            holder.schema = scope
            for c in P.conjuncts(cond):
                if c.kind == "binary" and c.op == "=" and c.args[0].kind == "column" and c.args[1].kind == "column":
                    a, b = c.args
                    ia, ib = a.with_inputs([holder]).getIndex(), b.with_inputs([holder]).getIndex()
                    if ia < nleft <= ib:
                        pairs.append((a, b))
                        continue
                    if ib < nleft <= ia:
                        pairs.append((b, a))
                        continue
                residual.append(c)
            return P.Join(left, right, src.how, pairs, P.conjunction(residual))
        self.err(f"Unsupported FROM item {src.kind}")

    # -- expressions --------------------------------------------------------------------------
    def bind_expr(self, e: Node, scope, aliases=None, order_by_fallback=None) -> PyExpr:
        k = e.kind
        if k == "lit":
            return P.lit(e.value)
        if k == "typed_lit":
            try:
                return P.lit(T.parse_date(e.value) if e.type == "DATE" else T.parse_timestamp(e.value))
            except ValueError as err:
                self.err(str(err))
        if k == "interval":
            try:
                return P.lit(T.parse_interval(e.value, e.unit))
            except ValueError as err:
                self.err(str(err))
        if k == "col":
            parts = e.parts
            if len(parts) == 1:
                name = parts[0]
                hits = [f for f in scope if f.getName() == name]
                if not hits and not self.case_sensitive:
                    hits = [f for f in scope if f.getName().lower() == name.lower()]
                if len(hits) == 1:
                    return P.col(hits[0].qualifier, hits[0].getName(), hits[0].sql_type)
                if len(hits) > 1:
                    if len({(h.qualifier, h.getName()) for h in hits}) == 1:
                        return P.col(hits[0].qualifier, hits[0].getName(), hits[0].sql_type)
                    self.err(f"Schema error: Ambiguous reference to unqualified field {name}")
                if aliases and name in aliases:
                    return aliases[name]
                if order_by_fallback:
                    for ex, al in order_by_fallback:
                        if al == name:
                            return P.col(None, name, ex.sql_type)
                outer = self._outer_column(e.parts)
                if outer is not None:
                    return outer
                self.err(f"Schema error: No field named {name}. Valid fields are "
                         f"{', '.join(f.getQualifiedName() for f in scope)}.")
            qual, name = parts[-2], parts[-1]
            hits = [f for f in scope if f.getName() == name and f.qualifier == qual]
            if len(hits) >= 1:
                return P.col(qual, name, hits[0].sql_type)
            outer = self._outer_column(e.parts)
            if outer is not None:
                return outer
            self.err(f"Schema error: No field named {qual}.{name}. Valid fields are "
                     f"{', '.join(f.getQualifiedName() for f in scope)}.")
        rec = lambda x: self.bind_expr(x, scope, aliases, order_by_fallback)  # noqa: E731
        if k == "bin":
            l, r = rec(e.l), rec(e.r)
            op = e.op
            if op in ("AND", "OR"):
                return PyExpr("binary", "BOOLEAN", op=op, args=[l, r])
            if op in ("=", "!=", "<", "<=", ">", ">="):
                return PyExpr("binary", "BOOLEAN", op=op, args=[l, r])
            if op in ("+", "-", "*", "/", "%"):
                if {l.sql_type, r.sql_type} & {"DATE", "TIMESTAMP", "INTERVAL"}:
                    return PyExpr("binary", self._temporal_arith(op, l, r), op=op, args=[l, r])
                return PyExpr("binary", _arith_type(l.sql_type, r.sql_type), op=op, args=[l, r])
            self.err(f"Unsupported operator {op}")
        if k == "not":
            return PyExpr("not", "BOOLEAN", args=[rec(e.e)])
        if k == "neg":
            inner = rec(e.e)
            return PyExpr("negative", _norm_type(inner.sql_type), args=[inner])
        if k == "isnull":
            return PyExpr("isnotnull" if e.negated else "isnull", "BOOLEAN", args=[rec(e.e)])
        if k == "istrue":
            return PyExpr("istrue", "BOOLEAN", args=[rec(e.e)], negated=e.negated, value=e.value)
        if k == "between":
            return PyExpr("between", "BOOLEAN", args=[rec(e.e), rec(e.lo), rec(e.hi)], negated=e.negated)
        if k == "inlist":
            return PyExpr("inlist", "BOOLEAN", args=[rec(e.e)] + [rec(i) for i in e["items"]], negated=e.negated)
        if k == "like":
            x, pattern = rec(e.e), rec(e.pattern)
            if pattern.kind != "literal" or not isinstance(pattern.value, (str, type(None))):
                raise NotImplementedError("[NOT] LIKE / ILIKE takes a string literal pattern")
            if x.sql_type not in ("VARCHAR", "NULL"):
                self.err(f"{'ILIKE' if e.ilike else 'LIKE'} takes a VARCHAR operand, not {x.sql_type}")
            return PyExpr("like", "BOOLEAN", name="ilike" if e.ilike else "like", args=[x, pattern],
                          negated=e.negated, value=e.escape)
        if k == "cast":
            ty = _CAST_TYPES.get(e.type)
            if ty is None:
                self.err(f"Unsupported CAST target type {e.type}")
            if ty == "VARCHAR":
                raise NotImplementedError("CAST to VARCHAR is not supported: VARCHAR columns are dictionary codes")
            return PyExpr("cast", ty, args=[rec(e.e)])
        if k == "case":
            args = []
            for w, t in e.whens:
                args += [rec(w), rec(t)]
            if e.other is not None:
                args.append(rec(e.other))
            thens = [args[i] for i in range(1, len(args) - (len(args) % 2), 2)] + \
                    ([args[-1]] if len(args) % 2 else [])
            ty = "NULL"
            for t in thens:
                ty = _arith_type(ty, t.sql_type) if t.sql_type in _NUMERIC + ("NULL",) and ty in _NUMERIC + ("NULL",) \
                    else t.sql_type
            return PyExpr("case", ty, args=args)
        if k == "window":
            return self._bind_window(e, rec)
        if k in ("insubquery", "exists", "scalarsubquery"):
            return self._bind_subquery(e, scope, rec)
        if k == "func":
            name = e.name
            if name in _WINDOW_ONLY:
                raise NotImplementedError(f"{name} is a window function: it needs an OVER (...) clause")
            if name in P.AGG_FUNCS:
                name = "AVG" if name == "MEAN" else name
                args = [] if e.star else [rec(a) for a in e.args]
                if name.startswith("REGR_"):
                    if len(args) != 2:
                        self.err(f"{name} takes exactly two arguments")
                    if any(a.sql_type not in _NUMERIC + ("NULL",) for a in args):
                        self.err(f"{name} takes numeric arguments")
                elif name != "COUNT" and len(args) != 1:
                    self.err(f"{name} takes exactly one argument")
                if any(a.contains_agg() for a in args):
                    self.err("Aggregate function calls cannot be nested")
                if any(a.contains_window() for a in args):
                    self.err(f"A window function cannot be the argument of the aggregate {name}")
                if name not in ("COUNT", "MIN", "MAX") and any(a.sql_type == "VARCHAR" for a in args):
                    raise NotImplementedError(f"{name} of a VARCHAR: only COUNT, MIN and MAX aggregate strings")
                if name not in ("COUNT", "MIN", "MAX") and any(a.sql_type in _TEMPORAL for a in args):
                    raise NotImplementedError(f"{name} of a {args[0].sql_type}: only COUNT, MIN and MAX aggregate "
                                              "dates and timestamps")
                if name.startswith("BIT_") and args[0].sql_type not in ("BIGINT", "INTEGER", "SMALLINT", "TINYINT"):
                    self.err(f"{name} takes an integer argument, not {args[0].sql_type}")
                if name == "EVERY" and args[0].sql_type != "BOOLEAN":
                    self.err(f"{name} takes a BOOLEAN argument, not {args[0].sql_type}")
                if name in ("COUNT", "REGR_COUNT"):
                    ty = "BIGINT"
                elif name == "AVG" or name.startswith(("STDDEV", "VAR", "REGR_")):
                    ty = "DOUBLE"
                elif name == "SUM":
                    ty = _norm_type(args[0].sql_type) if args[0].sql_type != "BOOLEAN" else "BIGINT"
                else:
                    ty = args[0].sql_type
                filt = rec(e.filter) if e.filter is not None else None
                if filt is not None and filt.contains_window():
                    self.err(f"A window function cannot be in the FILTER clause of the aggregate {name}")
                return PyExpr("agg", ty, name=name, args=args, distinct=e.distinct, filter=filt)
            if name in _TEMPORAL_FUNCS:
                return self._bind_temporal(name, e.args, rec)
            if name in _RAND_FUNCS:
                return self._bind_rand(name, e)
            args = [rec(a) for a in e.args]
            if name == "ABS" and len(args) == 1:
                return PyExpr("scalarfn", _norm_type(args[0].sql_type), name="abs", args=args)
            if name in _MATH_UNARY + _MATH_BINARY:
                return self._bind_math(name, args)
            self.err(f"Function {name} is outside the int64/float64 hot path of this layer")
        self.err(f"Unsupported expression {k}")

    # -- subqueries -----------------------------------------------------------------------------
    def _outer_column(self, parts) -> Optional[PyExpr]:
        """a column of the immediately enclosing block, for the WHERE of a correlated subquery"""
        def find(scope):
            if len(parts) == 1:
                hits = [f for f in scope if f.getName() == parts[0] or
                        (not self.case_sensitive and f.getName().lower() == parts[0].lower())]
            else:
                hits = [f for f in scope if f.getName() == parts[-1] and f.qualifier == parts[-2]]
            if len({(h.qualifier, h.getName()) for h in hits}) > 1:
                self.err(f"Schema error: Ambiguous reference to unqualified field {parts[-1]}")
            return hits[0] if hits else None

        if self._outer and self._outer[-1] is not None:
            f = find(self._outer[-1])
            if f is not None:
                return PyExpr("column", f.sql_type, qualifier=f.qualifier, name=f.getName(), value=_OUTER)
        if any(scope is not None and find(scope) is not None for scope in self._outer[:-1]):
            raise NotImplementedError(f"the column {'.'.join(parts)} belongs to a block that encloses this one "
                                      "further out, or is used outside a subquery's WHERE: a correlated subquery "
                                      "may refer to the immediately enclosing block, in its WHERE only")
        return None

    def _bind_subquery(self, e: Node, scope, rec) -> PyExpr:
        """[NOT] IN (SELECT ...), EXISTS (SELECT ...) and (SELECT ...): the body is bound and optimised on its
        own; correlated conjuncts of its WHERE become equality keys (inner = outer) and pair terms (the other
        comparisons), and the IN's own x = y is the key of an uncorrelated IN, a pair term of a correlated one."""
        from .optimizer import optimize
        self._outer.append(scope)
        self._corr.append([])
        self._kind.append({"insubquery": "in", "exists": "exists", "scalarsubquery": "scalar"}[e.kind])
        try:
            body = self.bind_query(e.query, self._ctes[-1] if self._ctes else {})
        finally:
            self._outer.pop()
            self._kind.pop()
            corr = self._corr.pop()
        count_kind = corr.pop() if e.kind == "scalarsubquery" and corr else None
        body = optimize(body)
        width = len(body.schema) - len(corr)
        keys = [(outer, out) for _, op, outer, out in corr if op == "="]
        terms = [(outer, out, _FLIP[op], True) for _, op, outer, out in corr if op != "="]
        if e.kind == "scalarsubquery":
            if width != 1:
                self.err(f"A scalar subquery returns one column, not {width}")
            ty = body.schema[0].sql_type
            if corr:
                return self._join_scalar(body, keys, count_kind, ty)
            if ty in _TEMPORAL:
                raise NotImplementedError(f"a scalar subquery of type {ty} is not supported")
            self.volatile = True                # its value is read when the statement is planned
            return PyExpr("subquery", ty, name="scalar subquery", value=P.Subquery(body, "scalar", [], [], False))
        if corr and not keys:
            raise NotImplementedError("a correlated IN / EXISTS subquery needs an equality key: a conjunct "
                                      "inner_expr = outer_expr in its WHERE")
        null_aware = False
        if e.kind == "insubquery":
            if width != 1:
                self.err(f"IN (subquery) takes a subquery of one column, not {width}")
            x = rec(e.e)
            if corr:
                terms.append((x, 0, "=", False))
            else:
                keys, null_aware = [(x, 0)], True
        names = [f for f in body.schema]
        if any(o.sql_type == "VARCHAR" or names[k].sql_type == "VARCHAR" for o, k, _, _ in terms):
            raise NotImplementedError("a correlated subquery compares VARCHAR expressions by equality keys only")
        if len(terms) > P.MARK_MAX_TERMS:
            raise NotImplementedError(f"a correlated subquery compares at most {P.MARK_MAX_TERMS} pairs of "
                                      f"expressions other than by equality keys, not {len(terms)}")
        spec = P.Subquery(body, "in" if e.kind == "insubquery" else "exists", [k for _, k in keys],
                          [(k, op, where) for _, k, op, where in terms], null_aware)
        out = PyExpr("subquery", "BOOLEAN", name="in subquery" if e.kind == "insubquery" else "exists",
                     args=[o for o, _ in keys] + [o for o, _, _, _ in terms], value=spec)
        return PyExpr("not", "BOOLEAN", args=[out]) if e.negated else out

    def _join_scalar(self, body, keys, count_kind, ty) -> PyExpr:
        """A correlated scalar subquery, decorrelated as DataFusion's scalar-subquery-to-join rule does: the body
        grouped by its inner key expressions, LEFT JOINed onto the enclosing block's rows on the outer keys; the
        value is its aggregate column, NULL for a row without a group, and COUNT's 0 there (COALESCE)."""
        if count_kind == "mixed":
            raise NotImplementedError("a correlated scalar subquery that uses COUNT inside an expression is not "
                                      "supported; use the COUNT alone")
        pairs = []
        self._nsq += 1
        alias = f"{_SQ_ALIAS}{self._nsq}"
        for outer, k in keys:
            if outer.kind != "column":
                raise NotImplementedError(f"a correlated scalar subquery is joined on columns of the enclosing block, "
                                          f"not on {outer.display()}")
            f = body.schema[k]
            pairs.append((outer, P.col(alias, f.getName(), f.sql_type)))
        self._joins[-1].append((alias, body, pairs))
        v = P.col(alias, body.schema[0].getName(), ty)
        if count_kind == "count":
            v = PyExpr("case", ty, args=[PyExpr("isnull", "BOOLEAN", args=[v]), P.lit(0), v.clone()])
        return v

    # -- window calls ---------------------------------------------------------------------------
    def _bind_window(self, node, rec) -> PyExpr:
        """f(args) OVER (PARTITION BY ... ORDER BY ... frame): frame -> (is_range, lo, hi), offsets from the row,
        -inf / +inf for UNBOUNDED.  Without ORDER BY the default frame is the whole partition; with it, RANGE
        BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW (through the row's last peer)."""
        f = node.func
        name = "AVG" if f.name == "MEAN" else f.name
        if name in _WINDOW_REFUSED:
            raise NotImplementedError(f"{name} is not supported as a window function; the window functions are "
                                      f"{', '.join(P.WINDOW_FUNCS)}")
        if name not in P.WINDOW_FUNCS:
            if name in P.AGG_FUNCS:
                raise NotImplementedError(f"{name} OVER (...) is not supported; the window aggregates are COUNT, SUM, "
                                          "AVG, MIN and MAX")
            self.err(f"{name} is not a window function")
        if f.distinct:
            raise NotImplementedError(f"{name}(DISTINCT ...) OVER (...) is not supported")
        if f.filter is not None:
            raise NotImplementedError(f"{name}(...) FILTER (WHERE ...) OVER (...) is not supported")
        args = [] if f.star else [rec(a) for a in f.args]
        if any(a.contains_window() for a in args):
            self.err("Window function calls cannot be nested")
        if name in ("ROW_NUMBER", "RANK", "DENSE_RANK"):
            if args or f.star:
                self.err(f"{name} takes no arguments")
        elif name == "COUNT":
            if len(args) > 1:
                self.err("COUNT takes one argument or *")
        elif len(args) != 1:
            self.err(f"{name} takes exactly one argument")
        if name in ("SUM", "AVG") and (args[0].sql_type == "VARCHAR" or args[0].sql_type in _TEMPORAL):
            raise NotImplementedError(f"{name} of a {args[0].sql_type}: only COUNT, MIN, MAX, FIRST_VALUE and "
                                      "LAST_VALUE take strings, dates and timestamps")
        if name in ("ROW_NUMBER", "RANK", "DENSE_RANK", "COUNT"):
            ty = "BIGINT"
        elif name == "AVG":
            ty = "DOUBLE"
        elif name == "SUM":
            ty = _norm_type(args[0].sql_type) if args[0].sql_type != "BOOLEAN" else "BIGINT"
        else:
            ty = args[0].sql_type
        partition = [rec(p) for p in node.partition]
        order = [(rec(x), asc, (not asc) if nf is None else nf) for x, asc, nf in node.order]
        if any(x.contains_window() for x in partition + [o for o, _, _ in order]):
            self.err("Window function calls cannot be nested")
        inf = float("inf")
        if node.frame is None:
            frame = (True, -inf, 0) if order else (False, -inf, inf)
        else:
            fr = node.frame

            def bound(b):
                kind, v = b
                return v * inf if kind == "unbounded" else v

            if fr.unit == "RANGE" and "offset" in (fr.lo[0], fr.hi[0]):
                raise NotImplementedError("RANGE frames with an offset (n PRECEDING / FOLLOWING) are not supported; "
                                          "use ROWS, or RANGE with UNBOUNDED and CURRENT ROW bounds")
            lo, hi = bound(fr.lo), bound(fr.hi)
            if lo == inf:
                self.err("A window frame cannot start at UNBOUNDED FOLLOWING")
            if hi == -inf:
                self.err("A window frame cannot end at UNBOUNDED PRECEDING")
            frame = (fr.unit == "RANGE", lo, hi)
        return PyExpr("window", ty, name=name, args=args, partition=partition, order=order, frame=frame)

    # -- RAND / RANDOM / RAND_INTEGER and TABLESAMPLE ------------------------------------------
    @staticmethod
    def _int_literal(node):
        """the value of an integer literal node (a negated one included), else None"""
        neg = node.kind == "neg"
        lit = node.e if neg else node
        if lit is None or lit.kind != "lit" or not isinstance(lit.value, int) or isinstance(lit.value, bool):
            return None
        return -lit.value if neg else lit.value

    def _key_of(self, seed_node, what) -> int:
        """the Philox key of a seed argument; no seed: the statement's key, drawn once per statement"""
        if seed_node is None:
            if self._key is None:
                self._key, self.volatile = R.key_of(None), True
            return self._key
        seed = self._int_literal(seed_node)
        if seed is None or not -2 ** 63 <= seed < 2 ** 64:
            self.err(f"{what} takes its seed as an integer literal")
        return R.key_of(seed)

    def _bind_rand(self, name, e) -> PyExpr:
        """RAND([seed]) / RANDOM([seed]) -> DOUBLE in [0, 1); RAND_INTEGER([seed,] h) -> BIGINT in [0, h): the
        reference's operator table (call.py:1087-1089), keyed per call site and row (rand.py)."""
        args = e.args
        if name == "RAND_INTEGER":
            if len(args) not in (1, 2):
                self.err(f"RAND_INTEGER takes 1 or 2 argument(s), not {len(args)}")
            h = self._int_literal(args[-1])
            if h is None or not 0 < h < 2 ** 63:
                self.err("RAND_INTEGER takes its bound h as a positive BIGINT literal")
            key = self._key_of(args[0] if len(args) == 2 else None, name)
            return PyExpr("scalarfn", "BIGINT", name="rand_integer", args=[P.lit(key), P.lit(e.site), P.lit(h)])
        if len(args) > 1:
            self.err(f"{name} takes 0 or 1 argument(s), not {len(args)}")
        key = self._key_of(args[0] if args else None, name)
        return PyExpr("scalarfn", "DOUBLE", name="rand", args=[P.lit(key), P.lit(e.site)])

    def _no_sample(self, what):
        raise NotImplementedError(f"TABLESAMPLE of {what}: only the rows of a base table have numbers to sample by")

    def _bind_sample(self, node) -> R.Sample:
        """TABLESAMPLE BERNOULLI | SYSTEM (p) [REPEATABLE (seed)]: p a numeric literal in [0, 100]"""
        p = node.p
        neg = p.kind == "neg"
        lit = p.e if neg else p
        if lit is None or lit.kind != "lit" or not isinstance(lit.value, (int, float)) or isinstance(lit.value, bool):
            self.err("TABLESAMPLE takes its percentage as a numeric literal")
        value = -lit.value if neg else lit.value
        if not 0 <= value <= 100:
            self.err(f"TABLESAMPLE percentage {value} is outside [0, 100]")
        return R.Sample(node.method, value, self._key_of(node.seed, "TABLESAMPLE ... REPEATABLE"), node.site)

    # -- numeric functions --------------------------------------------------------------------
    def _bind_math(self, name, args) -> PyExpr:
        """The numeric functions of the reference's operator table (call.py:1091-1113) and SQRT.  Result types:
        DataFusion's built-ins, and the reference's UDFs, which return Float64 (src/sql.rs:316-325); POWER of
        two integers stays BIGINT."""
        arity = (1, 2) if name == "ROUND" else (2,) if name in _MATH_BINARY else (1,)
        if len(args) not in arity:
            self.err(f"{name} takes {' or '.join(map(str, arity))} argument(s), not {len(args)}")
        values = args[:1] if name == "ROUND" else args
        for a in values:
            if _norm_type(a.sql_type) not in ("BIGINT", "DOUBLE", "NULL"):
                self.err(f"{name} takes numeric arguments, not {a.sql_type}")
        if name == "ROUND" and len(args) == 2:
            d = args[1]
            lit = d.args[0] if d.kind == "negative" else d
            if lit.kind != "literal" or not isinstance(lit.value, int) or isinstance(lit.value, bool):
                if d.kind != "literal" and _norm_type(d.sql_type) == "BIGINT":
                    raise NotImplementedError("ROUND(x, d) takes its digits d as an integer literal only")
                self.err(f"ROUND takes its digits as an integer literal, not {d.display()}")
        ty = "DOUBLE"
        if name == "POWER" and "DOUBLE" not in [_norm_type(a.sql_type) for a in args]:
            ty = "BIGINT"
        return PyExpr("scalarfn", ty, name=name.lower(), args=args)

    # -- DATE / TIMESTAMP ---------------------------------------------------------------------
    def _temporal_arith(self, op, l, r) -> str:
        """DATE / TIMESTAMP +- INTERVAL keeps its type; a DATE plus a sub-day interval is a TIMESTAMP."""
        if op in ("+", "-") and r.sql_type == "INTERVAL" and l.sql_type in _TEMPORAL + ("NULL",):
            if l.sql_type == "DATE" and r.kind == "literal" and r.value is not None and r.value.ns % T.NS_PER_DAY:
                return "TIMESTAMP"
            return l.sql_type
        if op == "+" and l.sql_type == "INTERVAL" and r.sql_type in _TEMPORAL:
            return self._temporal_arith(op, r, l)
        if op == "-" and l.sql_type in _TEMPORAL and r.sql_type in _TEMPORAL:
            raise NotImplementedError("the difference of two dates / timestamps is an interval, which is not a "
                                      "column type here; use TIMESTAMPDIFF(unit, a, b)")
        raise NotImplementedError(f"{l.sql_type} {op} {r.sql_type}: dates and timestamps take +/- INTERVAL only")

    def _unit_arg(self, node) -> str:
        """TIMESTAMPADD(YEAR, ...): the unit is a bare word (a column node) or a string."""
        word = node.parts[-1] if node.kind == "col" else node.value
        try:
            return T.norm_unit(word)
        except ValueError as err:
            self.err(str(err))

    def _temporal_arg(self, name, x):
        if x.sql_type not in _TEMPORAL + ("NULL",):
            self.err(f"{name} takes a DATE or TIMESTAMP argument, not {x.sql_type}")
        return x

    def _bind_temporal(self, name, nodes, rec) -> PyExpr:
        """EXTRACT / DATE_PART / YEAR / TIMESTAMPADD / TIMESTAMPDIFF / FLOOR, CEIL(x TO u) / LAST_DAY, under
        the operator names of the reference's table (call.py:1137-1155)."""
        want = {"EXTRACT": 2, "DATE_PART": 2, "DATEPART": 2, "YEAR": 1, "TIMESTAMPADD": 3, "TIMESTAMPDIFF": 3,
                "TIMESTAMPFLOOR": 2, "TIMESTAMPCEIL": 2, "LAST_DAY": 1}[name]
        if len(nodes) != want:
            self.err(f"{name} takes {want} argument(s)")
        if name in ("EXTRACT", "DATE_PART", "DATEPART"):
            try:
                field = T.extract_field(nodes[0].value)
            except NotImplementedError:
                self.err(f"EXTRACT: unknown field {nodes[0].value}")
            x = self._temporal_arg(name, rec(nodes[1]))
            return PyExpr("scalarfn", "DATE" if field == "DATE" else "BIGINT", name="date_part",
                          args=[P.lit(field), x])
        if name == "YEAR":
            return PyExpr("scalarfn", "BIGINT", name="year", args=[self._temporal_arg(name, rec(nodes[0]))])
        if name == "LAST_DAY":
            x = self._temporal_arg(name, rec(nodes[0]))
            return PyExpr("scalarfn", x.sql_type, name="last_day", args=[x])
        if name in ("TIMESTAMPFLOOR", "TIMESTAMPCEIL"):
            x = self._temporal_arg(name, rec(nodes[0]))
            return PyExpr("scalarfn", x.sql_type, name=name.lower(), args=[x, P.lit(self._unit_arg(nodes[1]))])
        unit = self._unit_arg(nodes[0])
        if name == "TIMESTAMPADD":
            n, x = rec(nodes[1]), self._temporal_arg(name, rec(nodes[2]))
            if n.sql_type not in ("BIGINT", "INTEGER", "SMALLINT", "TINYINT", "NULL"):
                self.err(f"TIMESTAMPADD takes an integer amount, not {n.sql_type}")
            ty = x.sql_type
            if ty == "DATE" and unit not in ("YEAR", "QUARTER", "MONTH", "WEEK", "DAY"):
                ty = "TIMESTAMP"
            return PyExpr("scalarfn", ty, name="timestampadd", args=[P.lit(unit), n, x])
        a, b = rec(nodes[1]), rec(nodes[2])
        if a.sql_type not in _TEMPORAL and b.sql_type not in _TEMPORAL:
            self.err("TIMESTAMPDIFF takes DATE or TIMESTAMP arguments")
        return PyExpr("scalarfn", "BIGINT", name="timestampdiff", args=[P.lit(unit), a, b])


_SQ_ALIAS = "__sq"      # qualifier of a decorrelated scalar subquery joined onto a block (hidden from *)
_OUTER = "outer"        # PyExpr.value of a column of the enclosing block, in a correlated subquery's WHERE
_FLIP = {"=": "=", "!=": "!=", "<": ">", "<=": ">=", ">": "<", ">=": "<="}


def _count_kind(e: PyExpr) -> Optional[str]:
    """"count": the item is COUNT / REGR_COUNT itself (0 over no rows); "mixed": a COUNT inside an expression"""
    if e.kind == "agg" and e.name in ("COUNT", "REGR_COUNT"):
        return "count"
    found = []

    def walk(x):
        if x.kind == "agg" and x.name in ("COUNT", "REGR_COUNT"):
            found.append(x)
        for c in x.args:
            walk(c)

    walk(e)
    return "mixed" if found else None


def _outer_columns(e: PyExpr) -> List[PyExpr]:
    return [c for c in e.columns() if c.value == _OUTER]


def _strip_outer(e: PyExpr) -> PyExpr:
    out = e.clone()
    for c in out.columns():
        c.value = None
    return out


_RAND_FUNCS = ("RAND", "RANDOM", "RAND_INTEGER")
_WINDOW_REFUSED = ("LAG", "LEAD", "NTILE", "NTH_VALUE", "PERCENT_RANK", "CUME_DIST", "SINGLE_VALUE")
_WINDOW_ONLY = ("ROW_NUMBER", "RANK", "DENSE_RANK", "FIRST_VALUE", "LAST_VALUE") + _WINDOW_REFUSED
_TEMPORAL_FUNCS = ("EXTRACT", "DATE_PART", "DATEPART", "YEAR", "TIMESTAMPADD", "TIMESTAMPDIFF", "TIMESTAMPFLOOR",
                   "TIMESTAMPCEIL", "LAST_DAY")
_MATH_UNARY = ("CEIL", "FLOOR", "TRUNCATE", "ROUND", "SIGN", "DEGREES", "RADIANS", "SQRT", "EXP", "LN", "LOG10", "CBRT",
               "SIN", "COS", "TAN", "COT", "ASIN", "ACOS", "ATAN")
_MATH_BINARY = ("ATAN2", "POWER", "MOD")
