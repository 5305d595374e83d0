"""Syntax tree -> logical plan (the job of DataFusion's SqlToRel in the reference,
src/sql.rs:586-596), for the hot-path grammar.  Produces the same plan SHAPES the reference's
plugins expect: Projection / Aggregate / Filter / Join / SubqueryAlias / TableScan."""
from typing import Callable, Dict, List, Optional, Tuple

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
        return self.bind_query(node, {})

    def bind_query(self, q: Node, ctes: Dict[str, P.LogicalPlan]) -> P.LogicalPlan:
        ctes = dict(ctes)
        for name, sub in q.ctes or []:
            ctes[name] = self.bind_query(sub, ctes)
        plan = self.bind_from(q.source, ctes) if q.source is not None else self._empty_relation()
        if q.where is not None:
            pred = self.bind_expr(q.where, plan.schema)
            if pred.contains_agg():
                self.err("Aggregate functions are not allowed in WHERE")
            plan = P.Filter(plan, pred)

        # select list
        items: List[Tuple[PyExpr, Optional[str]]] = []
        for e, alias in q["items"]:
            if e.kind == "star":
                fields = [f for f in plan.schema if e.qualifier is None or f.qualifier == e.qualifier]
                if not fields:
                    self.err(f"Invalid qualifier {e.qualifier}")
                for f in fields:
                    items.append((P.col(f.qualifier, f.getName(), f.sql_type), None))
            else:
                items.append((self.bind_expr(e, plan.schema), alias))
        aliases = {a: e for e, a in items if a}
        having = self.bind_expr(q.having, plan.schema, aliases) if q.having is not None else None
        is_agg = bool(q.group_by) or any(e.contains_agg() for e, _ in items) or \
            (having is not None and having.contains_agg())

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
            agg_calls: List[PyExpr] = []

            def collect(e: PyExpr):
                if e.kind == "agg":
                    if not any(a.display() == e.display() for a in agg_calls):
                        agg_calls.append(e)
                    return
                for c in e.args:
                    collect(c)

            for e, _ in items:
                collect(e)
            if having is not None:
                collect(having)
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
                return out

            plan = agg_plan
            if having is not None:
                plan = P.Filter(plan, rewrite(having))
            proj = []
            for e, alias in items:
                r = rewrite(e)
                name = alias if alias else None
                if name is None and e.kind != "column":
                    name = None  # display name of the aggregate output column
                proj.append(PyExpr("alias", r.sql_type, name=name, args=[r]) if name else r)
            plan = P.Projection(plan, proj)
        else:
            proj = [PyExpr("alias", e.sql_type, name=a, args=[e]) if a else e for e, a in items]
            plan = P.Projection(plan, proj)

        if q.distinct:
            plan = P.Distinct(plan)
        if q.order_by:
            keys = []
            for e, asc, nulls_first in q.order_by:
                if e.kind == "lit" and isinstance(e.value, int) and not isinstance(e.value, bool):
                    f = plan.schema[e.value - 1]
                    b = P.col(f.qualifier, f.getName(), f.sql_type)
                else:
                    b = self.bind_expr(e, plan.schema, order_by_fallback=items)
                keys.append((b, asc, (not asc) if nulls_first is None else nulls_first))
            plan = P.Sort(plan, keys)
        if q.limit is not None or q.offset is not None:
            fetch = q.limit.value if q.limit is not None else None
            skip = q.offset.value if q.offset is not None else 0
            plan = P.Limit(plan, skip, fetch)
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
                return P.SubqueryAlias(ctes[parts[0]], src.alias or parts[0])
            schema_name, table_name = (parts[-2], parts[-1]) if len(parts) >= 2 else (None, parts[0])
            found = self.catalog(schema_name, table_name)
            if found is None:
                self.err(f"Error during planning: table '{'.'.join(parts)}' not found")
            schema_name, cols = found
            fields = [RelDataTypeField(None, c, t, i) for i, (c, t) in enumerate(cols)]
            scan = P.TableScan(schema_name, table_name.lower(), table_name if not src.alias else table_name, fields)
            return P.SubqueryAlias(scan, src.alias) if src.alias else scan
        if src.kind == "subquery":
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
                self.err(f"Schema error: No field named {name}. Valid fields are "
                         f"{', '.join(f.getQualifiedName() for f in scope)}.")
            qual, name = parts[-2], parts[-1]
            hits = [f for f in scope if f.getName() == name and f.qualifier == qual]
            if len(hits) >= 1:
                return P.col(qual, name, hits[0].sql_type)
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
        if k == "func":
            name = e.name
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
                return PyExpr("agg", ty, name=name, args=args, distinct=e.distinct, filter=filt)
            if name in _TEMPORAL_FUNCS:
                return self._bind_temporal(name, e.args, rec)
            args = [rec(a) for a in e.args]
            if name == "ABS" and len(args) == 1:
                return PyExpr("scalarfn", _norm_type(args[0].sql_type), name="abs", args=args)
            if name in _MATH_UNARY + _MATH_BINARY:
                return self._bind_math(name, args)
            self.err(f"Function {name} is outside the int64/float64 hot path of this layer")
        self.err(f"Unsupported expression {k}")

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


_TEMPORAL_FUNCS = ("EXTRACT", "DATE_PART", "DATEPART", "YEAR", "TIMESTAMPADD", "TIMESTAMPDIFF", "TIMESTAMPFLOOR",
                   "TIMESTAMPCEIL", "LAST_DAY")
_MATH_UNARY = ("CEIL", "FLOOR", "TRUNCATE", "ROUND", "SIGN", "DEGREES", "RADIANS", "SQRT", "EXP", "LN", "LOG10", "CBRT",
               "SIN", "COS", "TAN", "COT", "ASIN", "ACOS", "ATAN")
_MATH_BINARY = ("ATAN2", "POWER", "MOD")
