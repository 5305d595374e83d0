"""Lazy, device-resident frame objects: the execution layer's stand-in for dask.dataframe.

The reference's plugins return DataContainer(df, cc) where df is a lazy dask DataFrame that
supports df[cols], df[mask], .assign, .merge, .groupby().agg, .columns, .dtypes, .compute()
(SURVEY 8b; datacontainer.py:190-231, context.py:908-910).  LazyFrame offers that surface, but
instead of a task graph of pandas calls it records

    source  (device table | join | aggregate)
    exprs   {output column -> expression over the source's columns}
    pred    [conjuncts over the source's columns]

so chains of Filter / Projection / TableScan nodes collapse into ONE fused kernel pass at
.compute() (executor.py) rather than one pandas pass per operator.
"""
import itertools
from collections import OrderedDict
from typing import Dict, List, Sequence

import numpy as np

from . import expr as E
from . import temporal as T
from .expr import Expr, ColRef, Lit, I64, F64, U8

_NP_DTYPE = {I64: np.dtype("int64"), F64: np.dtype("float64"), U8: np.dtype("bool")}
_uid = itertools.count()


# ---------------------------------------------------------------------------------------------
# sources
# ---------------------------------------------------------------------------------------------
class Source:
    """schema: OrderedDict name -> (dtype, logical)"""
    schema: "OrderedDict[str, tuple]"

    def colref(self, name) -> ColRef:
        dt, lg = self.schema[name]
        return ColRef(name, dt, lg)


# the U8 column of a TABLESAMPLE BERNOULLI scan that is 1 for the rows the sample keeps (b2_sample_mask); a
# sampled frame's first conjunct is this column, so every kernel that scans the table filters by it
SAMPLE_MASK = "__sample__"


class TableSource(Source):
    """sample: the TABLESAMPLE clause on this scan of the table (rand.Sample), or None.  numbered: a RAND
    draws over this source, so its scans carry every row's number in the table (executor.table_parts)."""

    def __init__(self, table, sample=None):
        self.table, self.sample = table, sample
        self.numbered = False
        self.schema = OrderedDict((n, (dt, lg)) for n, dt, lg in table.schema())
        if sample is not None and sample.method == "bernoulli":
            self.schema[SAMPLE_MASK] = (U8, "bool")


class JoinSource(Source):
    def __init__(self, left: "LazyFrame", right: "LazyFrame", left_on, right_on, how, broadcast=None):
        dup = set(left.columns) & set(right.columns)
        if dup:
            raise ValueError(f"join inputs share column names {sorted(dup)}; rename first")
        self.left, self.right = left, right
        self.left_on, self.right_on, self.how = list(left_on), list(right_on), how
        self.broadcast = broadcast
        self.schema = OrderedDict()
        for n in left.columns:
            self.schema[n] = left.col_type(n)
        if how not in ("leftsemi", "leftanti"):
            for n in right.columns:
                self.schema[n] = right.col_type(n)


MOMENT_FUNCS = ("var_samp", "var_pop", "stddev_samp", "stddev_pop", "regr_sxx", "regr_syy")


class AggSource(Source):
    """group_cols: child columns; aggs: [(input child column or None, output name, fn)] with
    fn in sum | count | mean | min | max | size | var_samp | var_pop | stddev_samp | stddev_pop | regr_sxx |
    regr_syy | bit_and | bit_or | bit_xor | every."""

    def __init__(self, child: "LazyFrame", group_cols, aggs, options=None):
        self.child, self.group_cols, self.aggs = child, list(group_cols), list(aggs)
        self.options = dict(options or {})
        self.schema = OrderedDict()
        for g in self.group_cols:
            self.schema[g] = child.col_type(g)
        for in_col, out, fn in self.aggs:
            if fn in ("count", "size"):
                self.schema[out] = (I64, "int64")
            elif fn == "mean" or fn in MOMENT_FUNCS:
                self.schema[out] = (F64, "float64")
            elif fn == "every":
                self.schema[out] = (U8, "bool")
            else:
                dt, lg = child.col_type(in_col)
                if E.is_varchar(child.exprs[in_col]) and fn not in ("min", "max"):
                    raise NotImplementedError(f"{fn.upper()} of a VARCHAR column: only COUNT, MIN and MAX aggregate "
                                              "strings")
                if T.is_temporal(lg) and fn not in ("min", "max"):
                    raise NotImplementedError(f"{fn.upper()} of a {T.sql_type_of(lg)} column: only COUNT, MIN and "
                                              "MAX aggregate dates and timestamps")
                if dt == U8:
                    dt, lg = I64, "int64"
                self.schema[out] = (dt, lg)


class SortSource(Source):
    """ORDER BY: keys = [(child column, ascending, nulls_first)], most significant first."""

    def __init__(self, child: "LazyFrame", keys):
        self.child, self.keys = child, list(keys)
        self.schema = OrderedDict((n, child.col_type(n)) for n in child.columns)


WINDOW_FUNCS = ("row_number", "rank", "dense_rank", "count", "sum", "avg", "min", "max", "first_value", "last_value")


class WindowSource(Source):
    """Window functions over the child's rows, output in the child's row order.  specs: one entry per distinct
    (PARTITION BY, ORDER BY): (partition columns, order keys [(column, ascending, nulls_first)], functions
    [(output column, fn, argument column or None, frame)]); fn is one of WINDOW_FUNCS, "count" without an
    argument is COUNT(*).  frame = (is_range, lo, hi): bounds relative to the row, -k for k PRECEDING, 0 for
    CURRENT ROW, +k for k FOLLOWING, -inf / +inf for UNBOUNDED; a RANGE frame takes only 0 and +-inf."""

    def __init__(self, child: "LazyFrame", specs):
        self.child, self.specs = child, [(list(p), list(o), list(f)) for p, o, f in specs]
        self.schema = OrderedDict((n, child.col_type(n)) for n in child.columns)
        for _, _, funcs in self.specs:
            for out, fn, arg, _ in funcs:
                self.schema[out] = self._result_type(fn, arg)

    def _result_type(self, fn, arg):
        if fn in ("row_number", "rank", "dense_rank", "count"):
            return I64, "int64"
        dt, lg = self.child.col_type(arg)
        if fn == "avg":
            return F64, "float64"
        if fn in ("first_value", "last_value"):
            return dt, lg
        if dt == U8:
            return I64, "int64"
        if fn == "sum":
            return (F64, "float64") if dt == F64 else (I64, "int64")
        return dt, lg                       # MIN / MAX keep a VARCHAR's dictionary and a DATE's type

    def inputs(self):
        """the child columns the window reads: keys and arguments"""
        out = []
        for part, order, funcs in self.specs:
            out += list(part) + [k for k, _, _ in order] + [a for _, _, a, _ in funcs if a is not None]
        return list(dict.fromkeys(out))


class MarkSource(Source):
    """The child's rows and columns plus `out`, the mark of an IN / EXISTS subquery (executor.run_mark): a
    three-valued BOOLEAN per child row.  inner: the subquery body's frame; keys: [(child column, inner
    column)] equality keys; terms: [(child column, inner column, cmp, where)] pair terms  child <cmp> inner;
    null_aware: the one key is the operand of an uncorrelated IN."""

    def __init__(self, child: "LazyFrame", inner: "LazyFrame", keys, terms, null_aware, out):
        self.child, self.inner = child, inner
        self.keys, self.terms, self.null_aware, self.out = list(keys), list(terms), null_aware, out
        self.schema = OrderedDict((n, child.col_type(n)) for n in child.columns)
        self.schema[out] = (U8, "bool")

    def inputs(self):
        """the child columns the mark reads"""
        return list(dict.fromkeys([k for k, _ in self.keys] + [t[0] for t in self.terms]))


class LimitSource(Source):
    """LIMIT / OFFSET over the child's row order."""

    def __init__(self, child: "LazyFrame", offset, fetch):
        self.child, self.offset, self.fetch = child, int(offset or 0), fetch
        self.schema = OrderedDict((n, child.col_type(n)) for n in child.columns)


# ---------------------------------------------------------------------------------------------
# series
# ---------------------------------------------------------------------------------------------
class LazySeries:
    """One lazily-evaluated column of a LazyFrame (an expression over the frame's source)."""

    def __init__(self, source: Source, pred: tuple, expr: Expr, name=None):
        self.source, self.pred, self.expr, self.name = source, pred, expr, name

    # -- pandas-ish metadata
    @property
    def dtype(self):
        if T.is_temporal(self.expr.logical):
            return T.numpy_dtype(self.expr.logical)
        if isinstance(self.expr, ColRef):
            lg = self.expr.logical
            try:
                return np.dtype(lg)
            except TypeError:
                import pandas as pd
                return pd.api.types.pandas_dtype(lg)
        return _NP_DTYPE[self.expr.dtype]

    def _wrap(self, e: Expr):
        return LazySeries(self.source, self.pred, e, self.name)

    def _other(self, o):
        if isinstance(o, LazySeries):
            if o.source is not self.source:
                raise ValueError("cannot combine columns of different frames without a join")
            return o.expr
        if isinstance(o, np.generic):
            o = o.item()
        if isinstance(o, (T.TScalar, T.Interval, str)):
            return o            # read against the other operand's type (expr.binop / temporal.py)
        return E.as_expr(o)

    def _bin(self, op, o, rev=False):
        a, b = self.expr, self._other(o)
        if rev:
            a, b = b, a
        return self._wrap(E.binop(op, a, b))

    def __add__(self, o): return self._bin("add", o)
    def __radd__(self, o): return self._bin("add", o, True)
    def __sub__(self, o): return self._bin("sub", o)
    def __rsub__(self, o): return self._bin("sub", o, True)
    def __mul__(self, o): return self._bin("mul", o)
    def __rmul__(self, o): return self._bin("mul", o, True)
    def __truediv__(self, o): return self._bin("truediv", o)
    def __rtruediv__(self, o): return self._bin("truediv", o, True)
    def __mod__(self, o): return self._bin("mod", o)
    def __rmod__(self, o): return self._bin("mod", o, True)
    def __gt__(self, o): return self._bin("gt", o)
    def __ge__(self, o): return self._bin("ge", o)
    def __lt__(self, o): return self._bin("lt", o)
    def __le__(self, o): return self._bin("le", o)
    def __eq__(self, o): return self._bin("eq", o)  # noqa: E711
    def __ne__(self, o): return self._bin("ne", o)
    def __and__(self, o): return self._bin("and", o)
    def __rand__(self, o): return self._bin("and", o, True)
    def __or__(self, o): return self._bin("or", o)
    def __ror__(self, o): return self._bin("or", o, True)
    def __invert__(self): return self._wrap(E.unop("not", self.expr))
    def __neg__(self): return self._wrap(E.unop("neg", self.expr))
    __hash__ = None

    def abs(self): return self._wrap(E.unop("abs", self.expr))
    def sqrt(self): return self._wrap(E.unop("sqrt", self.expr))
    def isna(self): return self._wrap(E.unop("isnull", self.expr))
    isnull = isna
    def notna(self): return ~self.isna()
    def fillna(self, v): return self._wrap(E.fillna(self.expr, self._other(v)))

    def sql_div(self, o, rev=False):
        """SQL division: truncating for integers (SQLDivisionOperator, call.py:165-189)."""
        return self._bin("divt", o, rev)

    def between(self, low, high, inclusive="both"):
        assert inclusive == "both"
        return (self >= low) & (self <= high)

    def isin(self, values):
        vals = list(values)
        if E.is_varchar(self.expr):      # absent literals match no row: only the codes of present ones remain
            from . import strings as S
            d = S.dictionary_of(self.expr)
            vals = [v for v in vals if not isinstance(v, str) or d.code_of(v) is not None]
        if not vals:
            return self._wrap(Lit(False))
        out = None
        for v in vals:
            t = self == v
            out = t if out is None else (out | t)
        # pandas isin never yields NULL
        return out.fillna(False)

    def like(self, pattern: str, escape="\\", ilike=False):
        """SQL [I]LIKE against a VARCHAR column (strings.like)"""
        from . import strings as S
        if not E.is_varchar(self.expr):
            raise NotImplementedError(f"LIKE on a {self.expr.logical} operand: only VARCHAR columns match patterns")
        return self._wrap(S.like(self.expr, pattern, escape, ilike))

    def where(self, cond, other=None):
        return self._wrap(E.case(self._other(cond), self.expr, self._other(other)))

    def astype(self, dtype):
        unit = T.unit_of(dtype)
        s = str(dtype).lower()
        if unit is not None:      # CAST AS DATE (datetime64[D]) / TIMESTAMP
            return self._wrap(T.cast_to(self.expr, "D" if unit == "D" else T.DEFAULT_UNIT))
        if s in ("boolean", "bool"):
            return self._wrap(E.cast(self.expr, U8))
        if s.startswith(("int", "uint")):
            return self._wrap(E.cast(self.expr, I64))
        if s.startswith("float"):
            return self._wrap(E.cast(self.expr, F64))
        raise NotImplementedError(f"astype({dtype}) is outside the int64/float64/bool hot path")

    def trunc(self):
        if self.expr.dtype != F64:
            return self
        return self._wrap(E.cast(E.cast(self.expr, I64), F64))

    def to_frame(self, name=None):
        name = name or self.name or "0"
        return LazyFrame(self.source, OrderedDict([(name, self.expr)]), list(self.pred))

    def compute(self):
        return self.to_frame().compute()[self.name or "0"]


# ---------------------------------------------------------------------------------------------
# frame
# ---------------------------------------------------------------------------------------------
class LazyFrame:
    def __init__(self, source: Source, exprs: "OrderedDict[str, Expr]" = None, pred: Sequence[Expr] = ()):
        self.source = source
        if exprs is None:
            exprs = OrderedDict((n, source.colref(n)) for n in source.schema)
        self.exprs: "OrderedDict[str, Expr]" = exprs
        self.pred: List[Expr] = list(pred)

    # -- metadata -------------------------------------------------------------------------
    @property
    def columns(self):
        return list(self.exprs.keys())

    @columns.setter
    def columns(self, names):
        names = [str(n) for n in names]
        assert len(names) == len(self.exprs)
        self.exprs = OrderedDict(zip(names, self.exprs.values()))

    def col_type(self, name):
        e = self.exprs[name]
        return e.dtype, e.logical

    def dtype_of(self, name):
        """numpy / pandas dtype of one column (cheap: no Series is built)."""
        return LazySeries(self.source, (), self.exprs[name]).dtype

    @property
    def dtypes(self):
        import pandas as pd
        return pd.Series({n: self.dtype_of(n) for n in self.exprs})

    @property
    def npartitions(self):
        from .executor import source_npartitions
        return source_npartitions(self.source)

    def _series(self, name):
        return LazySeries(self.source, tuple(self.pred), self.exprs[name], name)

    def copy(self):
        return LazyFrame(self.source, OrderedDict(self.exprs), list(self.pred))

    # -- indexing -------------------------------------------------------------------------
    def __getitem__(self, key):
        if isinstance(key, LazySeries):
            if key.source is not self.source:
                raise ValueError("filter condition belongs to a different frame")
            return LazyFrame(self.source, OrderedDict(self.exprs), self.pred + E.conjuncts(key.expr))
        if isinstance(key, (list, tuple)):
            return LazyFrame(self.source, OrderedDict((str(k), self.exprs[str(k)]) for k in key), self.pred)
        return self._series(str(key))

    @property
    def iloc(self):
        frame = self

        class _ILoc:
            def __getitem__(self, idx):
                rows, col = idx
                assert rows == slice(None)
                return frame._series(frame.columns[col])

        return _ILoc()

    def assign(self, **cols):
        exprs = OrderedDict(self.exprs)
        for n, v in cols.items():
            if isinstance(v, LazySeries):
                if v.source is not self.source:
                    raise ValueError("assigned column belongs to a different frame")
                exprs[n] = v.expr
            else:
                if isinstance(v, np.generic):
                    v = v.item()
                exprs[n] = E.as_expr(v)
        return LazyFrame(self.source, exprs, self.pred)

    def rename(self, columns):
        return LazyFrame(self.source, OrderedDict((columns.get(n, n), e) for n, e in self.exprs.items()), self.pred)

    def drop(self, columns, errors="raise"):
        columns = [columns] if isinstance(columns, str) else list(columns)
        return LazyFrame(self.source, OrderedDict((n, e) for n, e in self.exprs.items() if n not in columns),
                         self.pred)

    def head(self, n=5, compute=True, npartitions=-1):
        if n != 0:
            out = self.limit(n)
            return out.compute() if compute else out
        out = LazyFrame(self.source, OrderedDict(self.exprs), self.pred + [Lit(False)])
        return out.compute() if compute else out

    # -- relational ops -------------------------------------------------------------------
    def merge(self, right: "LazyFrame", on=None, left_on=None, right_on=None, how="inner", broadcast=None,
              indicator=False):
        if on is not None:
            left_on = right_on = [on] if isinstance(on, str) else list(on)
        left_on = [left_on] if isinstance(left_on, str) else list(left_on)
        right_on = [right_on] if isinstance(right_on, str) else list(right_on)
        if indicator:
            raise NotImplementedError("merge(indicator=True); use how='leftanti'")
        return LazyFrame(JoinSource(self, right, left_on, right_on, how, broadcast))

    def groupby(self, by, dropna=False):
        by = [by] if isinstance(by, str) else list(by)
        if dropna:
            raise NotImplementedError("groupby(dropna=True): SQL keeps the NULL group (aggregate.py:575-577)")
        return LazyGroupBy(self, by)

    def drop_duplicates(self, subset=None, **options):
        cols = list(subset) if subset is not None else self.columns
        return LazyFrame(AggSource(self[cols] if subset is None else self, cols, [], options))[cols]

    def reset_index(self, drop=False):
        return self

    def sort_values(self, by, ascending=True, na_position="last", nulls_first=None):
        by = [by] if isinstance(by, str) else list(by)
        asc = [ascending] * len(by) if isinstance(ascending, bool) else list(ascending)
        if nulls_first is None:
            nulls_first = [na_position == "first"] * len(by)
        elif isinstance(nulls_first, bool):
            nulls_first = [nulls_first] * len(by)
        return LazyFrame(SortSource(self, list(zip(by, asc, nulls_first))))

    def limit(self, fetch=None, offset=0):
        return LazyFrame(LimitSource(self, offset, fetch))

    # -- execution ------------------------------------------------------------------------
    def compute(self, **kwargs):
        from .executor import compute_frame
        return compute_frame(self)

    def persist(self):
        from .executor import persist_frame
        return persist_frame(self)

    def __len__(self):
        from .executor import count_rows
        return count_rows(self)

    def __repr__(self):
        return f"LazyFrame(columns={self.columns}, npred={len(self.pred)}, source={type(self.source).__name__})"


class LazyGroupBy:
    def __init__(self, frame: LazyFrame, by: List[str]):
        self.frame, self.by = frame, by

    def agg(self, spec: Dict[str, Dict[str, str]], **options):
        """spec: {input column: {output column: function}} (the shape DaskAggregatePlugin passes,
        aggregate.py:543-581).  Returns group columns followed by the outputs."""
        aggs = []
        for in_col, outs in spec.items():
            for out, fn in outs.items():
                aggs.append((in_col, out, fn))
        return LazyFrame(AggSource(self.frame, self.by, aggs, options))


def is_lazy(x):
    return isinstance(x, (LazyFrame, LazySeries))
