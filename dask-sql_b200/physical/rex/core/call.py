"""RexCall: SQL operator calls of the int64/float64/bool hot path (the reference's operator table is
dask_sql/physical/rex/core/call.py:1047-1156; SURVEY 2 row 6 lists the rows in scope): comparisons,
boolean logic, arithmetic, IS [NOT] NULL / TRUE / FALSE / UNKNOWN, BETWEEN, IN (list), CAST, CASE,
unary minus, ABS and the numeric functions (ROUND, CEIL / FLOOR, POWER, MOD, LN, SIN, ...).

A value is either a LazySeries -- a device expression that has not run yet -- or a Python scalar
(None is SQL NULL).  An operator here is a plain function  (operands, rex) -> value  that only
BUILDS expression nodes (dask-sql_b200/expr.py); the arithmetic happens later, fused into whichever
kernel consumes the expression.  Scalars are folded on the host with SQL's three-valued logic.
"""
import logging
import operator

import numpy as np

from .... import temporal as T
from ....mappings import SqlTypeName, cast_column_to_type, sql_to_python_type, sql_to_python_value
from ....utils import LoggableDataFrame, is_frame
from ..base import BaseRexPlugin
from ..convert import RexConverter

logger = logging.getLogger(__name__)


# ---------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------
def _left_fold(step, alone=None):
    """n-ary operator: ((a op b) op c) ...  (the planner hands `a + b + c` over as one call).
    `alone` is what a single operand means (unary plus / minus)."""
    def run(args, rex):
        if len(args) == 1 and alone is not None:
            return alone(args[0])
        acc = args[0]
        for nxt in args[1:]:
            acc = step(acc, nxt, rex)
        return acc
    return run


def _strict(fn):
    """Binary operator that is NULL as soon as a scalar operand is NULL.  (A NULL scalar next to a
    column becomes a NULL literal in the expression tree and the kernel propagates it.)"""
    def step(a, b, rex):
        if (a is None and not is_frame(b)) or (b is None and not is_frame(a)):
            return None
        return fn(a, b)
    return step


def _kleene_and(a, b, rex):
    if is_frame(a) or is_frame(b):
        return operator.and_(a, b)
    if a is False or b is False:
        return False
    return None if (a is None or b is None) else bool(a and b)


def _kleene_or(a, b, rex):
    if is_frame(a) or is_frame(b):
        return operator.or_(a, b)
    if a is True or b is True:
        return True
    return None if (a is None or b is None) else bool(a or b)


def _result_is_float(rex) -> bool:
    target = sql_to_python_type(SqlTypeName.fromString(str(rex.getType()).upper()))
    return bool(np.issubdtype(target, np.floating))


def _divide(a, b, rex):
    """SQL '/': true division when the plan types the result as floating point, otherwise the
    quotient truncated toward zero (not floored); an integer division by zero is NULL."""
    if _result_is_float(rex):
        if not is_frame(a) and not is_frame(b):
            return None if (a is None or b is None) else a / b
        return a / b
    if is_frame(a):
        return a.sql_div(b)
    if is_frame(b):
        return b.sql_div(a, rev=True)
    if a is None or b is None or b == 0:
        return None
    return int(np.trunc(a / b))


def _modulo(a, b):
    """SQL '%': floored like the reference's da.mod (NumPy) and the B2_OP_MOD_I kernel, -7 % 3 = 2;
    a zero divisor is NULL, for scalars as in _divide and in the kernel."""
    if is_frame(a) or is_frame(b):
        return a % b
    return None if b == 0 else a % b


def _unary(on_series, on_scalar):
    def run(args, rex):
        (x,) = args
        return on_series(x) if is_frame(x) else on_scalar(x)
    return run


def _is_null_scalar(x):
    return x is None or (isinstance(x, float) and x != x)


def _truth(expect: bool, negate: bool):
    """IS [NOT] TRUE / IS [NOT] FALSE: never NULL, an unknown operand counts as 'not that'."""
    def run(args, rex):
        (x,) = args
        if is_frame(x):
            as_bool = x.astype("boolean")
            hit = as_bool.fillna(False) if expect else ~as_bool.fillna(True)
            return ~hit if negate else hit
        hit = x is not None and bool(x) == expect
        return (not hit) if negate else hit
    return run


def _null_test(negate: bool):
    def run(args, rex):
        (x,) = args
        if is_frame(x):
            return x.notna() if negate else x.isna()
        return _is_null_scalar(x) != negate
    return run


def _case(args, rex):
    """CASE: operands are  when_1, then_1, when_2, then_2, ... [, else];  the first true WHEN wins.
    Built back to front so that each WHEN wraps what follows it."""
    from .... import expr as E
    from ....frame import LazySeries

    args = list(args)
    result = args.pop() if len(args) % 2 else None
    while args:
        then, when = args.pop(), args.pop()
        if not is_frame(when):
            if when:                         # a literal TRUE condition hides everything after it
                result = then
            continue
        if is_frame(then):
            result = then.where(when, other=result)
        else:
            other = result.expr if is_frame(result) else E.as_expr(result)
            result = LazySeries(when.source, when.pred, E.case(when.expr, E.as_expr(then), other))
    return result


def _cast(args, rex):
    (x,) = args
    sql_type = SqlTypeName.fromString(rex.getType())
    if not is_frame(x):
        return sql_to_python_value(sql_type, x)
    converted = cast_column_to_type(x, sql_to_python_type(sql_type))
    return x if converted is None else converted      # None: already of that type family


def _between(args, rex):
    x, low, high = args
    if any(is_frame(v) for v in (x, low, high)):
        inside = x.between(low, high, inclusive="both") if is_frame(x) else ((low <= x) & (high >= x))
        return ~inside if rex.isNegated() else inside
    if x is None or low is None or high is None:
        return None
    return (low <= x <= high) != bool(rex.isNegated())


def _in_list(args, rex):
    x, candidates = args[0], args[1:]
    if is_frame(x):
        found = x.isin(candidates)
        return ~found if rex.isNegated() else found
    return (x in candidates) != bool(rex.isNegated())


def _temporal(build, nstatic):
    """DATE / TIMESTAMP function: the first `nstatic` operands are words (field, unit), the rest values.
    Builds the device expression (temporal.py); on scalars the same tree is folded on the host."""
    from .... import expr as E
    from ....frame import LazySeries

    def run(args, rex):
        words, vals = list(args[:nstatic]), list(args[nstatic:])
        if any(v is None for v in vals):
            return None
        src = next((v for v in vals if is_frame(v)), None)
        exprs = [v.expr if is_frame(v) else (v if isinstance(v, str) else E.as_expr(v)) for v in vals]
        e = build(*words, *exprs)
        if src is None:
            return T.fold(e)
        return LazySeries(src.source, src.pred, e)
    return run


def _math(name):
    """Numeric function (expr.MATH_UNARY / MATH_BINARY); ROUND's optional second operand is its digits.
    Literal operands fold on the host through the same NumPy call; a column builds the device expression."""
    from .... import expr as E
    from ....frame import LazySeries

    def run(args, rex):
        vals = list(args)
        digits = vals.pop() if name == "round" and len(vals) == 2 else 0
        if any(v is None for v in vals) or digits is None:
            return None
        frames = [v for v in vals if is_frame(v)]
        if not frames:
            return E.math_fold(name, vals, digits)
        if any(f.source is not frames[0].source for f in frames):
            raise ValueError("cannot combine columns of different frames without a join")
        e = E.math(name, [v.expr if is_frame(v) else v for v in vals], digits)
        return LazySeries(frames[0].source, frames[0].pred, e)
    return run


def _rand(name, operands, dc):
    """RAND (operands: key, call site) and RAND_INTEGER (key, call site, h), bound by the planner from the
    reference's RAND / RANDOM / RAND_INTEGER (call.py:809-881).  A value is drawn per base-table row, so the
    frame must read one table: the rows of a join, an aggregate, a sort or a LIMIT have no number."""
    from .... import expr as E
    from ....executor import RAND_RULE
    from ....frame import LazySeries, TableSource
    df = getattr(dc, "df", dc)
    if not isinstance(getattr(df, "source", None), TableSource):
        raise NotImplementedError(RAND_RULE)
    df.source.numbered = True
    key, site = operands[0], operands[1]
    e = E.rand(key, site) if name == "rand" else E.rand_integer(key, site, operands[2])
    return LazySeries(df.source, tuple(df.pred), e)


def _like(ilike: bool):
    """[NOT] LIKE / ILIKE with a literal pattern; the ESCAPE character defaults to a backslash, as in the
    reference (call.py:414-416)."""
    from .... import strings as S

    def run(args, rex):
        x, pattern = args
        escape = getattr(rex, "value", None)
        escape = "\\" if escape is None else escape
        if x is None or pattern is None:
            return None
        if is_frame(x):
            hit = x.like(pattern, escape, ilike)
            return ~hit if rex.isNegated() else hit
        if not isinstance(x, str):
            raise NotImplementedError(f"LIKE on a {type(x).__name__} literal")
        return S.like_host(x, pattern, escape, ilike) != bool(rex.isNegated())
    return run


_COMPARISONS = {"=": operator.eq, "!=": operator.ne, "<>": operator.ne, ">": operator.gt, ">=": operator.ge,
                "<": operator.lt, "<=": operator.le}

OPERATORS = {name: _left_fold(_strict(fn)) for name, fn in _COMPARISONS.items()}
OPERATORS.update({
    "and": _left_fold(_kleene_and),
    "or": _left_fold(_kleene_or),
    "+": _left_fold(_strict(operator.add), alone=lambda x: x),
    "-": _left_fold(_strict(operator.sub), alone=lambda x: None if x is None else -x),
    "*": _left_fold(_strict(operator.mul)),
    "%": _left_fold(_strict(_modulo)),
    "/": _left_fold(_divide),
    "negative": _unary(operator.neg, lambda x: None if x is None else -x),
    "abs": _unary(lambda s: s.abs(), lambda x: None if x is None else abs(x)),
    "not": _unary(lambda s: ~s.astype("boolean"), lambda x: None if x is None else not x),
    "is null": _null_test(False),
    "is not null": _null_test(True),
    "is unknown": _null_test(False),
    "is not unknown": _null_test(True),
    "is true": _truth(True, False),
    "is not true": _truth(True, True),
    "is false": _truth(False, False),
    "is not false": _truth(False, True),
    "case": _case,
    "cast": _cast,
    "between": _between,
    "in list": _in_list,
    "like": _like(False),
    "ilike": _like(True),
    # DATE / TIMESTAMP (the reference's names, call.py:1137-1155)
    "date_part": _temporal(T.extract, 1),
    "datepart": _temporal(T.extract, 1),
    "extract_date": _temporal(lambda x: T.extract("DATE", x), 0),
    "year": _temporal(lambda x: T.extract("YEAR", x), 0),
    "timestampadd": _temporal(T.timestampadd, 1),
    "timestampdiff": _temporal(T.timestampdiff, 1),
    "timestampfloor": _temporal(lambda x, unit: T.floor_ceil(x, unit, False), 0),
    "timestampceil": _temporal(lambda x, unit: T.floor_ceil(x, unit, True), 0),
    "last_day": _temporal(lambda x: T.add_months_expr(x, 0, to_last=True), 0),
})

# numeric functions (call.py:1091-1113, and SQRT)
OPERATORS.update({name: _math(name) for name in ("ceil", "floor", "truncate", "round", "sign", "degrees", "radians",
                                                  "sqrt", "exp", "ln", "log10", "cbrt", "sin", "cos", "tan", "cot",
                                                  "asin", "acos", "atan", "atan2", "power", "mod")})


def _as_positional(fn):
    """The same operator callable the way the reference's table exposes it: f(*operands, rex=...)."""
    def call(*operands, rex=None, **_ignored):
        return fn(list(operands), rex)
    return call


class RexCallPlugin(BaseRexPlugin):
    """RexType.Call -> the function registered for the operator name; functions registered on the
    schema (context.schema[...].functions) are the fallback, as in call.py:1158-1216."""

    class_name = "RexCall"

    # name -> callable(*operands, rex=None): kept for code that looks operators up by name the way
    # it would in the reference (tests/unit/test_call.py:109-153 use the table like this)
    OPERATION_MAPPING = {name: _as_positional(fn) for name, fn in OPERATORS.items()}

    def convert(self, rel, expr, dc, context):
        operands = [RexConverter.convert(rel, o, dc, context=context) for o in expr.getOperands()]
        name = str(expr.getOperatorName()).lower()
        logger.debug("%s on %s", name, [str(LoggableDataFrame(o)) for o in operands])
        if name in ("rand", "rand_integer"):
            return _rand(name, operands, dc)
        if name in ("in subquery", "exists"):       # call.py:996-1030; the mark column attach_marks added
            from .subquery import mark_of
            return mark_of(expr, dc)
        fn = OPERATORS.get(name)
        if fn is not None:
            return fn(operands, expr)
        registered = context.schema[context.schema_name].functions
        if name in registered:
            return registered[name](*operands)
        raise NotImplementedError(f"RexCall operator '{name}' not (yet) implemented")
