"""Host-side expression IR of the execution layer.

The reference turns every REX node into one pandas call on whole Series
(physical/rex/core/call.py:1158-1216).  Here the same operators build a small typed tree; at
execution time a tree is either recognised as a conjunction of `column <cmp> literal` terms
(evaluated inside the fused scan kernels) or compiled to the postfix program of b2_expr_eval.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib as L
from . import temporal as T

I64, F64, U8 = L.I64, L.F64, L.U8
_DT_NAME = {I64: "int64", F64: "float64", U8: "bool"}

_CMP = {"eq": L.EQ, "ne": L.NE, "lt": L.LT, "le": L.LE, "gt": L.GT, "ge": L.GE}
_FLIP = {"eq": "eq", "ne": "ne", "lt": "gt", "le": "ge", "gt": "lt", "ge": "le"}

# An int64 column compared with a float literal compares in float64 (NumPy, and SQL's implicit cast to
# DOUBLE).  An integer-valued literal may become an exact int64 comparison only while |lit| < 2^53: there
# float(x) <op> lit  <=>  x <op> int(lit)  for every int64 x.  From 2^53 on float(x) rounds
# (float(2^53 + 1) == 2^53), so such a term keeps comparing in float64 (b2_term_t.as_f64).
F64_EXACT_INT = 2 ** 53


def int_literal_is_exact(lit: float) -> bool:
    return lit.is_integer() and abs(lit) < F64_EXACT_INT


class Expr:
    dtype: int = I64
    logical: str = "int64"

    def refs(self, out=None):
        out = set() if out is None else out
        self._refs(out)
        return out

    def _refs(self, out):
        pass


class ColRef(Expr):
    __slots__ = ("name", "dtype", "logical")

    def __init__(self, name, dtype, logical=None):
        self.name, self.dtype, self.logical = name, dtype, logical or _DT_NAME[dtype]

    def _refs(self, out):
        out.add(self.name)

    def __repr__(self):
        return f"col({self.name})"


class Lit(Expr):
    __slots__ = ("value", "dtype", "logical")

    def __init__(self, value, dtype=None, logical=None):
        if isinstance(value, T.TScalar):
            value, dtype, logical = value.ticks, I64, value.logical
        if dtype is None:
            if value is None:
                dtype = F64
            elif isinstance(value, (bool, np.bool_)):
                dtype, value = U8, bool(value)
            elif isinstance(value, (int, np.integer)):
                dtype, value = I64, int(value)
            elif isinstance(value, (float, np.floating)):
                dtype, value = F64, float(value)
            else:
                raise NotImplementedError(f"literal {value!r} of type {type(value).__name__} is outside the "
                                          "int64/float64/bool hot path")
        self.value, self.dtype, self.logical = value, dtype, logical or _DT_NAME[dtype]

    def __repr__(self):
        if T.is_temporal(self.logical):
            return f"lit({self.value!r}:{self.logical})"
        return f"lit({self.value!r})"


class Call(Expr):
    """`param`: the static operand of an operator (the field of datepart, the to-last-day flag of
    addmonths); `logical`: the result's logical dtype (a DATE / TIMESTAMP stays one through CASE, MIN ...)."""
    __slots__ = ("op", "args", "dtype", "logical", "param")

    def __init__(self, op, args, dtype, logical=None, param=None):
        self.op, self.args, self.dtype = op, tuple(args), dtype
        self.logical, self.param = logical or _DT_NAME[dtype], param

    def _refs(self, out):
        for a in self.args:
            a._refs(out)

    def __repr__(self):
        p = "" if self.param is None else f"[{self.param}]"
        return f"{self.op}{p}({', '.join(map(repr, self.args))})"


def as_expr(x) -> Expr:
    return x if isinstance(x, Expr) else Lit(x)


def cast(e: Expr, dtype: int) -> Expr:
    _no_varchar("CAST", e)
    if e.dtype == dtype:
        if dtype == I64 and T.is_temporal(e.logical):     # a DATE / TIMESTAMP as BIGINT: its ticks
            return Lit(e.value, I64) if isinstance(e, Lit) else Call("cast", [e], I64)
        return e
    if isinstance(e, Lit):
        if e.value is None:
            return Lit(None, dtype)
        if dtype == F64:
            return Lit(float(e.value), F64)
        if dtype == I64:
            return Lit(int(e.value), I64)
        return Lit(bool(e.value), U8)
    return Call("cast", [e], dtype)


def _arith_type(a: Expr, b: Expr):
    return F64 if F64 in (a.dtype, b.dtype) else I64


def is_temporal(x) -> bool:
    """A DATE / TIMESTAMP expression or host value, or an INTERVAL."""
    return isinstance(x, (T.TScalar, T.Interval)) or (isinstance(x, Expr) and T.is_temporal(x.logical))


def is_varchar(x) -> bool:
    """A VARCHAR (dictionary-coded) expression."""
    from . import strings as S
    return isinstance(x, Expr) and S.is_varchar(x)


def _no_varchar(what, *xs):
    if any(is_varchar(x) for x in xs):
        raise NotImplementedError(f"{what} of a VARCHAR: a string value can only be compared, matched with "
                                  "[NOT] LIKE / ILIKE, grouped, sorted, joined on, counted and MIN / MAX-ed here")


def binop(op: str, a, b) -> Expr:
    if is_varchar(a) or is_varchar(b):
        from . import strings as S
        return S.binop(op, a, b)
    if is_temporal(a) or is_temporal(b):
        return T.binop(op, a, b)
    if op in _CMP:
        r = T.rewrite_cmp(op, a, b)          # YEAR(x) <cmp> literal: a range on x
        if r is not None:
            return r
    a, b = as_expr(a), as_expr(b)
    if op in ("add", "sub", "mul", "mod"):
        t = _arith_type(a, b)
        return Call(op, [cast(a, t), cast(b, t)], t)
    if op == "truediv":
        return Call("truediv", [cast(a, F64), cast(b, F64)], F64)
    if op == "divt":  # SQL integer division: truncates toward zero (call.py:165-189)
        t = _arith_type(a, b)
        if t == F64:
            return Call("truediv", [cast(a, F64), cast(b, F64)], F64)
        return Call("divt", [cast(a, I64), cast(b, I64)], I64)
    if op in _CMP:
        t = _arith_type(a, b)
        return Call(op, [cast(a, t), cast(b, t)], U8)
    if op in ("and", "or"):
        return Call(op, [cast(a, U8), cast(b, U8)], U8)
    raise NotImplementedError(f"operator {op}")


def unop(op: str, a) -> Expr:
    a = as_expr(a)
    if op != "isnull":
        _no_varchar(op, a)
    if op == "neg":
        return Call("neg", [cast(a, I64) if a.dtype == U8 else a], F64 if a.dtype == F64 else I64)
    if op == "abs":
        return Call("abs", [a], a.dtype)
    if op == "sqrt":
        return Call("sqrt", [cast(a, F64)], F64)
    if op == "not":
        return Call("not", [cast(a, U8)], U8)
    if op == "isnull":
        if isinstance(a, Lit):
            return Lit(a.value is None or (isinstance(a.value, float) and a.value != a.value))
        return Call("isnull", [a], U8)
    raise NotImplementedError(f"operator {op}")


# Numeric SQL functions under the reference's operator names (call.py:1091-1113), each with the NumPy call
# the reference makes.  The device restates those calls (b200sql.h B2_OP_MATH_F / MATH2_F / POW_I); a call
# on literals folds on the host through the NumPy call itself (math_fold).
MATH_UNARY = {"ceil": (L.FN_CEIL, np.ceil), "floor": (L.FN_FLOOR, np.floor), "truncate": (L.FN_TRUNC, np.trunc),
              "round": (L.FN_ROUND, np.round), "sign": (L.FN_SIGN, np.sign), "degrees": (L.FN_DEGREES, np.degrees),
              "radians": (L.FN_RADIANS, np.radians), "exp": (L.FN_EXP, np.exp), "ln": (L.FN_LN, np.log),
              "log10": (L.FN_LOG10, np.log10), "cbrt": (L.FN_CBRT, np.cbrt), "sin": (L.FN_SIN, np.sin),
              "cos": (L.FN_COS, np.cos), "tan": (L.FN_TAN, np.tan), "cot": (L.FN_COT, lambda x: 1 / np.tan(x)),
              "asin": (L.FN_ASIN, np.arcsin), "acos": (L.FN_ACOS, np.arccos), "atan": (L.FN_ATAN, np.arctan),
              "sqrt": (None, np.sqrt)}
MATH_BINARY = {"atan2": (L.FN_ATAN2, np.arctan2), "power": (L.FN_POW, np.power), "mod": (L.FN_MOD, np.mod)}


def pow10(d: int) -> float:
    """NumPy's power of ten for np.round(x, d) (numpy/_core/src/multiarray/calculation.c, power_of_ten):
    a table up to 1e8, then repeated multiplication by 10 from 1e9 -- not always 10.0 ** d (d = 23, 25, ...)."""
    if d < 9:
        return float(10 ** d)
    r = 1e9
    for _ in range(d - 9):
        r *= 10.0
        if r == np.inf:
            break
    return r


def math(name: str, args, digits: int = 0) -> Expr:
    """The function `name` of MATH_UNARY / MATH_BINARY over expressions; `digits`: ROUND's second operand.
    Every result is a DOUBLE except POWER of two integers (BIGINT, np.power's wrapping integer power)."""
    args = [as_expr(a) for a in args]
    _no_varchar(name.upper(), *args)
    if name == "sqrt":
        return unop("sqrt", args[0])
    if name in MATH_UNARY:
        fn = MATH_UNARY[name][0]
        param = (fn, 0.0, 0)
        if name == "round":       # np.round: rint(x * f) / f, or rint(x / f) * f for negative digits
            param = (fn, pow10(abs(digits)), int(digits < 0))
        return Call("math", [cast(args[0], F64)], F64, param=param)
    x, y = args
    ints = F64 not in (x.dtype, y.dtype)
    if name == "mod":             # the integer modulo is floored like np.mod; either way a DOUBLE
        return cast(binop("mod", x, y), F64) if ints else binop("mod", x, y)
    if name == "power" and ints:
        return Call("powi", [cast(x, I64), cast(y, I64)], I64)
    return Call("math2", [cast(x, F64), cast(y, F64)], F64, param=MATH_BINARY[name][0])


def math_fold(name: str, vals, digits: int = 0):
    """`name` on host scalars (None is NULL), with the device's results: the NumPy call, except that an
    integer POWER with a negative exponent (where NumPy raises) and an integer MOD by zero are NULL."""
    if any(v is None for v in vals):
        return None
    ints = all(isinstance(v, (int, np.integer)) for v in vals)
    with np.errstate(all="ignore"):
        if name in MATH_BINARY and ints and name != "atan2":
            x, y = (np.int64(v) for v in vals)
            if name == "mod":
                return None if y == 0 else float(np.mod(x, y))
            return None if y < 0 else int(np.power(x, y))
        xs = [np.float64(v) for v in vals]
        if name == "round":
            return float(np.round(xs[0], digits))
        fn = MATH_UNARY[name][1] if name in MATH_UNARY else MATH_BINARY[name][1]
        return float(fn(*xs))


def rand(key: int, site: int) -> Expr:
    """RAND: a uniform DOUBLE in [0, 1) per base-table row, keyed on (key, call site) (rand.py)."""
    return Call("rand", [], F64, param=(int(key), int(site)))


def rand_integer(key: int, site: int, h) -> Expr:
    """RAND_INTEGER: a BIGINT in [0, h) per base-table row, from the same draw as RAND at that call site."""
    return Call("rand_int", [cast(as_expr(h), I64)], I64, param=(int(key), int(site)))


def has_rand(e: Expr) -> bool:
    """Does `e` draw per-row random numbers (so it needs its rows' numbers in the base table)?"""
    return isinstance(e, Call) and (e.op in ("rand", "rand_int") or any(has_rand(a) for a in e.args))


def rand_nodes(e: Expr, out=None) -> list:
    """The distinct rand / rand_int calls of `e`, in first-use order."""
    out = [] if out is None else out
    if isinstance(e, Call):
        if e.op in ("rand", "rand_int"):
            if not any(repr(n) == repr(e) for n in out):
                out.append(e)
        else:
            for a in e.args:
                rand_nodes(a, out)
    return out


def replace_nodes(e: Expr, mapping: Dict[str, Expr]) -> Expr:
    """Rewrite the sub-expressions whose repr is a key of `mapping`."""
    r = mapping.get(repr(e))
    if r is not None:
        return r
    if isinstance(e, Call):
        return Call(e.op, [replace_nodes(a, mapping) for a in e.args], e.dtype, e.logical, e.param)
    return e


def case(cond, then, other) -> Expr:
    if isinstance(then, str) or isinstance(other, str):
        raise NotImplementedError("CASE with a string result: a VARCHAR value built from two sources is not "
                                  "supported")
    cond, then, other = as_expr(cond), as_expr(then), as_expr(other)
    _no_varchar("CASE", then, other)
    if is_temporal(then) or is_temporal(other):
        then, other = T.unify(then, other)
        return Call("case", [cast(cond, U8), then, other], I64, then.logical)
    if isinstance(then, Lit) and then.value is None:
        t = other.dtype
    elif isinstance(other, Lit) and other.value is None:
        t = then.dtype
    else:
        t = F64 if F64 in (then.dtype, other.dtype) else (I64 if I64 in (then.dtype, other.dtype) else U8)
    return Call("case", [cast(cond, U8), cast(then, t), cast(other, t)], t)


def fillna(a, fill) -> Expr:
    if isinstance(fill, str):
        raise NotImplementedError("COALESCE / fillna with a string: a VARCHAR value built from two sources is "
                                  "not supported")
    a, fill = as_expr(a), as_expr(fill)
    _no_varchar("COALESCE", a, fill)
    if is_temporal(a) or is_temporal(fill):
        a, fill = T.unify(a, fill)
        return Call("fillna", [a, fill], I64, a.logical)
    return Call("fillna", [a, cast(fill, a.dtype)], a.dtype)


def substitute(e: Expr, mapping: Dict[str, Expr]) -> Expr:
    """Rewrite column references through `mapping` (composition of projections)."""
    if isinstance(e, ColRef):
        return mapping[e.name]
    if isinstance(e, Call):
        return Call(e.op, [substitute(a, mapping) for a in e.args], e.dtype, e.logical, e.param)
    return e


def conjuncts(e: Expr) -> List[Expr]:
    """Flatten AND under 'is TRUE' semantics; fillna(x, False) is the identity there
    (filter.py:38-39: a NULL predicate drops the row)."""
    if isinstance(e, Call):
        if e.op == "and":
            return conjuncts(e.args[0]) + conjuncts(e.args[1])
        if e.op == "fillna" and isinstance(e.args[1], Lit) and e.args[1].value in (False, 0):
            return conjuncts(e.args[0])
    return [e]


def _strip_cast(e: Expr):
    """cast(ColRef int -> f64) compares as float: report (colref, as_f64)."""
    if isinstance(e, Call) and e.op == "cast" and e.dtype == F64 and isinstance(e.args[0], ColRef) \
            and e.args[0].dtype == I64:
        return e.args[0], True
    if isinstance(e, ColRef):
        return e, False
    return None, False


def as_term(e: Expr) -> Optional[Tuple[str, int, object]]:
    """Recognise `col <cmp> literal`, `col IS [NOT] NULL`, or a boolean column.
    Returns (column name, B2 term op, literal) or None."""
    if isinstance(e, ColRef) and e.dtype == U8:
        return e.name, L.IS_TRUE, 0
    if not isinstance(e, Call):
        return None
    if e.op in _CMP:
        a, b = e.args
        op = e.op
        if isinstance(a, Lit) and not isinstance(b, Lit):
            a, b, op = b, a, _FLIP[op]
        if isinstance(b, Lit) and b.value is not None:
            col, as_f = _strip_cast(a)
            if col is None or col.dtype == U8:
                return None
            lit = b.value
            if as_f or col.dtype == F64:
                lit = float(lit)
                if col.dtype == I64 and int_literal_is_exact(lit):
                    lit = int(lit)
            return col.name, _CMP[op], lit
        return None
    if e.op == "isnull" and isinstance(e.args[0], ColRef):
        return e.args[0].name, L.IS_NULL, 0
    if e.op == "not" and isinstance(e.args[0], Call) and e.args[0].op == "isnull" \
            and isinstance(e.args[0].args[0], ColRef):
        return e.args[0].args[0].name, L.IS_NOT_NULL, 0
    return None


# ---------------------------------------------------------------------------------------------
# compilation to the postfix program of b2_expr_eval
# ---------------------------------------------------------------------------------------------
def map_tables(e: Expr, out=None) -> list:
    """The per-entry tables (strings.MapTable) that `e`'s "map" nodes look up, in first-use order: the
    program reads them as columns len(col_names), len(col_names) + 1, ..."""
    out = [] if out is None else out
    if isinstance(e, Call):
        if e.op == "map" and not any(t is e.param for t in out):
            out.append(e.param)
        for a in e.args:
            map_tables(a, out)
    return out


class _Compiler:
    def __init__(self, col_index: Dict[str, int], tables=()):
        self.col_index = col_index
        self.tables = list(tables)
        self.code: List[Tuple[int, int, int, float]] = []

    def emit(self, op, a=0, imm_i=0, imm_f=0.0):
        self.code.append((op, a, imm_i, imm_f))

    def lit(self, e: Lit):
        if e.value is None:
            self.emit(L.OP_CONST_NULL)
        elif e.dtype == F64:
            self.emit(L.OP_CONST_F, imm_f=float(e.value))
        else:
            self.emit(L.OP_CONST_I, imm_i=int(e.value))

    def visit(self, e: Expr):
        if isinstance(e, ColRef):
            self.emit(L.OP_LOAD, a=self.col_index[e.name])
            return
        if isinstance(e, Lit):
            self.lit(e)
            return
        op, args = e.op, e.args
        if op == "cast":
            src = args[0]
            self.visit(src)
            if e.dtype == F64 and src.dtype != F64:
                self.emit(L.OP_I2F)
            elif e.dtype == I64 and src.dtype == F64:
                self.emit(L.OP_F2I)
            elif e.dtype == U8 and src.dtype == I64:
                self.emit(L.OP_CONST_I, imm_i=0)
                self.emit(L.OP_EQ_I + L.NE)
            elif e.dtype == U8 and src.dtype == F64:
                self.emit(L.OP_CONST_F, imm_f=0.0)
                self.emit(L.OP_EQ_F + L.NE)
            return
        if op in ("add", "sub", "mul", "mod", "truediv", "divt"):
            self.visit(args[0])
            self.visit(args[1])
            f = e.dtype == F64
            table = {"add": (L.OP_ADD_I, L.OP_ADD_F), "sub": (L.OP_SUB_I, L.OP_SUB_F),
                     "mul": (L.OP_MUL_I, L.OP_MUL_F), "truediv": (None, L.OP_DIV_F),
                     "divt": (L.OP_DIV_I, None), "mod": (L.OP_MOD_I, L.OP_MATH2_F)}
            code = table[op][1 if f else 0]
            if code is None:
                raise NotImplementedError(f"{op} on {_DT_NAME[e.dtype]}")
            self.emit(code, a=L.FN_MOD if code == L.OP_MATH2_F else 0)
            return
        if op == "math":
            fn, f, div_first = e.param
            self.visit(args[0])
            self.emit(L.OP_MATH_F, a=fn, imm_i=div_first, imm_f=f)
            return
        if op in ("math2", "powi"):
            self.visit(args[0])
            self.visit(args[1])
            if op == "math2":
                self.emit(L.OP_MATH2_F, a=e.param)
            else:
                self.emit(L.OP_POW_I)
            return
        if op in _CMP:
            self.visit(args[0])
            self.visit(args[1])
            base = L.OP_EQ_F if args[0].dtype == F64 else L.OP_EQ_I
            self.emit(base + _CMP[op])
            return
        if op in ("and", "or"):
            self.visit(args[0])
            self.visit(args[1])
            self.emit(L.OP_AND if op == "and" else L.OP_OR)
            return
        if op == "not":
            self.visit(args[0])
            self.emit(L.OP_NOT)
            return
        if op == "neg":
            self.visit(args[0])
            self.emit(L.OP_NEG_F if e.dtype == F64 else L.OP_NEG_I)
            return
        if op == "abs":
            self.visit(args[0])
            self.emit(L.OP_ABS_F if e.dtype == F64 else L.OP_ABS_I)
            return
        if op == "sqrt":
            self.visit(args[0])
            self.emit(L.OP_SQRT_F)
            return
        if op == "isnull":
            self.visit(args[0])
            self.emit(L.OP_ISNULL_F if args[0].dtype == F64 else L.OP_ISNULL_I)
            return
        if op == "case":
            for a in args:
                self.visit(a)
            self.emit(L.OP_CASE)
            return
        if op == "fillna":
            # NaN in a float operand is NULL for fillna: route through CASE(isnull(x), fill, x)
            if args[0].dtype == F64:
                self.visit(args[0])
                self.emit(L.OP_ISNULL_F)
                self.visit(args[1])
                self.visit(args[0])
                self.emit(L.OP_CASE)
            else:
                self.visit(args[0])
                self.visit(args[1])
                self.emit(L.OP_FILLNA)
            return
        if op == "ord2f":
            self.visit(args[0])
            self.emit(L.OP_ORD2F)
            return
        if op == "datepart":
            field, tps = e.param
            self.visit(args[0])
            self.emit(L.OP_DATEPART, a=field, imm_i=tps)
            return
        if op == "addmonths":
            to_last, tps = e.param
            self.visit(args[0])
            self.visit(args[1])
            self.emit(L.OP_ADDMONTHS, a=to_last, imm_i=tps)
            return
        if op in ("rand", "rand_int"):
            key, site = e.param
            if op == "rand_int":
                self.visit(args[0])
            self.emit(L.OP_RAND_F if op == "rand" else L.OP_RAND_I, a=site, imm_i=key)
            return
        if op == "map":
            k = next((i for i, t in enumerate(self.tables) if t is e.param), None)
            if k is None:
                raise NotImplementedError("a map over a dictionary table needs the table among the program's columns")
            self.visit(args[0])
            self.emit(L.OP_MAP, a=len(self.col_index) + k, imm_i=len(e.param))
            return
        raise NotImplementedError(f"expression operator {op}")


def compile_expr(e: Expr, col_names: Sequence[str], tables=()) -> L.Prog:
    """Compile `e` over the columns `col_names` (their order defines LOAD indices), followed by the
    per-entry `tables` of its "map" nodes (map_tables(e))."""
    comp = _Compiler({n: i for i, n in enumerate(col_names)}, tables)
    comp.visit(e)
    if len(comp.code) > L.MAX_PROG:
        raise NotImplementedError(f"expression needs {len(comp.code)} instructions (max {L.MAX_PROG})")
    p = L.Prog()
    p.n = len(comp.code)
    p.out_dtype = e.dtype
    for i, (op, a, ii, ff) in enumerate(comp.code):
        ins = p.code[i]
        ins.op, ins.a, ins.imm_i, ins.imm_f = op, a, ii, ff
    return p


def may_be_null(e: Expr, col_nullable) -> bool:
    """Conservative: can the result carry a validity bitmap NULL?"""
    if isinstance(e, ColRef):
        return col_nullable(e.name)
    if isinstance(e, Lit):
        return e.value is None
    if e.op == "isnull":
        return False
    if e.op in ("divt", "mod", "map", "powi", "rand_int"):
        return True
    if e.op == "cast" and e.dtype == I64 and e.args[0].dtype == F64:
        return True
    return any(may_be_null(a, col_nullable) for a in e.args)
