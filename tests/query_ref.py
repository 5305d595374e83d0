"""Exact reference of whole SQL queries, as `Context.sql()` answers them, and an exact comparator for results.

A relation is an ordered dict name -> `rowwise_ref.Column`; a VARCHAR column is a Column of dtype STR whose
values are an object array of str (None = NULL).  The operators are the kernel references' rules, composed:
  * filters: `rowwise_ref.eval_term` (NULL fails every comparison, an int column against a float literal
    compares in float64, NaN is unordered);
  * joins: `join_ref.hash_matches` / `join_ref.emit` (NULL and NaN keys never match, -0.0 matches +0.0);
    an int key joined to a float key compares in float64, VARCHAR keys by string value; RIGHT is LEFT with
    the sides swapped, FULL is LEFT plus the build rows nothing matched, SEMI / ANTI keep the left columns;
  * GROUP BY: groups are `groupagg_ref.hashk_identity` (NULL and NaN form one NULL group, -0.0 joins +0.0;
    a float key comes out as +0.0, a NULL float key as NaN); aggregates are `groupagg_bits_ref.aggregate`;
  * ORDER BY: `rowwise_ref.sort_perm`, last key first (stable; NaN is NULL, -0.0 ties with 0.0; ASC puts
    NULLs last and DESC first unless NULLS FIRST / LAST says otherwise), then OFFSET / LIMIT.
What differs from SQL on purpose is DESIGN.md section 6: a global aggregate over no rows is 0 rows, EVERY and
BIT_* of a group with no input are NULL, REGR_* take the rows where both arguments are non-NULL.

A result is a `Result`: columns of cells, each column of one kind:
  "int"     Python int or None (int64, DATE / TIMESTAMP as their int64 words): compared word for word;
  "bool"    True / False / None;      "str"  str or None: by value;
  "float"   a float compared bit for bit (-0.0 is not +0.0); NaN and NULL are the same cell, as everywhere
            in the engine's float columns;
  "bounded" (exact, bound): the computed float must lie within `bound` of `exact` (specials exactly).
Float SUM / AVG are bounded by groupagg_ref's gamma bound unless their inputs are dyadic (every partial sum
exact), where they are "float".  VAR / STDDEV / REGR_SXX / REGR_SYY are bounded against the exact Fraction
value; see `moment_bound`.  No GPU and no package import."""
import math
from fractions import Fraction
from typing import Dict, List, Optional

import numpy as np

from tests import groupagg_bits_ref as GB
from tests import groupagg_ref as G
from tests import join_ref as J
from tests import rowwise_ref as R
from tests.rowwise_ref import F64, I64, U8, Column

STR = 3
U = 2.0 ** -53
CMP = {"=": R.EQ, "<>": R.NE, "<": R.LT, "<=": R.LE, ">": R.GT, ">=": R.GE}


# ---- relations -----------------------------------------------------------------------------------------------
def table(df) -> Dict[str, Column]:
    """pandas DataFrame -> relation: int64 / Int64 -> I64, float64 -> F64 (NaN kept as a value: it is NULL
    wherever the engine reads a float), bool / boolean -> U8, category / object of str -> STR"""
    import pandas as pd
    rel = {}
    for name in df.columns:
        s = df[name]
        null = s.isna().to_numpy()
        if isinstance(s.dtype, pd.CategoricalDtype) or pd.api.types.is_string_dtype(s.dtype):
            vals = np.array([None if pd.isna(x) else str(x) for x in s], dtype=object)
            rel[name] = Column(vals, vals == None, STR)  # noqa: E711
        elif pd.api.types.is_bool_dtype(s.dtype):
            rel[name] = Column(s.fillna(False).to_numpy(dtype=np.uint8), null if null.any() else None, U8)
        elif pd.api.types.is_integer_dtype(s.dtype):
            rel[name] = Column(s.fillna(0).to_numpy(dtype=np.int64), null if null.any() else None, I64)
        else:
            rel[name] = Column(s.to_numpy(dtype=np.float64, na_value=np.nan), None, F64)
    return rel


def take(col: Column, idx) -> Column:
    """rows idx of col; idx -1 gives NULL (0 / NaN / None in the value slot)"""
    idx = np.asarray(idx, np.int64)
    miss = idx < 0
    safe = np.where(miss, 0, idx)
    vals = col.values[safe] if len(col.values) else np.zeros(len(idx), col.values.dtype)
    null = (col.null_mask()[safe] if len(col.values) else np.zeros(len(idx), bool)) | miss
    if miss.any():
        vals = vals.copy()
        vals[miss] = None if col.dtype == STR else (np.nan if col.dtype == F64 else 0)
        if col.dtype == F64:
            null = null & ~miss              # a missing float is NaN, which is NULL already
    return Column(vals, null if null.any() else None, col.dtype)


def rows(rel, idx):
    return {n: take(c, idx) for n, c in rel.items()}


def nrows(rel) -> int:
    return len(next(iter(rel.values())).values)


def where(rel, mask):
    return rows(rel, np.flatnonzero(mask))


def cmp(col: Column, op: str, lit) -> np.ndarray:
    """`col op literal` as a WHERE conjunct: rows where it is TRUE"""
    if col.dtype == STR:
        v = col.values
        ok = np.array([x is not None and {"=": x == lit, "<>": x != lit, "<": x < lit, "<=": x <= lit,
                                            ">": x > lit, ">=": x >= lit}[op] for x in v], bool)
        return ok
    as_f = isinstance(lit, float) and col.dtype != F64
    return R.eval_term(col, CMP[op], as_f64=int(as_f), lit_i=0 if isinstance(lit, float) else int(lit),
                       lit_f=float(lit))


def is_null(col: Column) -> np.ndarray:
    return G.null_of(col) if col.dtype != STR else col.values == None  # noqa: E711


def _str_codes(*cols):
    """VARCHAR columns -> I64 columns of one shared code per distinct string, in code-point order"""
    words = sorted({x for c in cols for x in c.values if x is not None})
    code = {w: i for i, w in enumerate(words)}
    return [Column(np.array([code.get(x, 0) if x is not None else 0 for x in c.values], np.int64),
                   c.values == None, I64) for c in cols]  # noqa: E711


def _as_f64(col: Column) -> Column:
    v = col.values.astype(np.float64)
    return Column(np.where(col.null_mask(), np.nan, v), None, F64)


def _join_keys(lcols, rcols):
    outl, outr = [], []
    for a, b in zip(lcols, rcols):
        if a.dtype == STR or b.dtype == STR:
            a, b = _str_codes(a, b)
        if a.dtype == U8:
            a = Column(a.values.astype(np.int64), a.null, I64)
        if b.dtype == U8:
            b = Column(b.values.astype(np.int64), b.null, I64)
        if a.dtype != b.dtype:
            a, b = _as_f64(a), _as_f64(b)
        outl.append(a), outr.append(b)
    return outl, outr


def join(left, right, lkeys, rkeys, how="inner"):
    """equi-join; the column names of the two sides must differ.  how: inner / left / right / full / semi / anti"""
    if how == "right":
        out = join(right, left, rkeys, lkeys, "left")
        return {**{n: out[n] for n in left}, **{n: out[n] for n in right}}
    lk, rk = _join_keys([left[k] for k in lkeys], [right[k] for k in rkeys])
    nl, nr = nrows(left), nrows(right)
    m = J.hash_matches(lk, rk, np.ones(nl, bool))
    mode = {"inner": J.JOIN_INNER, "left": J.JOIN_LEFT, "full": J.JOIN_LEFT, "semi": J.JOIN_SEMI,
            "anti": J.JOIN_ANTI}[how]
    e = J.emit(mode, np.ones(nl, bool), m)
    if how in ("semi", "anti"):
        return rows(left, e.probe)
    lidx, ridx = e.probe, e.build
    if how == "full":
        unmatched = np.setdiff1d(np.arange(nr), m.rows)
        lidx = np.concatenate([lidx, np.full(len(unmatched), -1)])
        ridx = np.concatenate([ridx, unmatched])
    return {**rows(left, lidx), **rows(right, ridx)}


# ---- results ---------------------------------------------------------------------------------------------------
class Result:
    """columns of cells (see the module doc), plus the ORDER BY that produced them: `order` [(name, desc,
    nulls_first)] and the OFFSET / LIMIT window over the fully sorted rows `cols`"""

    def __init__(self, cols: Dict[str, list], kinds: Dict[str, str], order=None, offset=0, limit=None):
        self.cols, self.kinds, self.order, self.offset, self.limit = cols, kinds, order, offset, limit

    @property
    def names(self):
        return list(self.cols)

    @property
    def n(self):
        return len(next(iter(self.cols.values()))) if self.cols else 0

    def window(self):
        """the rows the query returns: (first, end) into cols"""
        lo = min(self.offset, self.n)
        return lo, self.n if self.limit is None else min(self.n, lo + self.limit)

    def as_got(self) -> Dict[str, list]:
        """the result a correct engine returns (bounded cells at their exact value), window applied"""
        lo, hi = self.window()
        return {k: [c[0] if self.kinds[k] == "bounded" else c for c in v[lo:hi]] for k, v in self.cols.items()}


def _cells(col: Column):
    null = col.null_mask()
    if col.dtype == STR:
        return "str", [None if x is None else str(x) for x in col.values]
    if col.dtype == F64:
        return "float", [math.nan if nl else float(x) for x, nl in zip(col.values, null)]
    if col.dtype == U8:
        return "bool", [None if nl else bool(x) for x, nl in zip(col.values, null)]
    return "int", [None if nl else int(x) for x, nl in zip(col.values, null)]


def select(rel, names=None) -> Result:
    names = list(rel) if names is None else names
    cols, kinds = {}, {}
    for n in names:
        kinds[n], cols[n] = _cells(rel[n])
    return Result(cols, kinds)


# ---- GROUP BY --------------------------------------------------------------------------------------------------
def _identity(cols: List[Column], n):
    """per row: a hashable group identity (hashk_identity per key: normalised bits + NULL bit; VARCHAR by value)"""
    per = []
    for c in cols:
        if c.dtype == STR:
            per.append([(x,) for x in c.values])
        else:
            per.append(G.hashk_identity([c]))
    return [tuple(p[i] for p in per) for i in range(n)]


def _key_cell(col: Column, ident):
    """output value of a group key from its identity (bits, null mask) / (str,)"""
    if col.dtype == STR:
        return ident[0]
    bits, null = ident
    if col.dtype == F64:
        return math.nan if null else float(np.int64(bits).view(np.float64))
    if null:
        return None
    return bool(bits) if col.dtype == U8 else int(bits)


def dyadic(x) -> bool:
    """every partial sum of x (in any order) is exact: small multiples of one power of two"""
    x = np.asarray(x, np.float64)
    if not len(x):
        return True
    if not np.isfinite(x).all():
        return False
    for p in (0, 8, 16, 24, 32, 40, 48):
        y = x * 2.0 ** p
        if (y == np.round(y)).all() and math.fsum(np.abs(y).tolist()) < 2.0 ** 53:
            return True
    return False


def moment_bound(ss: Fraction, n: int, span: float, denom: int) -> float:
    """bound on |computed - exact| of ss / denom, ss = sum of squared deviations of n values, when the engine
    forms it as S2 - S1^2 / n from the shifted moments S1 = sum fl(x - K), S2 = sum fl(x - K)^2 with K and
    every x in an interval of width `span` (K: the midpoint of the input's value range, DESIGN.md section 6):
    gamma-bounded sums of terms at most span^2 (twice: S2 and S1^2 / n <= S2), the rounding of each x - K
    (at most u * span, moving ss by at most 2 sqrt(ss n) u span + n u^2 span^2), and the final division"""
    s2 = float(span) ** 2
    err = 2 * (G.gamma(n + 2) + 2 * U) * n * s2 + 2 * math.sqrt(float(ss) * n) * U * span + n * U * U * s2
    return err / denom + 2 * U * float(ss) / denom


AGG_FUNCS = ("count", "count_star", "sum", "avg", "min", "max", "var_samp", "var_pop", "stddev_samp",
             "stddev_pop", "regr_sxx", "regr_syy", "regr_count", "bit_and", "bit_or", "bit_xor", "every",
             "count_distinct")


def aggregate(rel, keys: List[str], aggs, mask=None, span: Optional[Dict[str, float]] = None) -> Result:
    """SELECT keys..., aggs... FROM rel [WHERE mask] GROUP BY keys.  aggs: [(out name, func, arg[, arg2])],
    func one of AGG_FUNCS (regr_*: arg = y, arg2 = x).  span[arg]: width of an interval holding every value of
    the column (default: its range over all of rel, before `mask`)."""
    n = nrows(rel)
    passing = np.ones(n, bool) if mask is None else np.asarray(mask, bool)
    kcols = [rel[k] for k in keys]
    if keys:
        gid, groups = G.codes(_identity(kcols, n), passing)
    else:
        gid = np.where(passing, 0, -1).astype(np.int64)
        groups = [()] if passing.any() else []          # DESIGN.md section 6: no row in, no row out
    ng = len(groups)
    cols = {k: [_key_cell(c, g[i]) for g in groups] for i, (k, c) in enumerate(zip(keys, kcols))}
    kinds = {k: _cells(c)[0] for k, c in zip(keys, kcols)}
    span = dict(span or {})

    def col_span(name):
        if name not in span:
            c = rel[name]
            ok = ~G.null_of(c)
            v = c.values[ok].astype(np.float64)
            span[name] = float(v.max() - v.min()) if len(v) else 0.0
        return span[name]

    for spec in aggs:
        name, fn, arg = spec[0], spec[1], spec[2] if len(spec) > 2 else None
        arg2 = spec[3] if len(spec) > 3 else None
        assert fn in AGG_FUNCS, fn
        col = rel[arg] if arg is not None else None
        if fn == "count_star" or fn == "count":
            ex = G.aggregate([col], [G.AGG_COUNT], gid, ng)
            cols[name], kinds[name] = [int(v) for v in ex.cnt[0]], "int"
        elif fn == "count_distinct":
            ok = (gid >= 0) & ~is_null(col)
            img = J.key_image(col) if col.dtype != STR else col.values
            seen = [set() for _ in range(ng)]
            for g, v in zip(gid[ok], img[ok]):
                seen[g].add(v if col.dtype == STR else int(v))
            cols[name], kinds[name] = [len(s) for s in seen], "int"
        elif fn in ("sum", "avg"):
            op = G.AGG_SUMF if fn == "avg" and col.dtype != F64 else G.AGG_SUM
            ex = G.aggregate([col], [op], gid, ng)
            cnt = ex.cnt[0]
            if ex.exact[0] is None:              # int SUM: the wrapped word
                cols[name], kinds[name] = [int(w) if c else None for w, c in zip(ex.acc[0], cnt)], "int"
                continue
            ok = (gid >= 0) & ~G.null_of(col)
            exact_data = [dyadic(col.values[ok & (gid == g)]) for g in range(ng)]
            out = []
            for g in range(ng):
                if cnt[g] == 0:
                    out.append((math.nan, 0.0))
                    continue
                e, b = float(ex.exact[0][g]), float(ex.bound[0][g])
                if fn == "avg":
                    e, b = e / int(cnt[g]), b / int(cnt[g]) + U * abs(e / int(cnt[g]))
                out.append((e, 0.0 if exact_data[g] else b))
            if all(exact_data):
                cols[name], kinds[name] = [c[0] for c in out], "float"
            else:
                cols[name], kinds[name] = out, "bounded"
        elif fn in ("min", "max"):
            ex = G.aggregate([col], [G.AGG_MIN if fn == "min" else G.AGG_MAX], gid, ng)
            cnt = ex.cnt[0]
            if col.dtype == F64:
                f = R.bits2f(R.ordered(ex.acc[0]))
                cols[name], kinds[name] = [float(x) if c else math.nan for x, c in zip(f, cnt)], "float"
            else:
                cols[name], kinds[name] = [int(w) if c else None for w, c in zip(ex.acc[0], cnt)], "int"
        elif fn in ("bit_and", "bit_or", "bit_xor", "every"):
            op = {"bit_and": GB.AGG_AND, "bit_or": GB.AGG_OR, "bit_xor": GB.AGG_XOR, "every": GB.AGG_AND}[fn]
            ex = GB.aggregate([col], [op], gid, ng)
            cnt = ex.cnt[0]
            if fn == "every":
                cols[name], kinds[name] = [bool(w) if c else None for w, c in zip(ex.acc[0], cnt)], "bool"
            else:
                cols[name], kinds[name] = [int(w) if c else None for w, c in zip(ex.acc[0], cnt)], "int"
        else:
            # VAR / STDDEV over the non-NULL values of arg; REGR_*(y, x) over the rows where both are non-NULL
            if fn.startswith("regr"):
                both = ~G.null_of(rel[arg]) & ~G.null_of(rel[arg2])
                src = arg2 if fn == "regr_sxx" else arg
                use = both
            else:
                src, use = arg, ~G.null_of(col)
            ok = (gid >= 0) & use
            if fn == "regr_count":
                cols[name], kinds[name] = [int(v) for v in np.bincount(gid[ok], minlength=ng)], "int"
                continue
            vals = rel[src].values.astype(np.float64)
            ddof = 1 if fn.endswith("samp") else 0
            out = []
            for g in range(ng):
                xs = [Fraction(float(v)) for v in vals[ok & (gid == g)]]
                m = len(xs)
                if m <= ddof or m == 0:
                    out.append((math.nan, 0.0))
                    continue
                mean = sum(xs) / m
                ss = sum((x - mean) ** 2 for x in xs)
                denom = 1 if fn.startswith("regr") else m - ddof
                var = ss / denom
                b = moment_bound(ss, m, col_span(src), denom)
                if fn.startswith("stddev"):
                    sd = math.sqrt(float(var))
                    out.append((sd, (b / sd if sd > 0 else math.sqrt(b)) + 2 * U * sd))
                else:
                    out.append((float(var), b))
            cols[name], kinds[name] = out, "bounded"
    return Result(cols, kinds)


# ---- ORDER BY / LIMIT ------------------------------------------------------------------------------------------
def _sort_column(res: Result, name) -> Column:
    kind, cells = res.kinds[name], res.cols[name]
    if kind in ("float", "bounded"):
        v = np.array([c[0] if kind == "bounded" else c for c in cells], np.float64)
        return Column(v, None, F64)
    if kind == "str":
        return _str_codes(Column(np.array(cells, dtype=object), None, STR))[0]
    null = np.array([c is None for c in cells], bool)
    return Column(np.array([0 if c is None else int(c) for c in cells], np.int64), null, I64)


def order_by(res: Result, keys, offset=0, limit=None) -> Result:
    """keys: [(name, desc[, nulls_first])]; nulls_first defaults to desc (SQL: ASC NULLS LAST, DESC NULLS FIRST)"""
    order = [(k[0], bool(k[1]), bool(k[2]) if len(k) > 2 else bool(k[1])) for k in keys]
    idx = np.arange(res.n, dtype=np.int64)
    for name, desc, nf in reversed(order):
        idx = R.sort_perm(_sort_column(res, name), idx, desc, nf).astype(np.int64)
    cols = {k: [v[i] for i in idx] for k, v in res.cols.items()}
    return Result(cols, dict(res.kinds), order, offset, limit)


# ---- the comparator --------------------------------------------------------------------------------------------
def _fbits(x) -> int:
    return int(np.float64(x).view(np.int64))


def _hard(kind, v, what):
    """canonical, hashable form of a cell of an exactly compared column"""
    if kind == "int":
        if v is None:
            return ("null",)
        assert isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)), \
            f"{what}: {v!r} is not an integer"
        return ("i", int(v))
    if kind == "bool":
        if v is None:
            return ("null",)
        assert isinstance(v, (bool, np.bool_)), f"{what}: {v!r} is not a bool"
        return ("b", bool(v))
    if kind == "str":
        if v is None:
            return ("null",)
        assert isinstance(v, str), f"{what}: {v!r} is not a str"
        return ("s", v)
    if v is None or math.isnan(v):
        return ("null",)
    return ("f", _fbits(v))


def _soft_ok(g, cell) -> bool:
    e, b = cell
    g = math.nan if g is None else float(g)
    if math.isnan(e) or math.isnan(g):
        return math.isnan(e) and math.isnan(g)
    if math.isinf(e) or math.isinf(g) or b == 0.0:
        return _fbits(g) == _fbits(e)
    return abs(g - e) <= b


def _sort_soft(v):
    v = v[0] if isinstance(v, tuple) else v
    return (1, 0.0) if v is None or math.isnan(v) else (0, float(v))


def _match(got_rows, exp_rows, kinds, names, what):
    """got_rows / exp_rows: lists of row tuples.  Equal as multisets: exact cells identical, bounded cells within
    their bound (rows sorted on the exact cells, then on the bounded values, and compared in that order)."""
    assert len(got_rows) == len(exp_rows), f"{what}: {len(got_rows)} rows, expected {len(exp_rows)}"
    hard = [i for i, k in enumerate(kinds) if k != "bounded"]
    soft = [i for i, k in enumerate(kinds) if k == "bounded"]

    def key(r):
        return (tuple(_hard(kinds[i], r[i], f"{what} column {names[i]}") for i in hard),
                tuple(_sort_soft(r[i]) for i in soft))

    g, e = sorted(got_rows, key=key), sorted(exp_rows, key=key)
    for gr, er in zip(g, e):
        gk, ek = key(gr)[0], key(er)[0]
        assert gk == ek, f"{what}: row {dict(zip(names, gr))} where {dict(zip(names, er))} was expected"
        for i in soft:
            assert _soft_ok(gr[i], er[i]), \
                f"{what}: {names[i]} = {gr[i]!r}, expected {er[i][0]!r} within {er[i][1]!r} (row {dict(zip(names, er))})"


def _drawn_from(got_rows, exp_rows, kinds, names, what):
    """every got row is a distinct one of exp_rows: exact cells identical and bounded cells within their bound
    (a run of tied sort keys cut by LIMIT / OFFSET: which of the tied rows come back is not determined)"""
    hard = [i for i, k in enumerate(kinds) if k != "bounded"]
    soft = [i for i, k in enumerate(kinds) if k == "bounded"]
    pool = list(exp_rows)
    for r in got_rows:
        k = tuple(_hard(kinds[i], r[i], what) for i in hard)
        j = next((j for j, er in enumerate(pool) if tuple(_hard(kinds[i], er[i], what) for i in hard) == k
                  and all(_soft_ok(r[i], er[i]) for i in soft)), None)
        assert j is not None, f"{what}: row {dict(zip(names, r))} is not one of the tied rows"
        pool.pop(j)


def _order_key(res: Result, name, v):
    kind = res.kinds[name]
    if kind in ("float", "bounded"):
        v = v[0] if kind == "bounded" else v
        return None if v is None or math.isnan(v) else float(v) + 0.0
    return v


def assert_result(got: Dict[str, list], exp: Result, what="result"):
    """got: column name -> cells, in result order.  Fails unless got is exp: same columns, and the same rows as
    a multiset, or under ORDER BY in an order that sorts (every run of equal sort keys matched as a multiset;
    a run cut by LIMIT / OFFSET: got's rows drawn from it)."""
    names = exp.names
    assert list(got) == names, f"{what}: columns {list(got)}, expected {names}"
    kinds = [exp.kinds[n] for n in names]
    lo, hi = exp.window()
    glen = {n: len(v) for n, v in got.items()}
    assert len(set(glen.values())) <= 1, f"{what}: ragged columns {glen}"
    ng = next(iter(glen.values())) if glen else 0
    assert ng == hi - lo, f"{what}: {ng} rows, expected {hi - lo}"
    grows = list(zip(*[got[n] for n in names])) if names else []
    erows = list(zip(*[exp.cols[n] for n in names])) if names else []
    if exp.order is None:
        _match(grows, erows, kinds, names, what)
        return
    onames = [o[0] for o in exp.order]
    assert all(o in names for o in onames), "ORDER BY columns must be in the result"
    oi = [names.index(o) for o in onames]
    okey = lambda r: tuple(_order_key(exp, names[i], r[i]) for i in oi)
    s = 0
    while s < len(erows):
        e = s
        while e < len(erows) and okey(erows[e]) == okey(erows[s]):
            e += 1
        a, b = max(s, lo), min(e, hi)
        if a < b:
            seg = f"{what}: rows {a - lo}..{b - lo - 1} (sort key {okey(erows[s])})"
            if a == s and b == e:
                _match(grows[a - lo:b - lo], erows[s:e], kinds, names, seg)
            else:
                _drawn_from(grows[a - lo:b - lo], erows[s:e], kinds, names, seg)
        s = e
