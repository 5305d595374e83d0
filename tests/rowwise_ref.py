"""Exact NumPy reference of the row-wise kernels: the postfix interpreter (b2_expr_eval), predicate
terms (b2_eval_terms, shared by every fused scan), the stable ORDER BY permutation (b2_sort_by), gather
(b2_gather) and column statistics (b2_col_stats).  Every output bit of these kernels is determined, so
the expected values here are exact, not approximations.

A column is a `Column(values, null, dtype)`: `values` an int64 / float64 / uint8 array, `null` a bool
array (True = the validity bit is clear) or None.  The semantics follow the reference (pandas / NumPy):
  * int64 arithmetic wraps (two's complement); DIV_I truncates toward zero and MOD_I is floored (the
    result takes the divisor's sign, NumPy's np.mod and Python's %); x / 0 and x % 0 are NULL;
  * float64 + - * / sqrt are IEEE round-to-nearest (the library is built without fast-math), so NumPy
    reproduces them bit for bit;
  * AND / OR are Kleene (False wins over NULL in AND, True in OR); CASE takes the else branch on a NULL
    condition; ISNULL_F and the F64 IS [NOT] NULL terms count NaN as NULL;
  * F2I truncates toward zero, NaN -> NULL, and saturates: +inf and x >= 2^63 give INT64_MAX, -inf and
    x < -2^63 give INT64_MIN (DESIGN.md section 6);
  * comparisons are IEEE: NaN is unordered, only NE is true for it.
No GPU and no package import: this module only needs NumPy and the opcode numbers passed in by the
caller (the tests take them from dask_sql_b200._lib)."""
from dataclasses import dataclass
from typing import Optional

import numpy as np

I64, F64, U8 = 0, 1, 2
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIGN = np.uint64(1 << 63)

# opcodes and term operators: the numbers of include/b200sql.h
OP_LOAD, OP_CONST_I, OP_CONST_F, OP_CONST_NULL, OP_I2F, OP_F2I = 0, 1, 2, 3, 4, 5
OP_ADD_I, OP_SUB_I, OP_MUL_I, OP_DIV_I, OP_NEG_I, OP_ABS_I, OP_MOD_I = 10, 11, 12, 13, 14, 15, 16
OP_ADD_F, OP_SUB_F, OP_MUL_F, OP_DIV_F, OP_NEG_F, OP_ABS_F, OP_SQRT_F = 20, 21, 22, 23, 24, 25, 26
OP_EQ_I, OP_EQ_F = 30, 40
OP_AND, OP_OR, OP_NOT, OP_ISNULL_I, OP_ISNULL_F, OP_CASE, OP_FILLNA, OP_ORD2F = 50, 51, 52, 53, 54, 55, 56, 57
EQ, NE, LT, LE, GT, GE, IS_NULL, IS_NOT_NULL, IS_TRUE = range(9)


@dataclass
class Column:
    values: np.ndarray
    null: Optional[np.ndarray]
    dtype: int

    @property
    def n(self):
        return len(self.values)

    def null_mask(self):
        return np.zeros(self.n, bool) if self.null is None else self.null

    def raw(self):
        """the 64-bit words the kernels load (U8 widened to 0..255, F64 as its bit pattern)"""
        if self.dtype == U8:
            return self.values.astype(np.int64)
        return self.values.view(np.int64)


# ---- scalar helpers -----------------------------------------------------------------------------
def f2bits(x) -> np.ndarray:
    return np.asarray(x, dtype=np.float64).view(np.int64)


def bits2f(b) -> np.ndarray:
    return np.asarray(b, dtype=np.int64).view(np.float64)


def ordered(bits) -> np.ndarray:
    """order-preserving int64 image of float64 bits (b2_ordered_from_bits; an involution)"""
    b = np.asarray(bits, dtype=np.int64)
    return b ^ ((b >> 63) & np.int64(INT64_MAX))


def _u(a):
    return a.view(np.uint64)


def wrap_add(a, b):
    return (_u(a) + _u(b)).view(np.int64)


def wrap_sub(a, b):
    return (_u(a) - _u(b)).view(np.int64)


def wrap_mul(a, b):
    return (_u(a) * _u(b)).view(np.int64)


def wrap_neg(a):
    return (np.uint64(0) - _u(a)).view(np.int64)


def div_trunc(a, b):
    """(quotient truncated toward zero, is_null) with x / 0 NULL and INT64_MIN / -1 wrapping"""
    zero, m1 = b == 0, b == -1
    safe = np.where(zero | m1, 1, b)
    q = a // safe                                            # floored ...
    q = q + ((np.mod(a, safe) != 0) & ((a < 0) != (safe < 0)))  # ... one up when it rounded down
    return np.where(m1, wrap_neg(a), np.where(zero, 0, q)), zero


def mod_floor(a, b):
    """(a mod b floored, is_null): the sign of b, x % 0 NULL, x % -1 = 0"""
    zero, m1 = b == 0, b == -1
    safe = np.where(zero | m1, 1, b)
    return np.where(zero | m1, 0, np.mod(a, safe)), zero


def f2i(bits):
    """(F2I of float64 bits, is_null): truncate, NaN -> NULL, saturate at the int64 range"""
    d = bits2f(bits)
    nan = np.isnan(d)
    hi, lo = d >= 2.0 ** 63, d < -(2.0 ** 63)
    inside = ~(nan | hi | lo)
    v = np.zeros(d.shape, np.int64)
    v[inside] = np.trunc(d[inside]).astype(np.int64)
    v[hi], v[lo] = INT64_MAX, INT64_MIN
    return v, nan


def _cmp(op, a, b):
    with np.errstate(invalid="ignore"):
        return [a == b, a != b, a < b, a <= b, a > b, a >= b][op]


# ---- the postfix interpreter -----------------------------------------------------------------------
def eval_prog(code, out_dtype, cols, n):
    """code: [(op, a, imm_i, imm_f)].  Returns (out, valid): out as the kernel writes it (int64 words
    for I64 / F64, uint8 for U8; 0 on NULL rows), valid a bool array."""
    st = []
    for op, a, imm_i, imm_f in code:
        if op == OP_LOAD:
            c = cols[a]
            st.append((c.raw()[:n].copy(), c.null_mask()[:n].copy()))
        elif op == OP_CONST_I:
            st.append((np.full(n, imm_i, np.int64), np.zeros(n, bool)))
        elif op == OP_CONST_F:
            st.append((np.full(n, f2bits(imm_f), np.int64), np.zeros(n, bool)))
        elif op == OP_CONST_NULL:
            st.append((np.zeros(n, np.int64), np.ones(n, bool)))
        elif op in (OP_I2F, OP_F2I, OP_NEG_I, OP_ABS_I, OP_NEG_F, OP_ABS_F, OP_SQRT_F, OP_ORD2F, OP_NOT,
                    OP_ISNULL_I, OP_ISNULL_F):
            v, nl = st.pop()
            if op == OP_I2F:
                v = f2bits(v.astype(np.float64))
            elif op == OP_F2I:
                v, nan = f2i(v)
                nl = nl | nan
            elif op == OP_NEG_I:
                v = wrap_neg(v)
            elif op == OP_ABS_I:
                v = np.where(v < 0, wrap_neg(v), v)
            elif op == OP_NEG_F:
                v = (_u(v) ^ SIGN).view(np.int64)
            elif op == OP_ABS_F:
                v = (_u(v) & ~SIGN).view(np.int64)
            elif op == OP_SQRT_F:
                with np.errstate(invalid="ignore"):
                    v = f2bits(np.sqrt(bits2f(v)))
            elif op == OP_ORD2F:
                v = ordered(v)
            elif op == OP_NOT:
                v = (v == 0).astype(np.int64)
            elif op == OP_ISNULL_I:
                v, nl = nl.astype(np.int64), np.zeros(n, bool)
            else:  # ISNULL_F
                v, nl = (nl | np.isnan(bits2f(v))).astype(np.int64), np.zeros(n, bool)
            st.append((v, nl))
        elif op == OP_CASE:
            (ev, en), (tv, tn), (cv, cn) = st.pop(), st.pop(), st.pop()
            take = ~cn & (cv != 0)
            st.append((np.where(take, tv, ev), np.where(take, tn, en)))
        elif op == OP_FILLNA:
            (fv, fn), (xv, xn) = st.pop(), st.pop()
            st.append((np.where(xn, fv, xv), np.where(xn, fn, xn)))
        else:
            (b, bn), (a_, an) = st.pop(), st.pop()
            rn = an | bn
            if op == OP_AND:
                af, bf = ~an & (a_ == 0), ~bn & (b == 0)
                r, rn = (~an & (a_ != 0)) & (~bn & (b != 0)), rn & ~(af | bf)
            elif op == OP_OR:
                at, bt = ~an & (a_ != 0), ~bn & (b != 0)
                r, rn = at | bt, rn & ~(at | bt)
            elif OP_EQ_F <= op <= OP_EQ_F + 5:
                r = _cmp(op - OP_EQ_F, bits2f(a_), bits2f(b))
            elif OP_EQ_I <= op <= OP_EQ_I + 5:
                r = _cmp(op - OP_EQ_I, a_, b)
            elif op == OP_ADD_I:
                r = wrap_add(a_, b)
            elif op == OP_SUB_I:
                r = wrap_sub(a_, b)
            elif op == OP_MUL_I:
                r = wrap_mul(a_, b)
            elif op == OP_DIV_I:
                r, z = div_trunc(a_, b)
                rn = rn | z
            elif op == OP_MOD_I:
                r, z = mod_floor(a_, b)
                rn = rn | z
            elif OP_ADD_F <= op <= OP_DIV_F:
                x, y = bits2f(a_), bits2f(b)
                with np.errstate(all="ignore"):
                    r = f2bits([x + y, x - y, x * y, x / y][op - OP_ADD_F])
            else:
                raise ValueError(f"opcode {op}")
            st.append((np.asarray(r).astype(np.int64), rn))
    assert len(st) == 1, "program must leave exactly one value"
    v, nl = st[0]
    v = np.where(nl, 0, v)
    if out_dtype == U8:
        v = (v != 0).astype(np.uint8)
    return v, ~nl


def prog_code(prog):
    """[(op, a, imm_i, imm_f)] of a dask_sql_b200._lib.Prog"""
    return [(prog.code[i].op, prog.code[i].a, prog.code[i].imm_i, prog.code[i].imm_f) for i in range(prog.n)]


# ---- predicate terms ---------------------------------------------------------------------------------
def eval_term(col: Column, op, as_f64=0, lit_i=0, lit_f=0.0):
    """rows of `col` that pass one b2_term_t"""
    null = col.null_mask()
    if op in (IS_NULL, IS_NOT_NULL):
        nul = null | (np.isnan(col.values) if col.dtype == F64 else False)
        return nul if op == IS_NULL else ~nul
    if op == IS_TRUE:
        ok = col.raw() != 0
    elif col.dtype == F64:
        ok = _cmp(op, col.values, np.float64(lit_f))
    elif as_f64:
        ok = _cmp(op, col.raw().astype(np.float64), np.float64(lit_f))
    else:
        ok = _cmp(op, col.raw(), np.int64(lit_i))
    return ok & ~null


def eval_terms(cols, terms, n):
    """terms: [(col index, op, as_f64, lit_i, lit_f)]; a conjunction"""
    ok = np.ones(n, bool)
    for c, op, as_f64, lit_i, lit_f in terms:
        ok &= eval_term(cols[c], op, as_f64, lit_i, lit_f)[:n]
    return ok


# ---- ORDER BY -----------------------------------------------------------------------------------------
def sort_perm(col: Column, idx, descending, nulls_first):
    """b2_sort_by: `idx` reordered so that col[idx] is stably sorted.  NaN is NULL; -0.0 ties with 0.0."""
    idx = np.asarray(idx, np.int64)
    v = col.values[idx]
    null = col.null_mask()[idx]
    if col.dtype == F64:
        null = null | np.isnan(v)
        v = np.where(v == 0, 0.0, v)            # -0.0 -> 0.0
    v = np.where(null, v.dtype.type(0), v)
    _, rank = np.unique(v, return_inverse=True)
    rank = rank.reshape(-1).astype(np.int64)
    key = -rank if descending else rank
    nkey = (~null if nulls_first else null).astype(np.int64)
    return idx[np.lexsort((key, nkey))].astype(np.int32)


# ---- gather -------------------------------------------------------------------------------------------
def gather(col: Column, idx):
    """b2_gather: (out values, valid); idx -1 -> NULL with 0 (NaN for F64) in the value slot"""
    idx = np.asarray(idx, np.int64)
    miss = idx < 0
    safe = np.where(miss, 0, idx)
    out = col.values[safe].copy() if len(col.values) else np.zeros(len(idx), col.values.dtype)
    out[miss] = np.nan if col.dtype == F64 else 0
    valid = ~miss & ~col.null_mask()[safe] if len(col.values) else ~miss
    return out, valid


# ---- column statistics --------------------------------------------------------------------------------
def col_stats(col: Column):
    """{min, max, null_count, n_nan} as b2_col_stats reports them: min / max are int64 words (float bits
    for F64, ordered so that -0.0 < +0.0), INT64_MAX / INT64_MIN when no value qualifies"""
    null = col.null_mask()
    raw = col.raw()
    keep = ~null
    n_nan = 0
    if col.dtype == F64:
        nan = np.isnan(col.values) & keep
        n_nan = int(nan.sum())
        keep &= ~nan
        img = ordered(raw)
    else:
        img = raw
    if keep.any():
        mn, mx = int(img[keep].min()), int(img[keep].max())
        if col.dtype == F64:
            mn, mx = int(ordered(mn)), int(ordered(mx))
    else:
        mn, mx = INT64_MAX, INT64_MIN
    return {"min": mn, "max": mx, "null_count": int(null.sum()), "n_nan": n_nan}


# ---- validity bitmaps ----------------------------------------------------------------------------------
def pack_valid(valid: np.ndarray) -> np.ndarray:
    """bool[n] -> uint32 words, LSB first (Arrow), bits at and after n clear"""
    n = len(valid)
    out = np.zeros(((n + 31) // 32) * 4, np.uint8)
    b = np.packbits(valid.astype(bool), bitorder="little")
    out[: len(b)] = b
    return out.view(np.uint32)
