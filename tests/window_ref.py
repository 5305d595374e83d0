"""Exact reference of the window functions, as `Context.sql()` answers them (DESIGN.md section 6).

`window(rel, partition, order, fn, arg, frame)` -> the cells of one window column, in the relation's row order,
of the kind `tests.query_ref.Result` compares:
  * rows are ordered by the PARTITION BY keys (ascending, NULLs last), then the ORDER BY keys [(name, asc,
    nulls_first)], stably; two rows share a partition / are peers when all those keys are equal, with NULL and
    NaN one value and -0.0 == +0.0 (the sort's key images);
  * frame = (is_range, lo, hi): ROWS offsets from the row's sorted position, -inf / +inf for UNBOUNDED;
    RANGE takes -inf / 0 / +inf, and CURRENT ROW is the row's first (lo) or last (hi) peer; the frame is
    clamped to the partition and may be empty;
  * ROW_NUMBER = 1 + position in the partition, RANK = 1 + rows before the first peer, DENSE_RANK = 1 +
    peer groups before; COUNT(*) = frame rows, COUNT(x) = its non-NULL values; SUM / AVG / MIN / MAX skip
    NULLs and are NULL without a value; FIRST_VALUE / LAST_VALUE are the value at the frame's ends;
  * int64 SUM wraps; a float SUM or an AVG is "bounded": the exact (Fraction) value, within one rounding
    plus 2^-100 * sum |x| over the partition up to the frame's end (AVG: that over the count, plus one more
    rounding); MIN / MAX order -0.0 below +0.0.
No GPU and no package import."""
import math
from fractions import Fraction

import numpy as np

from tests.query_ref import STR, U, is_null
from tests.rowwise_ref import F64, I64, U8

INF = float("inf")


def _key_cells(col):
    """per row: (is NULL, comparable value) with -0.0 == +0.0"""
    null = is_null(col)
    out = []
    for v, nl in zip(col.values, null):
        if nl:
            out.append((True, 0))
        elif col.dtype == F64:
            out.append((False, float(v) + 0.0))
        elif col.dtype == STR:
            out.append((False, v))
        else:
            out.append((False, int(v)))
    return out


def sort_positions(rel, partition, order):
    """the sorted row order, and per sorted position its partition key and peer key"""
    n = len(next(iter(rel.values())).values)
    perm = list(range(n))
    keys = [(p, True, False) for p in partition] + list(order)
    cells = {name: _key_cells(rel[name]) for name, _, _ in keys}
    for name, asc, nulls_first in reversed(keys):
        c = cells[name]
        nonnull = sorted([r for r in perm if not c[r][0]], key=lambda r: c[r][1], reverse=not asc)
        nulls = [r for r in perm if c[r][0]]
        perm = nulls + nonnull if nulls_first else nonnull + nulls
    pkey = [tuple(cells[p][r] for p in partition) for r in perm]
    qkey = [tuple(cells[k][r] for k, _, _ in keys) for r in perm]
    return perm, pkey, qkey


def _runs(keys):
    """per position: (start, end) of its run of equal keys"""
    n = len(keys)
    start, end = [0] * n, [0] * n
    s = 0
    while s < n:
        e = s
        while e + 1 < n and keys[e + 1] == keys[s]:
            e += 1
        for i in range(s, e + 1):
            start[i], end[i] = s, e
        s = e + 1
    return start, end


def frame_bounds(i, ps, pe, qs, qe, frame):
    is_range, lo, hi = frame
    if is_range:
        a = ps if lo == -INF else qs if lo == 0 else pe + 1
        b = pe if hi == INF else qe if hi == 0 else ps - 1
    else:
        a = ps if lo == -INF else pe + 1 if lo == INF else i + int(lo)
        b = pe if hi == INF else ps - 1 if hi == -INF else i + int(hi)
    return max(a, ps), min(b, pe)


def _wrap(x: int) -> int:
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= 1 << 63 else x


def _image(col, v):
    """MIN / MAX order of a value: the int, or the ordered image of the double's bits"""
    if col.dtype == F64:
        b = int(np.float64(v).view(np.int64))
        return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)
    return v


def window(rel, partition, order, fn, arg, frame):
    """-> (kind, cells) of the window column in row order; fn in ROW_NUMBER / RANK / DENSE_RANK / COUNT /
    SUM / AVG / MIN / MAX / FIRST_VALUE / LAST_VALUE, arg a column name (None for COUNT(*) and the ranks)"""
    perm, pkey, qkey = sort_positions(rel, partition, order)
    n = len(perm)
    pstart, pend = _runs(pkey)
    qstart, qend = _runs(qkey)
    col = rel[arg] if arg is not None else None
    null = is_null(col) if col is not None else None
    vals = col.values if col is not None else None
    out = [None] * n
    # per sorted position, prefixes within the partition: non-NULL values, exact sum, |x| of finite values
    # (AVG of an integer column sums the values converted to double, as the GROUP BY AVG does: ftot)
    cnt, tot, ftot, span = [0] * n, [Fraction(0)] * n, [Fraction(0)] * n, [0.0] * n
    if col is not None:
        for i, r in enumerate(perm):
            first = i == pstart[i]
            c0, t0, f0, s0 = (0, Fraction(0), Fraction(0), 0.0) if first else \
                (cnt[i - 1], tot[i - 1], ftot[i - 1], span[i - 1])
            ok = not null[r]
            x = vals[r]
            finite = ok and (col.dtype != F64 or math.isfinite(float(x)))
            cnt[i] = c0 + ok
            tot[i] = t0 + (Fraction(int(x)) if col.dtype != F64 else Fraction(float(x))) if finite and \
                col.dtype in (I64, F64, U8) else t0
            ftot[i] = f0 + Fraction(float(x)) if finite and col.dtype in (I64, F64, U8) else f0
            span[i] = s0 + (abs(float(x)) if finite and col.dtype in (I64, F64, U8) else 0.0)
    if col is not None and col.dtype != STR:
        img = np.array([_image(col, vals[r]) if not null[r] else 0 for r in perm], np.int64)
        nulls = np.array([bool(null[r]) for r in perm])
        lo_img, hi_img = np.where(nulls, np.iinfo(np.int64).max, img), np.where(nulls, np.iinfo(np.int64).min, img)
        isf = col.dtype == F64
        pinf = np.cumsum([isf and not null[r] and float(vals[r]) == INF for r in perm])
        ninf = np.cumsum([isf and not null[r] and float(vals[r]) == -INF for r in perm])
    dense, prev_part, prev_q = 0, None, None
    for i, r in enumerate(perm):
        ps, pe, qs, qe = pstart[i], pend[i], qstart[i], qend[i]
        if ps != prev_part:
            dense, prev_part, prev_q = 0, ps, None
        if qs != prev_q:
            dense, prev_q = dense + 1, qs
        if fn == "ROW_NUMBER":
            out[r] = i - ps + 1
            continue
        if fn == "RANK":
            out[r] = qs - ps + 1
            continue
        if fn == "DENSE_RANK":
            out[r] = dense
            continue
        lo, hi = frame_bounds(i, ps, pe, qs, qe, frame)
        if lo > hi:
            out[r] = 0 if fn == "COUNT" else None
            continue
        if fn == "COUNT":
            out[r] = hi - lo + 1 if col is None else cnt[hi] - (cnt[lo - 1] if lo > ps else 0)
            continue
        if fn in ("FIRST_VALUE", "LAST_VALUE"):
            x = perm[lo] if fn == "FIRST_VALUE" else perm[hi]
            out[r] = None if null[x] else vals[x]
            continue
        if cnt[hi] - (cnt[lo - 1] if lo > ps else 0) == 0:
            out[r] = None
            continue
        if fn in ("MIN", "MAX"):
            if col.dtype == STR:
                present = [vals[x] for x in perm[lo:hi + 1] if not null[x]]
                out[r] = min(present) if fn == "MIN" else max(present)
            else:
                j = lo + int(np.argmin(lo_img[lo:hi + 1]) if fn == "MIN" else np.argmax(hi_img[lo:hi + 1]))
                out[r] = vals[perm[j]]
            continue
        if fn == "SUM" and col.dtype != F64:
            out[r] = _wrap(int(tot[hi] - (tot[lo - 1] if lo > ps else 0)))
            continue
        exact = ftot[hi] - (ftot[lo - 1] if lo > ps else 0)
        infs = ([INF] if pinf[hi] - (pinf[lo - 1] if lo else 0) else []) + \
            ([-INF] if ninf[hi] - (ninf[lo - 1] if lo else 0) else [])
        count = cnt[hi] - (cnt[lo - 1] if lo > ps else 0)
        out[r] = _float_sum(exact, infs, span[hi], count if fn == "AVG" else None)
    return _kind(fn, col), [_cell(fn, col, v) for v in out]


def _float_sum(exact, infs, span, count):
    """(exact, bound) of a float SUM (count None) or AVG: exact = the frame's exact sum of its finite values,
    infs = its infinities"""
    pinf, ninf = INF in infs, -INF in infs
    if pinf and ninf:
        return (math.nan, 0.0)
    if pinf or ninf:
        return (INF if pinf else -INF, 0.0)
    bound = abs(float(exact)) * U + span * 2.0 ** -100
    if count is not None:
        exact = exact / count
        bound = bound / count + abs(float(exact)) * U
    return (float(exact), bound)


def _kind(fn, col):
    if fn in ("ROW_NUMBER", "RANK", "DENSE_RANK", "COUNT"):
        return "int"
    if fn == "AVG" or (fn == "SUM" and col.dtype == F64):
        return "bounded"
    if col.dtype == F64:
        return "float"
    if col.dtype == STR:
        return "str"
    if col.dtype == U8 and fn in ("FIRST_VALUE", "LAST_VALUE"):
        return "bool"
    return "int"


def _cell(fn, col, v):
    if isinstance(v, tuple) or v is None:
        return v if v is not None or _kind(fn, col) != "bounded" else (math.nan, 0.0)
    if col is None or fn == "COUNT":
        return int(v)
    k = _kind(fn, col)
    if k == "float":
        return float(v)
    if k == "bool":
        return bool(v)
    if k == "str":
        return str(v)
    return int(v)
