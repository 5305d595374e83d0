"""NumPy restatement of the subquery mark (include/b200sql.h, b2_join_mark; DESIGN §3).

A column is (values, valid): a NumPy array and a bool array or None.  For each probe row i

  candidates(i) = build rows whose keys equal i's; a NULL key (validity clear, or NaN in a float key) equals
                  nothing, and -0.0 equals +0.0;
  mark(i)       = the three-valued OR over the candidates j of the three-valued AND of the pair terms
                  probe[i] <cmp> build[j], a term being NULL when either side's validity bit is clear
                  (NaN compares as IEEE).  A term of the subquery's own WHERE (`where` set) rejects the
                  candidate when it is NULL, as WHERE does; only the IN's own `x = y` stays NULL, and it takes a
                  float NaN for NULL too, as a key does;
  null_aware    : the single key is the IN operand x of `x IN (SELECT y ...)`: a NULL x gives NULL unless the
                  build side is empty, and a FALSE mark is NULL when the build side holds a NULL y.

Rows outside `passes` are FALSE.  The result is (values uint8, valid bool): NULL is valid False, value 0."""
import operator

import numpy as np

CMPS = {"=": operator.eq, "!=": operator.ne, "<": operator.lt, "<=": operator.le, ">": operator.gt,
        ">=": operator.ge}
CMP_CODE = {"=": 0, "!=": 1, "<": 2, "<=": 3, ">": 4, ">=": 5}


def _valid(col):
    vals, valid = col
    ok = np.ones(len(vals), bool) if valid is None else np.asarray(valid, bool).copy()
    if vals.dtype.kind == "f":
        ok &= ~np.isnan(vals)
    return ok


def _key(vals, i):
    v = vals[i]
    return 0.0 if vals.dtype.kind == "f" and v == 0 else v.item()


def mark(pkeys, bkeys, terms=(), null_aware=False, passes=None):
    """pkeys / bkeys: [column]; terms: [(probe column, build column, cmp[, where])] with cmp one of CMPS."""
    n = len(pkeys[0][0])
    m = len(bkeys[0][0])
    pok = np.logical_and.reduce([_valid(c) for c in pkeys])
    bok = np.logical_and.reduce([_valid(c) for c in bkeys]) if m else np.zeros(0, bool)
    table = {}
    for j in np.flatnonzero(bok):
        table.setdefault(tuple(_key(c[0], j) for c in bkeys), []).append(j)
    build_has_null = bool(m) and not bok.all()
    out = np.zeros(n, np.uint8)
    valid = np.ones(n, bool)
    pterms = [(t[0][0], np.ones(n, bool) if t[0][1] is None else np.asarray(t[0][1], bool),
               t[1][0], np.ones(m, bool) if t[1][1] is None else np.asarray(t[1][1], bool), CMPS[t[2]],
               len(t) > 3 and t[3]) for t in terms]
    for i in range(n):
        if passes is not None and not passes[i]:
            continue
        if not pok[i]:
            valid[i] = not (null_aware and m > 0)
            continue
        res = False                                  # False / None / True
        for j in table.get(tuple(_key(c[0], i) for c in pkeys), ()):
            t = True
            for pv, pvalid, bv, bvalid, fn, where in pterms:
                nan = not where and ((pv.dtype.kind == "f" and np.isnan(pv[i])) or
                                     (bv.dtype.kind == "f" and np.isnan(bv[j])))
                if not (pvalid[i] and bvalid[j]) or nan:
                    if where:
                        t = False
                        break
                    t = None
                elif not fn(pv[i], bv[j]):
                    t = False
                    break
            if t is True:
                res = True
                break
            if t is None:
                res = None
        if res is False and null_aware and build_has_null:
            res = None
        out[i] = res is True
        valid[i] = res is not None
    return out, valid


def sql_value(out, valid):
    """the mark as a list of SQL values: True / False / None"""
    return [bool(v) if ok else None for v, ok in zip(out, valid)]
