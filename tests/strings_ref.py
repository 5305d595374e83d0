"""Independent host reference of the VARCHAR rules: the dictionary (Python's sorted(set(...))), LIKE
(re.fullmatch with DOTALL on a translated pattern) and the lower bound (bisect on UTF-8 bytes)."""
import bisect
import re


def dictionary(values):
    """sorted unique non-NULL values: Python str order is code-point order is UTF-8 byte order"""
    return sorted(set(v for v in values if v is not None))


def codes(values, d):
    pos = {s: i for i, s in enumerate(d)}
    return [None if v is None else pos[v] for v in values]


def like_regex(pattern, escape="\\", fold=lambda c: c):
    """the escape character is recognised as written; `fold` applies to the literal characters only"""
    out, i = [], 0
    while i < len(pattern):
        ch = pattern[i]
        if escape is not None and ch == escape and i + 1 < len(pattern):
            out.append(re.escape(fold(pattern[i + 1])))
            i += 2
            continue
        out.append(".*" if ch == "%" else "." if ch == "_" else re.escape(fold(ch)))
        i += 1
    return "".join(out)


def like(s, pattern, escape="\\", ilike=False):
    fold = _fold if ilike else (lambda c: c)      # ILIKE folds ASCII A-Z only, on both sides
    return re.fullmatch(like_regex(pattern, escape, fold), fold(s), re.DOTALL) is not None


def _fold(s):
    return "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in s)


def lower_bound(a, s):
    """first position of sorted list `a` whose entry is >= s, by UTF-8 bytes"""
    return bisect.bisect_left([x.encode("utf-8") for x in a], s.encode("utf-8"))


def lb_match(a, b):
    """code of each entry of b in a, None when a lacks it"""
    pos = {s: i for i, s in enumerate(a)}
    return [pos.get(s) for s in b]


def lb_order(a, b):
    """2 * lower bound - (1 if absent)"""
    out = []
    for s in b:
        lb = lower_bound(a, s)
        out.append(2 * lb - (0 if lb < len(a) and a[lb] == s else 1))
    return out
