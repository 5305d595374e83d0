"""DATE and TIMESTAMP: the one place that knows units, ticks per unit and calendar rules.

Representation (physical I64 on the device, like every integer column):
  * TIMESTAMP -- the count of the column's own unit since 1970-01-01 00:00:00, logical dtype
    `datetime64[s|ms|us|ns]`: the unit the input arrived with.  Units are never normalised: ns -> us
    would truncate data, s -> ns overflows past 2262 (and 9999-12-31 is a common sentinel).
  * DATE -- days since 1970-01-01, logical dtype `date32[day]`.
  * NULL -- the validity bitmap (pandas NaT at the boundaries).
When two temporal operands meet (comparison, join key, CASE branches, DATE vs TIMESTAMP) the coarser
one is scaled to the finer unit by an int64 multiply, wrapping like NumPy's astype.  A value with no
unit of its own (a TIMESTAMP literal, CAST(date AS TIMESTAMP)) is in microseconds, pandas' default.

Calendar arithmetic on columns runs on the device (B2_OP_DATEPART / B2_OP_ADDMONTHS of b2_expr_eval);
the scalar functions here follow the same rules for constant folding and statistics.
"""
import datetime as _dt
import re
from typing import Optional

import numpy as np

DATE_LOGICAL = "date32[day]"
DEFAULT_UNIT = "us"
# ticks per second of each unit; "D" (days) has none, the device opcodes take 0 for it
TPS = {"D": 0, "s": 1, "ms": 10 ** 3, "us": 10 ** 6, "ns": 10 ** 9}
NS_PER_DAY = 86400 * 10 ** 9
_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1
_LOGICAL_RE = re.compile(r"datetime64\[(s|ms|us|ns)\]")


# ---------------------------------------------------------------------------------------------
# units
# ---------------------------------------------------------------------------------------------
def unit_of(logical) -> Optional[str]:
    """"D" for a DATE, the tick unit of a TIMESTAMP, None for anything else."""
    logical = str(logical)
    if logical in (DATE_LOGICAL, "datetime64[D]"):
        return "D"
    m = _LOGICAL_RE.fullmatch(logical)
    return m.group(1) if m else None


def is_temporal(logical) -> bool:
    return unit_of(logical) is not None


def logical_of(unit: str) -> str:
    return DATE_LOGICAL if unit == "D" else f"datetime64[{unit}]"


def sql_type_of(logical) -> Optional[str]:
    u = unit_of(logical)
    return None if u is None else ("DATE" if u == "D" else "TIMESTAMP")


def numpy_dtype(logical) -> np.dtype:
    """The dtype a lazy frame reports for a column of this logical type: datetime64[D] for a DATE.

    That is the SQL type the catalog reads back (mappings.python_to_sql_type: datetime64[D] is DATE, any
    finer unit is TIMESTAMP), so a DATE column of a registered frame or CREATE TABLE AS stays a DATE.  The
    values compute() returns are datetime64[s] at midnight instead (to_host_array): pandas has no
    datetime64[D] column type: a datetime64[D] array becomes datetime64[s] in a Series."""
    return np.dtype(f"datetime64[{unit_of(logical)}]")


def ticks_per_day(unit: str) -> int:
    return 1 if unit == "D" else TPS[unit] * 86400


def finer(u: str, v: str) -> str:
    return u if ticks_per_day(u) >= ticks_per_day(v) else v


def factor(src: str, dst: str) -> int:
    """dst ticks per src tick (src at least as coarse as dst)."""
    return ticks_per_day(dst) // ticks_per_day(src)


def wrap64(v: int) -> int:
    """int64 two's-complement wrap, what NumPy's astype and the device's MUL_I do on overflow."""
    return ((int(v) - _I64_MIN) % (1 << 64)) + _I64_MIN


def fits64(v: int) -> bool:
    return _I64_MIN <= v <= _I64_MAX


# ---------------------------------------------------------------------------------------------
# calendar (proleptic Gregorian; the device code in csrc/expr.cuh is the same algorithm)
# ---------------------------------------------------------------------------------------------
def days_from_civil(y: int, m: int, d: int) -> int:
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m - 3 if m > 2 else m + 9) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def civil_from_days(z: int):
    z += 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m, d


def month_days(y: int, m: int) -> int:
    return days_from_civil(y + (m == 12), 1 if m == 12 else m + 1, 1) - days_from_civil(y, m, 1)


# B2_OP_DATEPART fields (b200sql.h B2_DP_*)
FIELDS = ("DAYS", "YEAR", "QUARTER", "MONTH", "DAY", "DOY", "DOW", "ISOWEEK", "HOUR", "MINUTE", "SECOND",
          "MILLISECOND", "MICROSECOND")
FIELD = {f: i for i, f in enumerate(FIELDS)}


def datepart(ticks: int, field: str, unit: str) -> int:
    """Field `field` of a value of `unit` -- the host twin of B2_OP_DATEPART."""
    tpd, tps = ticks_per_day(unit), TPS[unit]
    day, tod = divmod(ticks, tpd)
    if field == "DAYS":
        return day
    if field == "DOW":
        return (day + 4) % 7                  # 1970-01-01 was a Thursday; 0 = Sunday
    if FIELD[field] >= FIELD["HOUR"]:
        if not tps:
            return 0
        sub = tod % tps
        return {"HOUR": tod // (tps * 3600), "MINUTE": tod // (tps * 60) % 60, "SECOND": tod // tps % 60,
                "MILLISECOND": sub * 1000 // tps, "MICROSECOND": sub * 1000000 // tps}[field]
    if field == "ISOWEEK":
        th = day - (day + 3) % 7 + 3           # the Thursday of the ISO week decides its year
        y, _, _ = civil_from_days(th)
        return (th - days_from_civil(y, 1, 1)) // 7 + 1
    y, m, d = civil_from_days(day)
    return {"YEAR": y, "QUARTER": (m - 1) // 3 + 1, "MONTH": m, "DAY": d,
            "DOY": day - days_from_civil(y, 1, 1) + 1}[field]


def add_months(ticks: int, n: int, unit: str, to_last: bool = False) -> int:
    """`ticks` moved by n calendar months, the day clamped to the target month's last day, the time of
    day kept; to_last: then moved to the last day of its month -- the host twin of B2_OP_ADDMONTHS."""
    tpd = ticks_per_day(unit)
    day, tod = divmod(ticks, tpd)
    y, m, d = civil_from_days(day)
    y2, m0 = divmod(y * 12 + m - 1 + n, 12)
    last = month_days(y2, m0 + 1)
    d2 = last if to_last else min(d, last)
    return wrap64((days_from_civil(y2, m0 + 1, d2)) * tpd + tod)


# ---------------------------------------------------------------------------------------------
# host scalars
# ---------------------------------------------------------------------------------------------
class TScalar:
    """A DATE (unit "D") or TIMESTAMP value on the host: ticks of `unit` since the epoch."""
    __slots__ = ("ticks", "unit")

    def __init__(self, ticks: int, unit: str):
        self.ticks, self.unit = int(ticks), unit

    @property
    def logical(self):
        return logical_of(self.unit)

    def at(self, unit: str) -> int:
        """ticks at a unit at least as fine as this one (exact)"""
        return self.ticks * factor(self.unit, unit)

    def _cmp_key(self, other):
        if isinstance(other, str):
            other = parse_like(other, self)
        if not isinstance(other, TScalar):
            return NotImplemented
        u = finer(self.unit, other.unit)
        return self.at(u), other.at(u)

    def _cmp(self, other, fn):
        k = self._cmp_key(other)
        return k if k is NotImplemented else fn(*k)

    def __eq__(self, o): return self._cmp(o, lambda a, b: a == b)
    def __ne__(self, o): return self._cmp(o, lambda a, b: a != b)
    def __lt__(self, o): return self._cmp(o, lambda a, b: a < b)
    def __le__(self, o): return self._cmp(o, lambda a, b: a <= b)
    def __gt__(self, o): return self._cmp(o, lambda a, b: a > b)
    def __ge__(self, o): return self._cmp(o, lambda a, b: a >= b)

    def __hash__(self):
        return hash(self.at("ns")) if self.unit != "ns" else hash(self.ticks)

    def __add__(self, o):
        if isinstance(o, Interval):
            return add_interval_scalar(self, o, 1)
        raise NotImplementedError(f"{sql_type_of(self.logical)} + {type(o).__name__}: add an INTERVAL")

    __radd__ = __add__

    def __sub__(self, o):
        if isinstance(o, Interval):
            return add_interval_scalar(self, o, -1)
        raise NotImplementedError("the difference of two dates / timestamps is an interval, which is not a "
                                  "column type here; use TIMESTAMPDIFF(unit, a, b)")

    def to_numpy(self):
        return np.datetime64(self.ticks, self.unit)

    def __str__(self):
        if self.unit == "D":
            return str(np.datetime64(self.ticks, "D"))
        return str(np.datetime64(self.ticks, self.unit)).replace("T", " ")

    def __repr__(self):
        return f"{sql_type_of(self.logical)} '{self}'"


class Interval:
    """INTERVAL literal: whole months (calendar part) and nanoseconds (fixed part)."""
    __slots__ = ("months", "ns")

    def __init__(self, months: int = 0, ns: int = 0):
        self.months, self.ns = int(months), int(ns)

    def __neg__(self):
        return Interval(-self.months, -self.ns)

    def __eq__(self, o):
        return isinstance(o, Interval) and (o.months, o.ns) == (self.months, self.ns)

    def __hash__(self):
        return hash((self.months, self.ns))

    def __str__(self):
        return f"{self.months} months {self.ns} ns"

    __repr__ = __str__


# interval / TIMESTAMPADD / TIMESTAMPDIFF units -> (months, nanoseconds)
_UNIT_SIZE = {"YEAR": (12, 0), "QUARTER": (3, 0), "MONTH": (1, 0), "WEEK": (0, 7 * NS_PER_DAY),
              "DAY": (0, NS_PER_DAY), "HOUR": (0, 3600 * 10 ** 9), "MINUTE": (0, 60 * 10 ** 9),
              "SECOND": (0, 10 ** 9), "MILLISECOND": (0, 10 ** 6), "MICROSECOND": (0, 10 ** 3),
              "NANOSECOND": (0, 1)}


def norm_unit(name: str) -> str:
    u = str(name).upper()
    u = {"YEARS": "YEAR", "QUARTERS": "QUARTER", "MONTHS": "MONTH", "WEEKS": "WEEK", "DAYS": "DAY",
         "HOURS": "HOUR", "MINUTES": "MINUTE", "SECONDS": "SECOND", "MILLISECONDS": "MILLISECOND",
         "MICROSECONDS": "MICROSECOND", "NANOSECONDS": "NANOSECOND", "SQL_TSI_YEAR": "YEAR",
         "SQL_TSI_MONTH": "MONTH", "SQL_TSI_DAY": "DAY"}.get(u, u)
    if u not in _UNIT_SIZE:
        raise ValueError(f"unknown time unit {name!r}")
    return u


def tick_unit_of_ns(ns: int) -> str:
    """The coarsest unit that holds a nanosecond amount exactly ("D" for whole days)."""
    if ns % NS_PER_DAY == 0:
        return "D"
    for u in ("s", "ms", "us"):
        if ns % (10 ** 9 // TPS[u]) == 0:
            return u
    return "ns"


def ns_to_ticks(ns: int, unit: str) -> int:
    return ns // (NS_PER_DAY // ticks_per_day(unit))


# ---------------------------------------------------------------------------------------------
# parsing
# ---------------------------------------------------------------------------------------------
_DATE_RE = re.compile(r"\s*([+-]?\d{1,6})-(\d{1,2})-(\d{1,2})\s*")
_TS_RE = re.compile(r"\s*([+-]?\d{1,6})-(\d{1,2})-(\d{1,2})(?:[ T](\d{1,2}):(\d{1,2})(?::(\d{1,2})(?:\.(\d{1,9}))?)?)?\s*")


def _check_civil(y, m, d):
    if not (1 <= m <= 12 and 1 <= d <= month_days(y, m)):
        raise ValueError(f"{y:04d}-{m:02d}-{d:02d} is not a calendar date")


def parse_date(s: str) -> TScalar:
    m = _DATE_RE.fullmatch(s)
    if m is None:
        raise ValueError(f"{s!r} is not a DATE (YYYY-MM-DD)")
    y, mo, d = (int(g) for g in m.groups())
    _check_civil(y, mo, d)
    return TScalar(days_from_civil(y, mo, d), "D")


def parse_timestamp(s: str) -> TScalar:
    """'YYYY-MM-DD[ HH:MM[:SS[.fffffffff]]]' -> microseconds, or nanoseconds when the fraction needs them."""
    m = _TS_RE.fullmatch(s)
    if m is None:
        raise ValueError(f"{s!r} is not a TIMESTAMP (YYYY-MM-DD HH:MM:SS[.ffffff])")
    y, mo, d, hh, mi, ss, frac = m.groups()
    y, mo, d = int(y), int(mo), int(d)
    _check_civil(y, mo, d)
    hh, mi, ss = int(hh or 0), int(mi or 0), int(ss or 0)
    if hh > 23 or mi > 59 or ss > 59:
        raise ValueError(f"{s!r}: time of day out of range")
    frac = frac or ""
    unit = "ns" if len(frac) > 6 else "us"
    sub = int((frac + "0" * 9)[:9]) // (10 ** 9 // TPS[unit])
    return TScalar(((days_from_civil(y, mo, d) * 86400 + hh * 3600 + mi * 60 + ss) * TPS[unit]) + sub, unit)


def parse_like(s: str, like) -> TScalar:
    """A string met by a temporal operand is read as that operand's type."""
    return parse_date(s) if unit_of(getattr(like, "logical", like)) == "D" else parse_timestamp(s)


_IV_PART = re.compile(r"\s*([+-]?\d+)\s*([A-Za-z_]+)\s*")


def parse_interval(text: str, unit: Optional[str] = None) -> Interval:
    """INTERVAL '<n> <unit>[s] [<n> <unit> ...]'  or  INTERVAL '<n>' <unit>."""
    months = ns = 0
    if unit is not None:
        n = int(str(text).strip())
        mo, nsz = _UNIT_SIZE[norm_unit(unit)]
        return Interval(n * mo, n * nsz)
    pos, text = 0, str(text)
    if not text.strip():
        raise ValueError("empty INTERVAL")
    while pos < len(text):
        m = _IV_PART.match(text, pos)
        if m is None:
            raise ValueError(f"cannot read INTERVAL {text!r}")
        n = int(m.group(1))
        mo, nsz = _UNIT_SIZE[norm_unit(m.group(2))]
        months, ns = months + n * mo, ns + n * nsz
        pos = m.end()
    return Interval(months, ns)


# ---------------------------------------------------------------------------------------------
# host folding (same rules as the device expressions built below)
# ---------------------------------------------------------------------------------------------
def interval_result_unit(unit: str, ns: int) -> str:
    """Unit of `value(unit) + ns`: a DATE plus a sub-day amount becomes a TIMESTAMP (us at least)."""
    need = tick_unit_of_ns(ns) if ns else "D"
    if unit == "D":
        return "D" if need == "D" else finer(DEFAULT_UNIT, need)
    return finer(unit, need) if need != "D" else unit


def add_interval_scalar(x: TScalar, iv: Interval, sign: int) -> TScalar:
    months, ns = sign * iv.months, sign * iv.ns
    ticks, unit = x.ticks, x.unit
    if months:
        ticks = add_months(ticks, months, unit)
    ru = interval_result_unit(unit, ns)
    ticks = wrap64(ticks * factor(unit, ru) + ns_to_ticks(ns, ru))
    return TScalar(ticks, ru)


def stat_to_ticks(v, unit: str):
    """A Parquet statistic of a temporal column (datetime.date / datetime / pandas Timestamp / int) as ticks
    of the column's unit, so that min / max compare with the integer literals of the fused scans."""
    if v is None or isinstance(v, (int, np.integer)):
        return v
    if unit == "D":
        if isinstance(v, _dt.datetime):
            v = v.date()
        return int(np.datetime64(v, "D").astype(np.int64))
    if hasattr(v, "value") and hasattr(v, "tz"):          # pandas Timestamp: exact nanoseconds
        return int(v.value) // (10 ** 9 // TPS[unit])
    return int(np.datetime64(v).astype(f"datetime64[{unit}]").astype(np.int64))


def to_host_array(vals: np.ndarray, unit: str, mask=None) -> np.ndarray:
    """int64 ticks -> datetime64 (DATE as datetime64[s] at midnight, what pyarrow makes of date32);
    NULL -> NaT."""
    if unit == "D":
        out = vals.astype("datetime64[D]").astype("datetime64[s]")
    else:
        out = vals.view(f"datetime64[{unit}]")
    if mask is not None:
        out = out.copy()
        out[mask] = np.datetime64("NaT")
    return out


def from_host_array(vals: np.ndarray):
    """datetime64[D|s|ms|us|ns] -> (int64 ticks, null mask or None, logical)"""
    unit = np.datetime_data(vals.dtype)[0]
    if unit not in TPS:
        raise NotImplementedError(f"column dtype {vals.dtype} is outside the DATE / TIMESTAMP units s, ms, us, ns")
    nat = np.isnat(vals)
    ticks = vals.view(np.int64)
    if nat.any():
        ticks = np.where(nat, 0, ticks)
    return ticks, (nat if nat.any() else None), logical_of(unit)


# ---------------------------------------------------------------------------------------------
# device expressions (expr.Expr trees; B2_OP_DATEPART / B2_OP_ADDMONTHS plus the integer opcodes)
# ---------------------------------------------------------------------------------------------
_FLIP = {"eq": "eq", "ne": "ne", "lt": "gt", "le": "ge", "gt": "lt", "ge": "le"}


def _E():
    from . import expr
    return expr


def unit_of_expr(e) -> Optional[str]:
    if isinstance(e, TScalar):
        return e.unit
    return unit_of(getattr(e, "logical", ""))


def at_unit(e, unit: str):
    """Expression `e` (DATE / TIMESTAMP) in ticks of a unit at least as fine as its own."""
    E = _E()
    u = unit_of_expr(e)
    if u == unit:
        return e
    k = factor(u, unit)
    if isinstance(e, E.Lit):
        return E.Lit(None if e.value is None else wrap64(e.value * k), E.I64, logical_of(unit))
    return E.Call("mul", [e, E.Lit(k)], E.I64, logical_of(unit))


def _operand(x, like=None):
    """Python value / Expr -> Expr; a string next to a temporal operand is read as its type."""
    E = _E()
    if isinstance(x, str):
        if like is None:
            raise NotImplementedError("string values are outside the int64/float64/bool/DATE/TIMESTAMP hot path")
        try:
            x = parse_like(x, like)
        except ValueError as err:
            from .utils import ParsingException
            raise ParsingException(x, str(err)) from None
    if isinstance(x, Interval):
        raise NotImplementedError("INTERVAL values are not a column type here; add them to a DATE / TIMESTAMP")
    e = E.as_expr(x)
    if isinstance(e, E.Lit) and e.value is None and like is not None:
        return E.Lit(None, E.I64, like.logical)
    return e


def _round_literal(op: str, lit: int, k: int):
    """x * k <op> lit  <=>  x <op'> lit'  for integer x (k > 1): the literal, rounded toward the side that
    keeps the result.  None for = / <> when lit is not a multiple of k."""
    q, r = divmod(lit, k)
    if r == 0:
        return op, q
    if op in ("lt", "ge"):
        return op, q + 1
    if op in ("le", "gt"):
        return op, q
    return None


def _out_of_range(op: str, col, above: bool):
    """`col <op> literal` where the literal, scaled exactly onto the column's finer unit, lies above (or
    below) every int64: the comparison has the same truth value for every non-NULL row, and NULL rows stay
    NULL.  Expressed as a fused-scan term against INT64_MAX / INT64_MIN (e.g. a datetime64[ns] column
    against DATE '9999-12-31'); wrapping the literal like the column scaling does would flip the result."""
    E = _E()
    lit = lambda v: E.Lit(v, E.I64, col.logical)  # noqa: E731
    if above:    # every value < literal
        true = op in ("lt", "le", "ne")
        return E.Call("le", [col, lit(_I64_MAX)], E.U8) if true else E.Call("gt", [col, lit(_I64_MAX)], E.U8)
    true = op in ("gt", "ge", "ne")
    return E.Call("ge", [col, lit(_I64_MIN)], E.U8) if true else E.Call("lt", [col, lit(_I64_MIN)], E.U8)


def compare(op: str, a, b):
    """`a <op> b` with at least one DATE / TIMESTAMP operand."""
    E = _E()
    ta = isinstance(a, (E.Expr, TScalar)) and unit_of_expr(a) is not None
    if not ta:
        a, b, op = b, a, _FLIP[op]
    a = _operand(a)
    b = _operand(b, like=a)
    ua, ub = unit_of_expr(a), unit_of_expr(b)
    if ub is None:
        raise NotImplementedError(f"cannot compare a {sql_type_of(a.logical)} with {b.logical}")
    if isinstance(a, E.Lit) and not isinstance(b, E.Lit):      # the literal on the right
        a, b, op, ua, ub = b, a, _FLIP[op], ub, ua
    r = rewrite_cmp(op, a, b)
    if r is not None:
        return r
    if isinstance(b, E.Lit) and not isinstance(a, E.Lit) and b.value is not None and ua != ub \
            and ticks_per_day(ua) > ticks_per_day(ub):
        lit = b.value * factor(ub, ua)
        if not fits64(lit):
            return _out_of_range(op, a, lit > 0)
    if isinstance(b, E.Lit) and not isinstance(a, E.Lit) and b.value is not None and ua != ub \
            and ticks_per_day(ub) > ticks_per_day(ua):
        # a literal finer than the column: round it onto the column's unit (a fused-scan term on the
        # column's own bytes) when the comparison allows, else scale the column
        rounded = _round_literal(op, b.value, factor(ua, ub))
        if rounded is not None and fits64(rounded[1]):
            return E.Call(rounded[0], [a, E.Lit(rounded[1], E.I64, a.logical)], E.U8)
    u = finer(ua, ub)
    return E.Call(op, [at_unit(a, u), at_unit(b, u)], E.U8)


def unify(a, b):
    """CASE branches / COALESCE: both at the finer unit."""
    ua, ub = unit_of_expr(a), unit_of_expr(b)
    if ua is None or ub is None:
        E = _E()
        if isinstance(a, E.Lit) and a.value is None and ub is not None:
            return E.Lit(None, E.I64, b.logical), b
        if isinstance(b, E.Lit) and b.value is None and ua is not None:
            return a, E.Lit(None, E.I64, a.logical)
        raise NotImplementedError("a DATE / TIMESTAMP and a number cannot be branches of one CASE")
    u = finer(ua, ub)
    return at_unit(a, u), at_unit(b, u)


def datepart_expr(x, field: str):
    E = _E()
    u = unit_of_expr(x)
    if field == "DAYS":
        if u == "D":
            return x
        return E.Call("datepart", [x], E.I64, DATE_LOGICAL, (FIELD["DAYS"], TPS[u]))
    return E.Call("datepart", [x], E.I64, "int64", (FIELD[field], TPS[u]))


def rewrite_cmp(op: str, a, b):
    """YEAR(x) <op> literal and CAST(x AS DATE) <op> literal (op not <>) as one or two `x <cmp> literal`
    conjuncts on x's own unit: both functions are monotone, and the plain comparisons stay fused-scan
    terms (and prune Parquet row groups).  None when the shape does not apply."""
    E = _E()
    if op == "ne":
        return None
    if not (isinstance(a, E.Call) and a.op == "datepart"):
        if isinstance(b, E.Call) and b.op == "datepart" and isinstance(a, (E.Lit, TScalar, int, str)):
            return rewrite_cmp(_FLIP[op], b, a)
        return None
    field = FIELDS[a.param[0]]
    if field not in ("YEAR", "DAYS"):
        return None
    (x,) = a.args
    u = unit_of_expr(x)
    if field == "YEAR":
        v = b.value if isinstance(b, E.Lit) else b
        if isinstance(v, float) and v.is_integer():
            v = int(v)
        if not isinstance(v, int) or isinstance(v, bool) or (isinstance(b, E.Lit) and b.logical != "int64") \
                or abs(v) > 300000:
            return None
        lo = days_from_civil(v, 1, 1) * ticks_per_day(u)
        hi = days_from_civil(v + 1, 1, 1) * ticks_per_day(u)
    else:
        if isinstance(b, (str, TScalar)):
            b = _operand(b, like=a)
        if not isinstance(b, E.Lit) or b.value is None or unit_of_expr(b) is None:
            return None
        days = b.value if b.logical == DATE_LOGICAL else None
        if days is None:                          # CAST(x AS DATE) vs a TIMESTAMP literal: leave it
            return None
        lo, hi = days * ticks_per_day(u), (days + 1) * ticks_per_day(u)
    if not (fits64(lo) and fits64(hi)):
        return None
    L = lambda v: E.Lit(v, E.I64, x.logical)  # noqa: E731
    if op == "lt":
        return E.Call("lt", [x, L(lo)], E.U8)
    if op == "le":
        return E.Call("lt", [x, L(hi)], E.U8)
    if op == "gt":
        return E.Call("ge", [x, L(hi)], E.U8)
    if op == "ge":
        return E.Call("ge", [x, L(lo)], E.U8)
    return E.Call("and", [E.Call("ge", [x, L(lo)], E.U8), E.Call("lt", [x, L(hi)], E.U8)], E.U8)


def _add_ticks(x, n, unit: str):
    """x (promoted to `unit`) + n ticks of `unit`; n an int or an int64 expression."""
    E = _E()
    x = at_unit(x, unit)
    return E.Call("add", [x, n if isinstance(n, E.Expr) else E.Lit(int(n))], E.I64, logical_of(unit))


def add_months_expr(x, n, to_last=False):
    E = _E()
    n = n if isinstance(n, E.Expr) else E.Lit(int(n))
    return E.Call("addmonths", [x, E.cast(n, E.I64)], E.I64, x.logical, (1 if to_last else 0, TPS[unit_of_expr(x)]))


def add_interval(x, iv: Interval, sign: int):
    """DATE / TIMESTAMP expression +- INTERVAL: calendar months first, then the fixed ticks."""
    months, ns = sign * iv.months, sign * iv.ns
    if months:
        x = add_months_expr(x, months)
    if ns:
        ru = interval_result_unit(unit_of_expr(x), ns)
        x = _add_ticks(x, ns_to_ticks(ns, ru), ru)
    return x


def binop(op: str, a, b):
    """Any binary operator with a DATE / TIMESTAMP / INTERVAL operand."""
    E = _E()
    if op in _FLIP:
        return compare(op, a, b)
    if op in ("add", "sub"):
        if isinstance(b, Interval) and unit_of_expr(a) is not None:
            if isinstance(a, TScalar):
                return E.Lit(add_interval_scalar(a, b, 1 if op == "add" else -1))
            return add_interval(a, b, 1 if op == "add" else -1)
        if op == "add" and isinstance(a, Interval) and unit_of_expr(b) is not None:
            return binop("add", b, a)
        if op == "sub" and unit_of_expr(a) is not None and unit_of_expr(b) is not None:
            raise NotImplementedError("the difference of two dates / timestamps is an interval, which is not a "
                                      "column type here; use TIMESTAMPDIFF(unit, a, b)")
    raise NotImplementedError(f"operator {op} on DATE / TIMESTAMP operands (only +/- INTERVAL and comparisons)")


def timestampadd(unit: str, n, x):
    E = _E()
    unit = norm_unit(unit)
    months, ns = _UNIT_SIZE[unit]
    if months:
        n = E.binop("mul", n, months) if months != 1 else n
        return add_months_expr(x, n)
    ru = interval_result_unit(unit_of_expr(x), ns)
    k = ns_to_ticks(ns, ru)
    return _add_ticks(x, E.binop("mul", n, k) if k != 1 else E.cast(E.as_expr(n), E.I64), ru)


def timestampdiff(unit: str, a, b):
    """whole `unit`s from a to b, truncated toward zero; MONTH / QUARTER / YEAR from the whole days:
    trunc(12 days / 365), trunc(4 days / 365), trunc(days / 365)."""
    E = _E()
    unit = norm_unit(unit)
    a, b = unify(_operand(a, like=b if unit_of_expr(b) else None), _operand(b, like=a))
    u = unit_of_expr(a)
    d = E.Call("sub", [b, a], E.I64)
    months, ns = _UNIT_SIZE[unit]
    if months:
        days = E.binop("divt", d, ticks_per_day(u)) if u != "D" else d
        num = {12: 1, 3: 4, 1: 12}[months]
        return E.binop("divt", E.binop("mul", days, num) if num != 1 else days, 365)
    tick_ns = NS_PER_DAY // ticks_per_day(u)
    if ns >= tick_ns:
        return E.binop("divt", d, ns // tick_ns)
    return E.binop("mul", d, tick_ns // ns)


_FLOOR_UNITS = ("DAY", "HOUR", "MINUTE", "SECOND", "MILLISECOND", "MICROSECOND")


def floor_ceil(x, unit: str, ceil: bool):
    """FLOOR / CEIL(x TO unit) for DAY .. MICROSECOND, from the floored MOD_I."""
    E = _E()
    unit = norm_unit(unit)
    if unit not in _FLOOR_UNITS:
        raise NotImplementedError(f"{'CEIL' if ceil else 'FLOOR'}(... TO {unit}): only DAY down to MICROSECOND")
    u = unit_of_expr(x)
    ns = _UNIT_SIZE[unit][1]
    k = ns * ticks_per_day(u) // NS_PER_DAY
    if k <= 1:
        return x
    if ceil:      # x + ((-x) mod k)
        return E.Call("add", [x, E.Call("mod", [E.Call("neg", [x], E.I64), E.Lit(k)], E.I64)], E.I64, x.logical)
    return E.Call("sub", [x, E.Call("mod", [x, E.Lit(k)], E.I64)], E.I64, x.logical)


_EXTRACT = {"YEAR": "YEAR", "QUARTER": "QUARTER", "MONTH": "MONTH", "WEEK": "ISOWEEK", "DAY": "DAY",
            "DOW": "DOW", "DOY": "DOY", "HOUR": "HOUR", "MINUTE": "MINUTE", "SECOND": "SECOND",
            "MILLISECOND": "MILLISECOND", "MICROSECOND": "MICROSECOND", "DATE": "DAYS"}
_EXTRACT_ALIAS = {"MILLENIUM": "MILLENNIUM", "MILLENIUMS": "MILLENNIUM", "MILLENNIUMS": "MILLENNIUM",
                  "CENTURIES": "CENTURY", "DECADES": "DECADE", "ISOWEEK": "WEEK"}
_BY_YEAR = {"DECADE": 10, "CENTURY": 100, "MILLENNIUM": 1000}


def extract_field(name: str) -> str:
    f = str(name).upper()
    f = _EXTRACT_ALIAS.get(f, f)
    if f not in _EXTRACT and f not in _BY_YEAR:
        try:
            f = norm_unit(f)
        except ValueError:
            raise NotImplementedError(f"EXTRACT({name} FROM ...)") from None
        if f not in _EXTRACT:
            raise NotImplementedError(f"EXTRACT({name} FROM ...)")
    return f


def extract(field: str, x):
    """EXTRACT(field FROM x); DECADE / CENTURY / MILLENNIUM are trunc(year / 10^k)."""
    E = _E()
    f = extract_field(field)
    if f in _BY_YEAR:
        return E.binop("divt", datepart_expr(x, "YEAR"), _BY_YEAR[f])
    return datepart_expr(x, _EXTRACT[f])


def cast_to(x, unit: str):
    """CAST(x AS DATE) (unit "D") / CAST(x AS TIMESTAMP) (the operand's unit, us for a DATE)."""
    if isinstance(x, str):
        return _E().Lit(parse_date(x) if unit == "D" else parse_timestamp(x))
    u = unit_of_expr(x)
    if u is None:
        raise NotImplementedError(f"CAST of {getattr(x, 'logical', type(x).__name__)} to DATE / TIMESTAMP")
    if unit == "D":
        return datepart_expr(x, "DAYS")
    return at_unit(x, DEFAULT_UNIT) if u == "D" else x


def fold(e):
    """Constant expression tree -> TScalar / int / None, with the device's integer semantics (host
    constant folding of the builders above)."""
    E = _E()
    if isinstance(e, E.Lit):
        if e.value is None:
            return None
        u = unit_of(e.logical)
        return TScalar(e.value, u) if u else e.value
    vals = [fold(a) for a in e.args]
    raw = [v.ticks if isinstance(v, TScalar) else v for v in vals]
    if any(v is None for v in raw):
        return None
    op = e.op
    if op == "datepart":
        field, _ = e.param
        r = datepart(raw[0], FIELDS[field], unit_of_expr(vals[0]))
    elif op == "addmonths":
        r = add_months(raw[0], raw[1], unit_of_expr(vals[0]), bool(e.param[0]))
    elif op == "add":
        r = wrap64(raw[0] + raw[1])
    elif op == "sub":
        r = wrap64(raw[0] - raw[1])
    elif op == "mul":
        r = wrap64(raw[0] * raw[1])
    elif op == "neg":
        r = wrap64(-raw[0])
    elif op == "divt":
        if raw[1] == 0:
            return None
        q = abs(raw[0]) // abs(raw[1])
        r = wrap64(q if (raw[0] < 0) == (raw[1] < 0) else -q)
    elif op == "mod":
        if raw[1] == 0:
            return None
        r = raw[0] % raw[1]
    elif op == "cast":
        r = raw[0]
    else:
        raise NotImplementedError(f"folding {op}")
    u = unit_of(e.logical)
    return TScalar(r, u) if u else r
