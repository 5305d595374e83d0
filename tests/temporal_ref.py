"""Exact NumPy reference of the calendar opcodes (B2_OP_DATEPART, B2_OP_ADDMONTHS) on int64 ticks.

No GPU and no package import: test_temporal_ref_cpu.py checks it against pandas / datetime, and the GPU
tests compare the kernels with it bit for bit.  NumPy's `//` and `%` floor, like the kernels' split of a
tick count into (day, time of day)."""
import numpy as np

TPS = {"D": 0, "s": 1, "ms": 10 ** 3, "us": 10 ** 6, "ns": 10 ** 9}
FIELDS = ("DAYS", "YEAR", "QUARTER", "MONTH", "DAY", "DOY", "DOW", "ISOWEEK", "HOUR", "MINUTE", "SECOND",
          "MILLISECOND", "MICROSECOND")


def tpd(unit):
    return 1 if unit == "D" else TPS[unit] * 86400


def civil_from_days(z):
    z = np.asarray(z, dtype=np.int64) + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    return yoe + era * 400 + (m <= 2), m, d


def days_from_civil(y, m, d):
    y = np.asarray(y, dtype=np.int64) - (np.asarray(m) <= 2)
    m = np.asarray(m, dtype=np.int64)
    era = y // 400
    yoe = y - era * 400
    doy = (153 * np.where(m > 2, m - 3, m + 9) + 2) // 5 + np.asarray(d, dtype=np.int64) - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def month_days(y, m):
    nxt_y = y + (m == 12)
    nxt_m = np.where(m == 12, 1, m + 1)
    return days_from_civil(nxt_y, nxt_m, 1) - days_from_civil(y, m, 1)


def datepart(ticks, field, unit):
    x = np.asarray(ticks, dtype=np.int64)
    per_day, tps = tpd(unit), TPS[unit]
    day, tod = x // per_day, x % per_day
    if field == "DAYS":
        return day
    if field == "DOW":
        return (day + 4) % 7
    if FIELDS.index(field) >= FIELDS.index("HOUR"):
        if not tps:
            return np.zeros_like(x)
        sub = tod % tps
        return {"HOUR": lambda: tod // (tps * 3600), "MINUTE": lambda: tod // (tps * 60) % 60,
                "SECOND": lambda: tod // tps % 60, "MILLISECOND": lambda: sub * 1000 // tps,
                "MICROSECOND": lambda: sub * 1000000 // tps}[field]()
    if field == "ISOWEEK":
        th = day - (day + 3) % 7 + 3
        y, _, _ = civil_from_days(th)
        return (th - days_from_civil(y, 1, 1)) // 7 + 1
    y, m, d = civil_from_days(day)
    if field == "YEAR":
        return y
    if field == "QUARTER":
        return (m - 1) // 3 + 1
    if field == "MONTH":
        return m
    if field == "DAY":
        return d
    return day - days_from_civil(y, 1, 1) + 1      # DOY


def add_months(ticks, n, unit, to_last=False):
    x = np.asarray(ticks, dtype=np.int64)
    n = np.asarray(n, dtype=np.int64)
    per_day = tpd(unit)
    day, tod = x // per_day, x % per_day
    y, m, d = civil_from_days(day)
    total = y * 12 + (m - 1) + n
    y2 = total // 12
    m2 = total - y2 * 12 + 1
    last = month_days(y2, m2)
    d2 = last if to_last else np.minimum(d, last)
    with np.errstate(over="ignore"):
        return (days_from_civil(y2, m2, d2).astype(np.uint64) * np.uint64(per_day) + tod.astype(np.uint64)).astype(np.int64)
