"""The calendar reference (tests/temporal_ref.py) against pandas .dt / DateOffset / isocalendar(),
datetime.date and numpy datetime64[D] arithmetic.  CPU only."""
import datetime

import numpy as np
import pandas as pd
import pytest

from tests import temporal_ref as R


def _days(lo, hi):
    return np.arange(np.datetime64(lo, "D").astype(np.int64), np.datetime64(hi, "D").astype(np.int64) + 1)


def test_every_day_1600_to_2400_matches_pandas():
    days = _days("1600-01-01", "2400-12-31")
    ts = pd.Series(days.astype("datetime64[D]").astype("datetime64[s]"))
    y, m, d = R.civil_from_days(days)
    np.testing.assert_array_equal(y, ts.dt.year)
    np.testing.assert_array_equal(m, ts.dt.month)
    np.testing.assert_array_equal(d, ts.dt.day)
    np.testing.assert_array_equal(R.days_from_civil(y, m, d), days)
    np.testing.assert_array_equal(R.datepart(days, "DOY", "D"), ts.dt.dayofyear)
    np.testing.assert_array_equal(R.datepart(days, "QUARTER", "D"), ts.dt.quarter)
    np.testing.assert_array_equal(R.datepart(days, "DOW", "D"), (ts.dt.dayofweek + 1) % 7)
    np.testing.assert_array_equal(R.datepart(days, "ISOWEEK", "D"), ts.dt.isocalendar().week.astype(np.int64))
    np.testing.assert_array_equal(R.month_days(y, m), ts.dt.days_in_month)


@pytest.mark.parametrize("n", [-25, -13, -12, -1, 0, 1, 11, 12, 13, 48])
def test_add_months_matches_dateoffset(n):
    days = _days("1899-12-01", "1901-03-31")[::3].tolist() + _days("1999-12-15", "2000-03-31").tolist()
    days = np.array(days + _days("2023-01-25", "2024-03-05")[::2].tolist())
    ts = pd.Series(days.astype("datetime64[D]").astype("datetime64[s]"))
    want = (ts + pd.DateOffset(months=n)).to_numpy().astype("datetime64[D]").astype(np.int64)
    np.testing.assert_array_equal(R.add_months(days, n, "D"), want)
    last = (ts + pd.DateOffset(months=n)) + pd.offsets.MonthEnd(0)
    np.testing.assert_array_equal(R.add_months(days, n, "D", to_last=True),
                                  last.to_numpy().astype("datetime64[D]").astype(np.int64))


def _edge_ticks(unit):
    per_s = R.TPS[unit]
    base = [0, 1, -1, per_s - 1, -per_s, 86400 * per_s - 1, -86400 * per_s, -86400 * per_s + 1]
    for s in ("1600-02-29", "1900-02-28", "2000-02-29", "2100-03-01", "2262-04-11", "1677-09-22",
              "1969-12-31", "2020-12-31", "2021-01-01"):
        t = int(np.datetime64(s, "D").astype(np.int64)) * 86400 * per_s
        base += [t, t - 1, t + 1, t + 43210 * per_s + per_s // 3]
    lim = {"s": 10 ** 11, "ms": 10 ** 14, "us": 9 * 10 ** 16, "ns": 9 * 10 ** 18}[unit]
    rng = np.random.default_rng(7)
    base = [t for t in base if -(2 ** 63) < t < 2 ** 63 - 86400 * per_s]
    ticks = np.array(base + rng.integers(-lim, lim, 5000).tolist(), dtype=np.int64)
    keep = np.abs(ticks // (86400 * per_s)) < 106751        # where pandas (ns) can check the result
    return ticks[keep]


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
def test_fields_of_every_unit_match_pandas(unit):
    ticks = _edge_ticks(unit)
    ts = pd.Series(ticks.view(f"datetime64[{unit}]"))
    dt = ts.dt
    np.testing.assert_array_equal(R.datepart(ticks, "YEAR", unit), dt.year)
    np.testing.assert_array_equal(R.datepart(ticks, "MONTH", unit), dt.month)
    np.testing.assert_array_equal(R.datepart(ticks, "DAY", unit), dt.day)
    np.testing.assert_array_equal(R.datepart(ticks, "HOUR", unit), dt.hour)
    np.testing.assert_array_equal(R.datepart(ticks, "MINUTE", unit), dt.minute)
    np.testing.assert_array_equal(R.datepart(ticks, "SECOND", unit), dt.second)
    np.testing.assert_array_equal(R.datepart(ticks, "MICROSECOND", unit), dt.microsecond)
    np.testing.assert_array_equal(R.datepart(ticks, "MILLISECOND", unit), dt.microsecond // 1000)
    np.testing.assert_array_equal(R.datepart(ticks, "DOY", unit), dt.dayofyear)
    np.testing.assert_array_equal(R.datepart(ticks, "DOW", unit), (dt.dayofweek + 1) % 7)
    np.testing.assert_array_equal(R.datepart(ticks, "ISOWEEK", unit), dt.isocalendar().week.astype(np.int64))
    np.testing.assert_array_equal(R.datepart(ticks, "DAYS", unit), ts.to_numpy().astype("datetime64[D]").astype(np.int64))
    for n in (-14, 1, 12):
        want = (ts + pd.DateOffset(months=n)).to_numpy().astype(f"datetime64[{unit}]").astype(np.int64)
        ok = np.abs(ticks // (86400 * R.TPS[unit])) < 106000
        np.testing.assert_array_equal(R.add_months(ticks, n, unit)[ok], want[ok])


def test_negative_tick_is_the_previous_day():
    assert R.datepart(np.array([-1]), "DAYS", "us")[0] == -1
    assert R.datepart(np.array([-1]), "MICROSECOND", "us")[0] == 999999
    assert R.datepart(np.array([-1]), "HOUR", "us")[0] == 23


def test_date32_extremes_against_numpy():
    days = np.array([-(2 ** 31), -(2 ** 31) + 1, 2 ** 31 - 2, 2 ** 31 - 1, -719528, 2932896], dtype=np.int64)
    y, m, d = R.civil_from_days(days)
    np.testing.assert_array_equal(R.days_from_civil(y, m, d), days)
    # numpy datetime64[D] covers these days: years through its astype to datetime64[Y]/[M]
    dd = days.astype("datetime64[D]")
    np.testing.assert_array_equal(y, dd.astype("datetime64[Y]").astype(np.int64) + 1970)
    np.testing.assert_array_equal(m, dd.astype("datetime64[M]").astype(np.int64) % 12 + 1)
    np.testing.assert_array_equal(d, (dd - dd.astype("datetime64[M]")).astype(np.int64) + 1)


def test_python_dates_round_trip():
    for s in ("0001-01-01", "1582-10-15", "1970-01-01", "9999-12-31"):
        day = datetime.date.fromisoformat(s)
        z = (day - datetime.date(1970, 1, 1)).days
        assert tuple(int(v[0]) for v in R.civil_from_days(np.array([z]))) == (day.year, day.month, day.day)
