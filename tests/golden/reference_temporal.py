"""Golden vectors for DATE / TIMESTAMP, TRANSCRIBED from the reference's known-answer tests
(dask-contrib/dask-sql @ f186de3, tests/integration/).  Inputs and expected outputs are the literals its
maintainers wrote down; every case cites file:line.  tests/test_sql_temporal_gpu.py runs every case
through Context.sql() on the GPU.

A case is {"where", "tables": {name: {column: (values, dtype)}}, "sql", "expected": {column: [values]}}.
Timestamps are ISO strings; an expected timestamp compares equal as a pandas Timestamp.  "raises" names
the exception a case expects instead of a result.  "note" records where a case departs from the reference
text and why (DESIGN §6 lists the divergences).
"""

_D = "2021-10-03 15:53:42.000047"          # test_rex.py:738: datetime(2021, 10, 3, 15, 53, 42, 47)

CASES = [
    {"where": "test_rex.py:114-128 (test_date_interval_math)",
     "tables": {"one": {"k": ([0], "int64")}},
     "sql": """SELECT DATE '1998-08-18' - INTERVAL '4 days' AS "before",
                      DATE '1998-08-18' + INTERVAL '4 days' AS "after" FROM one""",
     "expected": {"before": ["1998-08-14"], "after": ["1998-08-22"]},
     "note": "the reference's statement has no FROM; here it reads a one-row table (a FROM-less SELECT is "
             "outside this layer's planner)"},
    {"where": "test_rex.py:737-834 (test_date_functions)",
     "tables": {"df": {"d": ([_D], "datetime64[us]")}},
     "sql": """SELECT EXTRACT(CENTURY FROM d) AS "century", EXTRACT(DAY FROM d) AS "day",
        EXTRACT(DECADE FROM d) AS "decade", EXTRACT(DOW FROM d) AS "dow", EXTRACT(DOY FROM d) AS "doy",
        EXTRACT(HOUR FROM d) AS "hour", EXTRACT(MICROSECONDS FROM d) AS "microsecond",
        EXTRACT(MILLENNIUM FROM d) AS "millennium", EXTRACT(MILLISECONDS FROM d) AS "millisecond",
        EXTRACT(MINUTE FROM d) AS "minute", EXTRACT(MONTH FROM d) AS "month", EXTRACT(QUARTER FROM d) AS "quarter",
        EXTRACT(SECOND FROM d) AS "second", EXTRACT(WEEK FROM d) AS "week", EXTRACT(YEAR FROM d) AS "year",
        EXTRACT(DATE FROM d) AS "date", LAST_DAY(d) as "last_day",
        TIMESTAMPADD(YEAR, 1, d) as "plus_1_year", TIMESTAMPADD(MONTH, 1, d) as "plus_1_month",
        TIMESTAMPADD(WEEK, 1, d) as "plus_1_week", TIMESTAMPADD(DAY, 1, d) as "plus_1_day",
        TIMESTAMPADD(HOUR, 1, d) as "plus_1_hour", TIMESTAMPADD(MINUTE, 1, d) as "plus_1_min",
        TIMESTAMPADD(SECOND, 1, d) as "plus_1_sec", TIMESTAMPADD(MICROSECOND, 999*1000, d) as "plus_999_millisec",
        TIMESTAMPADD(MICROSECOND, 999, d) as "plus_999_microsec", TIMESTAMPADD(QUARTER, 1, d) as "plus_1_qt",
        CEIL(d TO DAY) as ceil_to_day, CEIL(d TO HOUR) as ceil_to_hour, CEIL(d TO MINUTE) as ceil_to_minute,
        CEIL(d TO SECOND) as ceil_to_seconds, CEIL(d TO MILLISECOND) as ceil_to_millisec,
        FLOOR(d TO DAY) as floor_to_day, FLOOR(d TO HOUR) as floor_to_hour, FLOOR(d TO MINUTE) as floor_to_minute,
        FLOOR(d TO SECOND) as floor_to_seconds, FLOOR(d TO MILLISECOND) as floor_to_millisec
        FROM df""",
     "expected": {
         "century": [20], "day": [3], "decade": [202], "dow": [0], "doy": [276], "hour": [15], "microsecond": [47],
         "millennium": [2], "millisecond": [0], "minute": [53], "month": [10], "quarter": [4], "second": [42],
         "week": [39], "year": [2021], "date": ["2021-10-03"], "last_day": ["2021-10-31 15:53:42.000047"],
         "plus_1_year": ["2022-10-03 15:53:42.000047"], "plus_1_month": ["2021-11-03 15:53:42.000047"],
         "plus_1_week": ["2021-10-10 15:53:42.000047"], "plus_1_day": ["2021-10-04 15:53:42.000047"],
         "plus_1_hour": ["2021-10-03 16:53:42.000047"], "plus_1_min": ["2021-10-03 15:54:42.000047"],
         "plus_1_sec": ["2021-10-03 15:53:43.000047"], "plus_999_millisec": ["2021-10-03 15:53:42.999047"],
         "plus_999_microsec": ["2021-10-03 15:53:42.001046"], "plus_1_qt": ["2022-01-03 15:53:42.000047"],
         "ceil_to_day": ["2021-10-04"], "ceil_to_hour": ["2021-10-03 16:00:00"],
         "ceil_to_minute": ["2021-10-03 15:54:00"], "ceil_to_seconds": ["2021-10-03 15:53:43"],
         "ceil_to_millisec": ["2021-10-03 15:53:42.001"], "floor_to_day": ["2021-10-03"],
         "floor_to_hour": ["2021-10-03 15:00:00"], "floor_to_minute": ["2021-10-03 15:53:00"],
         "floor_to_seconds": ["2021-10-03 15:53:42"], "floor_to_millisec": ["2021-10-03 15:53:42"]},
     "note": "millisecond: the reference expects 47000 (1000 * microsecond, test_rex.py:802); here EXTRACT"
             "(MILLISECOND) is the millisecond within the second, 0 -- a recorded divergence (DESIGN §6)"},
    {"where": "test_rex.py:836-845 (test_date_functions, FLOOR TO YEAR)",
     "tables": {"df": {"d": ([_D], "datetime64[us]")}},
     "sql": "SELECT FLOOR(d TO YEAR) as floor_to_year FROM df",
     "raises": "NotImplementedError"},
    {"where": "test_rex.py:847-886 (test_timestampdiff, literal row)",
     "tables": {"df": {"ts_literal1": (["2002-03-07 09:10:05.000123"], "datetime64[us]"),
                       "ts_literal2": (["2001-06-05 10:11:06.000234"], "datetime64[us]")}},
     "sql": """SELECT timestampdiff(NANOSECOND, ts_literal1, ts_literal2) as res0,
        timestampdiff(MICROSECOND, ts_literal1, ts_literal2) as res1,
        timestampdiff(SECOND, ts_literal1, ts_literal2) as res2, timestampdiff(MINUTE, ts_literal1, ts_literal2) as res3,
        timestampdiff(HOUR, ts_literal1, ts_literal2) as res4, timestampdiff(DAY, ts_literal1, ts_literal2) as res5,
        timestampdiff(WEEK, ts_literal1, ts_literal2) as res6, timestampdiff(MONTH, ts_literal1, ts_literal2) as res7,
        timestampdiff(QUARTER, ts_literal1, ts_literal2) as res8, timestampdiff(YEAR, ts_literal1, ts_literal2) as res9
        FROM df""",
     "expected": {"res0": [-23756338999889000], "res1": [-23756338999889], "res2": [-23756338], "res3": [-395938],
                  "res4": [-6598], "res5": [-274], "res6": [-39], "res7": [-9], "res8": [-3], "res9": [0]}},
    {"where": "test_rex.py:888-938 (test_timestampdiff, three rows)",
     "tables": {"test": {
         "a": (["2002-06-05 02:01:05.000200", "2002-09-01", "1970-12-03"], "datetime64[ns]"),
         "b": (["2002-06-07 01:00:02.000100", "2003-06-05", "2038-06-05"], "datetime64[ns]")}},
     "sql": ("SELECT timestampdiff(NANOSECOND, a, b) as nanoseconds, timestampdiff(MICROSECOND, a, b) as microseconds,"
             "timestampdiff(SECOND, a, b) as seconds, timestampdiff(MINUTE, a, b) as minutes,"
             "timestampdiff(HOUR, a, b) as hours, timestampdiff(DAY, a, b) as days,"
             "timestampdiff(WEEK, a, b) as weeks, timestampdiff(MONTH, a, b) as months,"
             "timestampdiff(QUARTER, a, b) as quarters, timestampdiff(YEAR, a, b) as years FROM test"),
     "expected": {"nanoseconds": [169136999900000, 23932800000000000, 2130278400000000000],
                  "microseconds": [169136999900, 23932800000000, 2130278400000000],
                  "seconds": [169136, 23932800, 2130278400], "minutes": [2818, 398880, 35504640],
                  "hours": [46, 6648, 591744], "days": [1, 277, 24656], "weeks": [0, 39, 3522],
                  "months": [0, 9, 810], "quarters": [0, 3, 270], "years": [0, 0, 67]}},
]

_T3 = {"df": {"a": ([1, 2, 3], "int64"), "b": ([4, 5, 6], "int64"),
              "t": (["2021-01-01", "2022-02-02", "2023-03-03"], "datetime64[us]")}}     # test_rex.py:1058-1064
CASES += [
    {"where": "test_rex.py:1066-1070 (test_extract_date)", "tables": _T3,
     "sql": "SELECT EXTRACT(DATE FROM t) AS e FROM df",
     "expected": {"e": ["2021-01-01", "2022-02-02", "2023-03-03"]}},
    {"where": "test_rex.py:1072-1081 (test_extract_date)", "tables": _T3,
     "sql": "SELECT * FROM df WHERE EXTRACT(DATE FROM t) > '2021-02-01'",
     "expected": {"a": [2, 3], "b": [5, 6], "t": ["2022-02-02", "2023-03-03"]}},
    {"where": "test_rex.py:1082-1088 (test_extract_date)", "tables": _T3,
     "sql": "SELECT * FROM df WHERE EXTRACT(DATE FROM t) BETWEEN '2020-10-01' AND '2022-10-10'",
     "expected": {"a": [1, 2], "b": [4, 5], "t": ["2021-01-01", "2022-02-02"]}},
    {"where": "test_rex.py:1090-1094 (test_extract_date)", "tables": _T3,
     "sql": "SELECT TIMESTAMPADD(YEAR, 1, EXTRACT(DATE FROM t)) AS ta FROM df",
     "expected": {"ta": ["2022-01-01", "2023-02-02", "2024-03-03"]}},
    {"where": "test_rex.py:1096-1100 (test_extract_date)", "tables": _T3,
     "sql": "SELECT EXTRACT(DATE FROM t) + INTERVAL '2 days' AS i FROM df",
     "expected": {"i": ["2021-01-03", "2022-02-04", "2023-03-05"]}},
]

# fixtures.py:105-118 datetime_table: 2014-08-01 09:00, every 8 hours, 6 rows.  Only its `no_timezone` column:
# time-zone-aware columns are outside this layer (they raise NotImplementedError at create_table).
_NO_TZ = ["2014-08-01 09:00", "2014-08-01 17:00", "2014-08-02 01:00", "2014-08-02 09:00", "2014-08-02 17:00",
          "2014-08-03 01:00"]
CASES += [
    {"where": "test_filter.py:86-98 (test_filter_cast_date, no_timezone column)",
     "tables": {"datetime_table": {"no_timezone": (_NO_TZ, "datetime64[ns]")}},
     "sql": "SELECT * FROM datetime_table WHERE CAST(no_timezone AS DATE) > DATE '2014-08-01'",
     "expected": {"no_timezone": _NO_TZ[2:]},
     "note": "the reference filters the time-zone-aware `timezone` column; the same rule on `no_timezone`"},
    {"where": "test_filter.py:130-139 (test_filter_year)",
     "tables": {"datetime_test": {"year": ([2015, 2016], "int64"), "month": ([2, 3], "int64"),
                                  "day": ([4, 5], "int64"),
                                  "dt": (["2015-02-04", "2016-03-05"], "datetime64[ns]")}},
     "sql": "select * from datetime_test where year(dt) < 2016",
     "expected": {"year": [2015], "month": [2], "day": [4], "dt": ["2015-02-04"]}},
    {"where": "test_select.py:155-178 (test_date_casting, no_timezone column)",
     "tables": {"datetime_table": {"no_timezone": (_NO_TZ, "datetime64[ns]")}},
     "sql": "SELECT CAST(no_timezone AS DATE) AS no_timezone FROM datetime_table",
     "expected": {"no_timezone": ["2014-08-01", "2014-08-01", "2014-08-02", "2014-08-02", "2014-08-02",
                                  "2014-08-03"]},
     "note": "time-zone-aware columns of the fixture are out of scope; a DATE comes back as datetime64[s], "
             "the reference's as datetime64[ns] (both midnight)"},
]
