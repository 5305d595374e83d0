"""The window reference (tests/window_ref.py) against sqlite3's window functions on seeded tables with ties, NULLs
in keys and values, one-row partitions and frames wider than their partition, and against the reference's known
answers (tests/golden/reference_window.py).  ROW_NUMBER among peers, and FIRST_VALUE / LAST_VALUE under tied
ORDER BY keys, are compared as multisets per peer group: SQL leaves their order open."""
import math
import sqlite3
from collections import Counter

import numpy as np
import pandas as pd
import pytest

from tests import query_ref as Q
from tests import window_ref as W
from tests.golden import reference_window as GW

INF = float("inf")
FRAMES = ["ROWS BETWEEN 2 PRECEDING AND CURRENT ROW", "ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING",
          "ROWS BETWEEN 2 PRECEDING AND UNBOUNDED FOLLOWING", "ROWS BETWEEN CURRENT ROW AND 3 FOLLOWING",
          "ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING", "ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW",
          "ROWS BETWEEN UNBOUNDED PRECEDING AND 3 FOLLOWING",
          "ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING", "ROWS BETWEEN 3 FOLLOWING AND 3 FOLLOWING",
          "ROWS BETWEEN 3 PRECEDING AND 1 PRECEDING", "ROWS BETWEEN 10 PRECEDING AND 10 FOLLOWING",
          "RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW", "RANGE BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING",
          "RANGE BETWEEN CURRENT ROW AND CURRENT ROW"]


def _frame(text):
    words = text.split()
    unit = words[0] == "RANGE"

    def bound(ws):
        if ws[0] == "UNBOUNDED":
            return -INF if ws[1] == "PRECEDING" else INF
        if ws[0] == "CURRENT":
            return 0
        return -int(ws[0]) if ws[1] == "PRECEDING" else int(ws[0])
    lo, hi = " ".join(words[2:]).split(" AND ")
    return (unit, bound(lo.split()), bound(hi.split()))


def _table(seed, n=60):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 6, n).astype(float)
    k[rng.random(n) < 0.15] = np.nan
    k[-1] = 99.0                                                 # a one-row partition
    t = rng.integers(0, 8, n)                                    # ties
    v = pd.array(rng.integers(-20, 20, n), dtype="Int64")
    v[rng.random(n) < 0.15] = pd.NA
    return pd.DataFrame({"k": k, "t": t, "v": v, "u": np.arange(n)})


def _sqlite(df, sql):
    con = sqlite3.connect(":memory:")
    df.astype(object).where(df.notna(), None).to_sql("w", con, index=False)
    return [r[0] for r in con.execute(sql).fetchall()]


pytestmark = pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 28), reason="sqlite3 without EXCLUDE-era windows")


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("fn", ["SUM", "COUNT", "MIN", "MAX", "AVG"])
@pytest.mark.parametrize("frame", FRAMES)
def test_aggregates_match_sqlite(seed, fn, frame):
    df = _table(seed)
    rel = Q.table(df)
    # sqlite sorts NULLs first ascending: state the engine's NULLS LAST for the partition key
    got = _sqlite(df, f"SELECT {fn}(v) OVER (PARTITION BY k ORDER BY t {frame}) FROM w ORDER BY u")
    kind, exp = W.window(rel, ["k"], [("t", True, False)], fn, "v", _frame(frame))
    for g, e in zip(got, exp):
        if kind == "bounded":
            assert (g is None and math.isnan(e[0])) or abs(g - e[0]) <= e[1] + 1e-12
        else:
            assert g == e


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ranks_match_sqlite(seed):
    df = _table(seed)
    rel = Q.table(df)
    for fn in ("RANK", "DENSE_RANK"):
        got = _sqlite(df, f"SELECT {fn}() OVER (PARTITION BY k ORDER BY t DESC) FROM w ORDER BY u")
        assert got == W.window(rel, ["k"], [("t", False, True)], fn, None, None)[1]
    # ROW_NUMBER among peers: the numbers of each peer group as a multiset
    got = _sqlite(df, "SELECT ROW_NUMBER() OVER (PARTITION BY k ORDER BY t) FROM w ORDER BY u")
    exp = W.window(rel, ["k"], [("t", True, False)], "ROW_NUMBER", None, None)[1]
    groups = list(zip(df["k"].fillna(-1), df["t"]))
    for g in set(groups):
        rows = [i for i, x in enumerate(groups) if x == g]
        assert Counter(got[i] for i in rows) == Counter(exp[i] for i in rows)


@pytest.mark.parametrize("fn", ["FIRST_VALUE", "LAST_VALUE"])
@pytest.mark.parametrize("frame", FRAMES)
def test_first_last_value_match_sqlite_per_peer_group(fn, frame):
    df = _table(3)
    rel = Q.table(df)
    # a unique second key pins the order, so the values are determined
    got = _sqlite(df, f"SELECT {fn}(v) OVER (PARTITION BY k ORDER BY t, u {frame}) FROM w ORDER BY u")
    exp = W.window(rel, ["k"], [("t", True, False), ("u", True, False)], fn, "v", _frame(frame))[1]
    assert got == exp


def test_int64_sum_wraps():
    big = (1 << 63) - 1
    rel = Q.table(pd.DataFrame({"x": np.array([big, 1, 1], np.int64), "u": [0, 1, 2]}))
    assert W.window(rel, [], [("u", True, False)], "SUM", "x", (True, -INF, 0))[1] == [big, -(1 << 63), -(1 << 63) + 1]


def test_nan_and_null_keys_share_a_partition_and_signed_zeros_are_peers():
    df = pd.DataFrame({"k": [np.nan, 1.0, np.nan, -0.0, 0.0], "u": [0, 1, 2, 3, 4]})
    rel = Q.table(df)
    assert W.window(rel, ["k"], [], "COUNT", None, (False, -INF, INF))[1] == [2, 1, 2, 2, 2]
    assert W.window(rel, [], [("k", True, False)], "RANK", None, None)[1] == [4, 3, 4, 1, 1]


# the reference's answers restated as window_ref calls: (function, argument, partition, order, frame)
_GOLDEN = {
    "over_with_partitioning": {"R": ("ROW_NUMBER", None, ["c"], [], None)},
    "over_with_grouping_and_sort": {"R": ("ROW_NUMBER", None, ["user_id"], [("b", True, False)], None)},
    "over_with_different": {"R1": ("ROW_NUMBER", None, ["user_id"], [("b", True, False)], None),
                            "R2": ("ROW_NUMBER", None, [], [("user_id", True, False), ("b", True, False)], None)},
    "over_calls": {"O1": ("ROW_NUMBER", None, ["user_id"], [("b", True, False)], None),
                   "O5": ("SUM", "user_id", ["user_id"], [("b", True, False)], (True, -INF, 0)),
                   "O7": ("COUNT", None, ["user_id"], [("b", True, False)], (True, -INF, 0)),
                   "O7b": ("COUNT", "b", ["user_id"], [("b", True, False)], (True, -INF, 0)),
                   "O8": ("MAX", "b", ["user_id"], [("b", True, False)], (True, -INF, 0)),
                   "O9": ("MIN", "b", ["user_id"], [("b", True, False)], (True, -INF, 0))},
    "over_with_windows": {f"O{i}": ("SUM", "a", [], [("a", True, False)], _frame(FRAMES[i - 1])) for i in range(1, 9)},
}
_GOLDEN["over_with_windows"].update({"O9": ("SUM", "a", [], [("a", True, False)], (False, 3, 3)),
                                     "O9a": ("COUNT", "a", [], [("a", True, False)], (False, 3, 3)),
                                     "O10": ("SUM", "a", [], [("a", True, False)], (False, -3, -1))})


@pytest.mark.parametrize("case", list(GW.CASES))
def test_reference_known_answers(case):
    table, rows, sql, expected = GW.CASES[case]
    rel = Q.table(pd.DataFrame(rows))
    for name, (fn, arg, part, order, frame) in _GOLDEN[case].items():
        assert W.window(rel, part, order, fn, arg, frame)[1] == expected[name], f"{case} {name}"
