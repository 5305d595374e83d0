"""BIT_AND / BIT_OR / BIT_XOR / EVERY and REGR_COUNT / REGR_SXX / REGR_SYY end to end through Context.sql():
the reference's test_aggregations (tests/golden/reference_aggregations.py) at 1 and 3 partitions, NULL handling, FILTER, DISTINCT, global aggregates, the fused star path, the reference's REGR identities
(tests/integration/test_groupby.py:363-422, with an integer group key), rows where only one REGR argument is
NULL, and REGR_SXX on large-mean data held to VAR's accuracy."""
from fractions import Fraction
from functools import reduce

import numpy as np
import pandas as pd
import pytest

from tests.golden import reference_aggregations as GA
from tests.golden import reference_vectors as GV
from tests.test_sql_gpu import _groups, assert_same

pytestmark = pytest.mark.gpu

MIN, MAX = -2 ** 63, 2 ** 63 - 1
POOL = np.array([MIN, -1, 0, MAX, 1, 2, 5, -6, 12, 0x5555555555555555], np.int64)


@pytest.fixture()
def c():
    from dask_sql_b200 import Context
    return Context()


@pytest.mark.parametrize("case", GA.CASES, ids=[c["name"] for c in GA.CASES])
@pytest.mark.parametrize("npartitions", [1, 3])
def test_reference_aggregations_known_answers(c, case, npartitions):
    """the reference's test_aggregations through Context.sql(), like test_reference_known_answers"""
    tables = GV.tables_of(case)
    for name, df in tables.items():
        c.create_table(name, df, npartitions=npartitions)
    assert_same(c.sql(case["sql"]).compute(), GV.expected_of(case, tables), case.get("float_cols", ()))


def _bits_frame(n=50_000, seed=1):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 12, n)
    v = pd.array(rng.choice(POOL, n), dtype="Int64")
    v[rng.random(n) < 0.1] = pd.NA
    v[k == 11] = pd.NA                                   # a group whose inputs are all NULL
    b = pd.array(rng.random(n) < 0.97, dtype="boolean")
    b[rng.random(n) < 0.05] = pd.NA
    b[k == 11] = pd.NA
    b[k == 3] = True                                     # an EVERY that holds
    return pd.DataFrame({"k": k, "v": v, "b": b})


def _fold(vals, f):
    vals = [int(x) for x in vals if not pd.isna(x)]
    return None if not vals else reduce(f, vals)


@pytest.mark.parametrize("npartitions", [1, 3])
def test_bitwise_group_by_with_nulls_filter_and_distinct(c, npartitions):
    df = _bits_frame()
    c.create_table("t", df, npartitions=npartitions)
    got = _groups(c.sql("""SELECT k, BIT_AND(v) AS a, BIT_OR(v) AS o, BIT_XOR(v) AS x, EVERY(b) AS e,
                           BIT_OR(v) FILTER (WHERE v > 0) AS fo, BIT_XOR(DISTINCT v) AS xd,
                           EVERY(v < 3) AS ev FROM t GROUP BY k""", return_futures=False), "k")
    assert set(got) == set(range(12))
    for k, r in got.items():
        g = df[df.k == k]
        vs = g.v.tolist()
        exp = {"a": _fold(vs, lambda p, q: p & q), "o": _fold(vs, lambda p, q: p | q),
               "x": _fold(vs, lambda p, q: p ^ q), "fo": _fold([x for x in vs if not pd.isna(x) and x > 0],
                                                              lambda p, q: p | q),
               "xd": _fold(pd.unique(g.v.dropna()).tolist(), lambda p, q: p ^ q),
               "e": None if g.b.isna().all() else bool(g.b.dropna().all()),
               "ev": None if g.v.isna().all() else bool((g.v.dropna() < 3).all())}
        for name, e in exp.items():
            if e is None:
                assert pd.isna(r[name]), (k, name, r[name])
            else:
                assert r[name] == e, (k, name, r[name], e)
    # XOR over the rows differs from XOR over the distinct values: the DISTINCT pass is a separate one
    assert any(got[k]["x"] != got[k]["xd"] for k in range(11))


@pytest.mark.parametrize("npartitions", [1, 3])
def test_bitwise_global_aggregates(c, npartitions):
    df = _bits_frame(seed=2)
    c.create_table("t", df, npartitions=npartitions)
    got = c.sql("SELECT BIT_AND(v) AS a, BIT_OR(v) AS o, BIT_XOR(v) AS x, EVERY(b) AS e FROM t WHERE k < 11",
                return_futures=False)
    sub = df[df.k < 11]
    vs = sub.v.tolist()
    assert int(got.a[0]) == _fold(vs, lambda p, q: p & q)
    assert int(got.o[0]) == _fold(vs, lambda p, q: p | q)
    assert int(got.x[0]) == _fold(vs, lambda p, q: p ^ q)
    assert bool(got.e[0]) == bool(sub.b.dropna().all())
    got = c.sql("SELECT BIT_AND(v) AS a, BIT_OR(v) AS o, EVERY(b) AS e FROM t WHERE k = 11", return_futures=False)
    assert len(got) == 1 and pd.isna(got.a[0]) and pd.isna(got.o[0]) and pd.isna(got.e[0])
    got = c.sql("SELECT BIT_XOR(v) AS x, EVERY(k < 5) AS e FROM t WHERE k = 4", return_futures=False)
    assert int(got.x[0]) == _fold(df[df.k == 4].v.tolist(), lambda p, q: p ^ q) and bool(got.e[0])


def test_bit_or_star_query_takes_the_fused_path(c):
    from dask_sql_b200 import executor
    rng = np.random.default_rng(4)
    nd, nf = 20_000, 400_000
    dim = pd.DataFrame({"pk": rng.permutation(nd), "flag": rng.integers(0, 10, nd), "grp": rng.integers(0, 500, nd)})
    fact = pd.DataFrame({"fk": rng.integers(0, nd, nf), "x": rng.choice(POOL, nf)})
    c.create_table("fact", fact, npartitions=4, persist=True)
    c.create_table("dim", dim, persist=True)
    before = executor.stats["star_fused"]
    got = c.sql("""SELECT d.grp, BIT_OR(f.x) AS o, BIT_AND(f.x) AS a, BIT_XOR(f.x) AS x FROM fact f
                   JOIN dim d ON f.fk = d.pk WHERE d.flag < 5 GROUP BY d.grp""", return_futures=False)
    assert executor.stats["star_fused"] == before + 1
    j = fact.merge(dim[dim.flag < 5], left_on="fk", right_on="pk")
    g = j.groupby("grp").x
    exp = pd.DataFrame({"grp": g.apply(lambda s: 0).index,
                        "o": g.apply(lambda s: np.bitwise_or.reduce(s.to_numpy())).values,
                        "a": g.apply(lambda s: np.bitwise_and.reduce(s.to_numpy())).values,
                        "x": g.apply(lambda s: np.bitwise_xor.reduce(s.to_numpy())).values})
    got = got.sort_values("grp").reset_index(drop=True)
    for col in ("grp", "o", "a", "x"):
        assert got[col].astype(np.int64).tolist() == exp[col].astype(np.int64).tolist(), col


# ---- REGR_* ----------------------------------------------------------------------------------------------
def _timeseries(n=30_000, seed=6):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, n)
    y = rng.normal(0, 1, n)
    x[rng.random(n) < 0.1] = np.nan
    y[rng.random(n) < 0.1] = np.nan
    return pd.DataFrame({"name": rng.integers(0, 26, n), "x": x, "y": y})


def test_regr_identities_of_the_reference(c):
    """tests/integration/test_groupby.py:363-422 with an integer group key"""
    c.create_table("timeseries", _timeseries(), npartitions=3)
    got = c.sql("""SELECT name, COUNT(x) FILTER (WHERE y IS NOT NULL) AS expected, REGR_COUNT(y, x) AS calculated
                   FROM timeseries GROUP BY name""", return_futures=False)
    assert got.expected.fillna(0).astype(int).tolist() == got.calculated.astype(int).tolist()
    for a in ("y", "x"):
        f = "REGR_SYY(y, x)" if a == "y" else "REGR_SXX(y, x)"
        got = c.sql(f"""SELECT name, (REGR_COUNT(y, x) * VAR_POP({a})) AS expected, {f} AS calculated
                        FROM timeseries WHERE x IS NOT NULL AND y IS NOT NULL GROUP BY name""", return_futures=False)
        np.testing.assert_allclose(got.calculated.to_numpy(), got.expected.to_numpy(), rtol=1e-9)


def test_regr_with_one_argument_null_against_numpy(c):
    df = _timeseries(seed=7)
    df.loc[df.name == 25, "y"] = np.nan                 # a group where no row has both arguments
    c.create_table("t", df, npartitions=2)
    got = _groups(c.sql("""SELECT name, REGR_COUNT(y, x) AS n, REGR_SXX(y, x) AS sxx, REGR_SYY(y, x) AS syy
                           FROM t GROUP BY name""", return_futures=False), "name")
    for k, r in got.items():
        g = df[df.name == k]
        ok = g.x.notna() & g.y.notna()
        xs, ys = g.x[ok].to_numpy(), g.y[ok].to_numpy()
        assert int(r["n"]) == ok.sum(), k
        if ok.sum() == 0:
            assert pd.isna(r["sxx"]) and pd.isna(r["syy"]), k
            continue
        np.testing.assert_allclose([r["sxx"], r["syy"]], [((xs - xs.mean()) ** 2).sum(), ((ys - ys.mean()) ** 2).sum()],
                                   rtol=1e-9, err_msg=str(k))
    assert int(got[25]["n"]) == 0
    got = c.sql("SELECT REGR_COUNT(y, x) AS n, REGR_SXX(y, x) AS s FROM t", return_futures=False)
    ok = df.x.notna() & df.y.notna()
    assert int(got.n[0]) == ok.sum()
    xs = df.x[ok].to_numpy()
    np.testing.assert_allclose(got.s[0], ((xs - xs.mean()) ** 2).sum(), rtol=1e-9)


def test_regr_sxx_on_large_mean_data_is_as_accurate_as_var(c):
    """x ~ N(1e9, 1): against the exact two-pass sum of squared deviations, at VAR's 1e-9"""
    rng = np.random.default_rng(9)
    n = 20_000
    k = rng.integers(0, 10, n)
    x = 1e9 + rng.normal(0, 1, n)
    y = rng.normal(0, 1, n)
    y[rng.random(n) < 0.1] = np.nan
    c.create_table("t", pd.DataFrame({"k": k, "x": x, "y": y}), npartitions=3)
    got = _groups(c.sql("SELECT k, REGR_SXX(y, x) AS s, REGR_COUNT(y, x) AS n FROM t GROUP BY k",
                        return_futures=False), "k")
    for key, r in got.items():
        xs = [Fraction(float(a)) for a in x[(k == key) & ~np.isnan(y)]]
        mean = sum(xs) / len(xs)
        exact = float(sum((a - mean) ** 2 for a in xs))
        assert int(r["n"]) == len(xs)
        np.testing.assert_allclose(r["s"], exact, rtol=1e-9, err_msg=str(key))
