"""The numeric SQL functions end to end through Context.sql() on the GPU: the reference's test_math_operations
(tests/golden/reference_math.py) and queries that put the functions on every expression path -- SELECT lists,
aggregate inputs, mask predicates, computed group keys and the Q3 star join -- against pandas, over
multi-partition tables with NULL and NaN rows."""
import numpy as np
import pandas as pd
import pytest

from tests import mathfn_ref as M
from tests.golden import reference_math as G
from tests.golden import reference_vectors as V

pytestmark = pytest.mark.gpu

EXACT_COLS = {"abs", "ceil", "floor", "mod", "round", "round2", "sign", "truncate"}
BOUND = {"acos": M.FN_ACOS, "asin": M.FN_ASIN, "atan": M.FN_ATAN, "atan2": M.FN_ATAN2, "cbrt": M.FN_CBRT,
         "cos": M.FN_COS, "cot": M.FN_COT, "exp": M.FN_EXP, "log10": M.FN_LOG10, "ln": M.FN_LN,
         "power": M.FN_POW, "power2": M.FN_POW, "sin": M.FN_SIN, "tan": M.FN_TAN}


def _same(got, exp):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    return bool(((got.view(np.int64) == exp.view(np.int64)) | (np.isnan(got) & np.isnan(exp))).all())


def _within(got, exp, ulps):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    both_nan = np.isnan(got) & np.isnan(exp)
    return bool((both_nan | (M.ulp_distance(got, exp) <= ulps)).all())


def test_reference_math_operations():
    from dask_sql_b200 import Context
    df = V.df()
    c = Context()
    c.create_table("df", df, npartitions=3)
    got = c.sql(G.SQL).compute().reset_index(drop=True)
    assert list(got.columns) == [a for _, a in G.SELECT]
    for name, fn in G.EXPECTED.items():
        exp = np.asarray(fn(df), np.float64)
        col = got[name].to_numpy(np.float64)
        assert got[name].dtype == np.float64, name
        if name in EXACT_COLS:
            assert _same(col, exp), (G.CITE, name)
        elif name in ("degrees", "radians"):
            # exact against np.degrees / np.radians; the reference writes b / pi * 180, a rounding apart
            assert _same(col, (np.degrees if name == "degrees" else np.radians)(df.b)), name
            assert _within(col, exp, 2), (G.CITE, name)
        else:
            # NumPy is within 1 ulp of the exact value, the device within its bound
            assert _within(col, exp, M.ULP_BOUND[BOUND[name]] + 1), (G.CITE, name)


@pytest.fixture(scope="module")
def ctx():
    from dask_sql_b200 import Context
    rng = np.random.default_rng(11)
    n = 50_000
    v = rng.uniform(0.01, 10.0, n)
    v[rng.random(n) < 0.03] = np.nan
    i = pd.array(rng.integers(-40, 40, n), dtype="Int64")
    i[rng.random(n) < 0.05] = pd.NA
    t = pd.DataFrame({"k": rng.integers(0, 7, n), "v": v, "x": rng.uniform(-100, 100, n), "i": i,
                      "w": rng.choice([0.5, 0.45, 0.55, 0.44999999999999996, 1.25, 2.0], n)})
    nd = 500
    dim = pd.DataFrame({"pk": rng.permutation(nd), "grp": rng.integers(0, 20, nd), "flag": rng.integers(0, 10, nd)})
    fact = pd.DataFrame({"fk": rng.integers(0, nd, 200_000), "val": rng.normal(0, 3, 200_000)})
    fact.loc[fact.index % 97 == 0, "val"] = np.nan
    c = Context()
    c.create_table("t", t, npartitions=4)
    c.create_table("d", dim)
    c.create_table("f", fact, npartitions=3)
    return c, t, dim, fact


def _sorted(df, by):
    return df.sort_values(by).reset_index(drop=True)


def test_round_of_a_sum_per_group(ctx):
    c, t, _, _ = ctx
    got = _sorted(c.sql("SELECT k, ROUND(SUM(v), 2) AS s FROM t GROUP BY k").compute(), "k")
    exp = t.groupby("k")["v"].sum()
    assert got["s"].dtype == np.float64
    # the float sums differ in their last bits with the summation order; ROUND to 2 digits then agrees
    np.testing.assert_allclose(got["s"], np.round(exp.to_numpy(), 2), rtol=0, atol=0.011)


def test_sum_of_ln_with_a_filter(ctx):
    c, t, _, _ = ctx
    got = c.sql("SELECT SUM(LN(v)) AS s FROM t WHERE x > 0").compute()
    exp = np.log(t.v[t.x > 0]).sum()
    np.testing.assert_allclose(got["s"].iloc[0], exp, rtol=1e-12)


def test_round_in_a_mask_predicate(ctx):
    c, t, _, _ = ctx
    got = c.sql("SELECT k, w FROM t WHERE ROUND(w, 1) = 0.5").compute()
    exp = t[np.round(t.w, 1) == 0.5]
    assert len(got) == len(exp) and sorted(got["w"].tolist()) == sorted(exp["w"].tolist())


def test_floor_as_a_group_key(ctx):
    c, t, _, _ = ctx
    got = c.sql("SELECT g, COUNT(*) AS n, SUM(v) AS s FROM (SELECT FLOOR(x / 10) AS g, v FROM t) AS q "
                "GROUP BY g").compute()
    got = _sorted(got, "g")
    exp = t.assign(g=np.floor(t.x / 10)).groupby("g").agg(n=("v", "size"), s=("v", "sum")).reset_index()
    assert got["g"].dtype == np.float64
    assert got["g"].tolist() == exp["g"].tolist() and got["n"].tolist() == exp["n"].tolist()
    np.testing.assert_allclose(got["s"], exp["s"], rtol=1e-9)


def test_integer_power_of_a_nullable_bigint(ctx):
    c, t, _, _ = ctx
    got = c.sql("SELECT i, i * i AS sq, POWER(i, 2) AS p, POWER(i, 13) AS p13, MOD(i, 7) AS m FROM t").compute()
    # a BIGINT result with NULL rows comes back as every nullable integer expression does (i * i)
    assert got["p"].dtype == got["sq"].dtype and got["m"].dtype == np.float64
    i = t.i
    null = i.isna().to_numpy()
    assert (got["p"].isna().to_numpy() == null).all()
    vals = i.fillna(0).to_numpy(np.int64)
    with np.errstate(all="ignore"):
        for col, e in (("p", 2), ("p13", 13)):     # 40 ** 13 wraps modulo 2^64, as in NumPy
            exp = np.power(vals, e).astype(np.float64)[~null]
            assert (got[col].to_numpy(np.float64, na_value=np.nan)[~null] == exp).all(), col
    assert _same(got["m"].to_numpy(np.float64)[~null], np.mod(vals, 7)[~null].astype(np.float64))
    assert got["m"].isna().to_numpy()[null].all()


def test_mod_and_percent_on_doubles(ctx):
    c, t, _, _ = ctx
    got = c.sql("SELECT x, MOD(x, 4) AS a, x % 2.5 AS b, MOD(x, -3.5) AS c, MOD(i, 0) AS z FROM t").compute()
    for col, exp in (("a", np.mod(t.x, 4.0)), ("b", np.mod(t.x, 2.5)), ("c", np.mod(t.x, -3.5))):
        assert got[col].dtype == np.float64 and _same(got[col], exp), col
    assert got["z"].isna().all()


def test_sum_of_a_power_in_the_q3_shape(ctx):
    c, _, dim, fact = ctx
    got = c.sql("SELECT d.grp, SUM(POWER(f.val, 2)) AS s FROM f JOIN d ON f.fk = d.pk WHERE d.flag < 5 "
                "GROUP BY d.grp").compute()
    got = _sorted(got, "grp")
    m = fact.merge(dim[dim.flag < 5], left_on="fk", right_on="pk")
    exp = m.assign(p=np.power(m.val, 2)).groupby("grp")["p"].sum().reset_index()
    assert got["grp"].tolist() == exp["grp"].tolist() and got["s"].dtype == np.float64
    np.testing.assert_allclose(got["s"], exp["p"], rtol=1e-9)
