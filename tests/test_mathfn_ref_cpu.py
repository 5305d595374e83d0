"""The numeric SQL functions on the host: the NumPy restatements of tests/mathfn_ref.py against NumPy itself, the
planner's arity / argument / result types, and the folding of calls on literals.  No kernel is launched."""
import math

import numpy as np
import pandas as pd
import pytest

from tests import mathfn_ref as M

HALVES = [0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 0.125, 0.375, 1.0005, 2.675, 1234.5, -1234.5, 0.0, -0.0,
          2.0 ** 52 + 0.5, 2.0 ** 52 - 0.5, -(2.0 ** 52 + 0.5), 2.0 ** 53, 1e22, 1e-22, 5e-324, 1.7976931348623157e308,
          math.inf, -math.inf, math.nan, 123456.789, -9.87e15, 0.045, 1e300, -1e-300]


def _same_words(got, exp):
    """bit for bit, except that any NaN matches any NaN"""
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    ok = (got.view(np.int64) == exp.view(np.int64)) | (np.isnan(got) & np.isnan(exp))
    return bool(ok.all())


@pytest.mark.parametrize("d", list(range(-25, 26)) + [300, 308, 309, 320, 400])
def test_round_factor_rule_is_numpys(d):
    x = np.array(HALVES + list(np.random.default_rng(d + 100).normal(0, 10.0 ** (d % 7), 200)))
    with np.errstate(all="ignore"):
        exp = np.round(x, d)
    assert _same_words(M.round_(x, d), exp), d
    if d >= 309:
        assert math.isinf(M.pow10(d)) and np.isnan(exp[np.isfinite(x)]).all()


def test_pow10_differs_from_the_plain_power():
    for d in (23, 25, 300, 308):
        assert M.pow10(d) != 10.0 ** d, d
    from dask_sql_b200 import expr as E
    for d in list(range(0, 40)) + [300, 308, 309, 400]:
        assert E.pow10(d) == M.pow10(d), d


def _pool():
    rng = np.random.default_rng(7)
    base = np.array(HALVES + [1.0, -1.0, 3.0, -3.0, 4.0, -4.0, 2.5e-300, 7.0, -7.0, 0.1, 1e308])
    return np.concatenate([base, rng.normal(0, 100, 2000), rng.uniform(-1e6, 1e6, 2000)])


def test_mod_sign_degrees_radians_restate_numpy():
    x = _pool()
    a, b = np.meshgrid(x[:60], x[:60])
    with np.errstate(all="ignore"):
        assert _same_words(M.mod(a, b), np.mod(a, b))
        assert _same_words(M.mod(x, 2.5), np.mod(x, 2.5)) and _same_words(M.mod(x, -4.0), np.mod(x, -4.0))
    assert _same_words(M.sign(x), np.sign(x))
    assert _same_words(M.sign(np.array([-0.0])), [0.0]) and M.sign(np.array([-0.0])).view(np.int64)[0] == 0
    assert _same_words(M.degrees(x), np.degrees(x)) and _same_words(M.radians(x), np.radians(x))


def test_integer_power_wraps_like_numpy():
    rng = np.random.default_rng(1)
    x = np.concatenate([np.array([0, 1, -1, 2, -2, 3, 10, -10, 2 ** 31, -(2 ** 62), 2 ** 63 - 1, -(2 ** 63)]),
                        rng.integers(-(2 ** 63), 2 ** 63 - 1, 300, dtype=np.int64)])
    y = np.array([0, 1, 2, 3, 5, 62, 63, 64, 65, 127, 1000, 2 ** 40])
    a, b = np.meshgrid(x, y)
    got, null = M.pow_i(a, b)
    with np.errstate(all="ignore"):
        assert (got == np.power(a, b)).all() and not null.any()
    got, null = M.pow_i(np.array([2, 0, 1]), np.array([-1, -2, -(2 ** 63)]))
    assert null.all() and (got == 0).all()
    with pytest.raises(ValueError):
        np.power(np.int64(2), np.int64(-1))


def test_ulp_distance_and_the_correctly_rounded_reference():
    assert M.ulp_distance(1.0, np.nextafter(1.0, 2.0))[0] == 1
    assert M.ulp_distance(0.0, -0.0)[0] == 0 and M.ulp_distance(-5e-324, 5e-324)[0] == 2
    assert M.ulp_distance(2.0 ** 62, np.nextafter(2.0 ** 62, 0))[0] == 1
    assert M.ulp_error(math.exp(1.0), M.exact_mp(M.FN_EXP, 1.0)) <= 0.5
    assert M.ulp_error(math.sin(1e22), M.exact_mp(M.FN_SIN, 1e22)) <= 0.5    # needs the raised precision
    assert M.ulp_error(math.cos(1e300), M.exact_mp(M.FN_COS, 1e300)) <= 0.5
    assert M.ulp_error(np.cbrt(-27.0), M.exact_mp(M.FN_CBRT, -27.0)) == 0


# ---- the planner -----------------------------------------------------------------------------------------
def _ctx():
    from dask_sql_b200 import Context
    c = Context()
    c.create_table("t", pd.DataFrame({"i": np.array([1, 2, 3], np.int64), "v": [1.0, 2.0, 3.0],
                                      "b": [True, False, True],
                                      "ts": np.array([0, 1, 2], dtype="datetime64[us]")}))
    return c


UNARY = ["CEIL", "FLOOR", "TRUNCATE", "ROUND", "SIGN", "DEGREES", "RADIANS", "SQRT", "EXP", "LN", "LOG10", "CBRT",
         "SIN", "COS", "TAN", "COT", "ASIN", "ACOS", "ATAN"]


@pytest.mark.parametrize("arg", ["i", "v"])
def test_result_types(arg):
    c = _ctx()
    items = [f"{f}({arg}) AS {f.lower()}" for f in UNARY] + \
        [f"{f}({arg}, {arg}) AS {f.lower()}" for f in ("ATAN2", "POWER", "MOD")] + \
        [f"ROUND({arg}, 2) AS round2", f"ROUND({arg}, -1) AS roundm", f"{arg} % 2 AS pct", f"POWER({arg}, 2) AS p2"]
    lf = c.sql(f"SELECT {', '.join(items)} FROM t")
    types = {k: str(v) for k, v in lf.dtypes.items()}
    big = "int64" if arg == "i" else "float64"
    exp = {f.lower(): "float64" for f in UNARY + ["ATAN2", "MOD"]}
    exp.update(power=big, p2=big, round2="float64", roundm="float64", pct=big)
    assert types == exp


@pytest.mark.parametrize("sql,name", [("SIN(v, v)", "SIN"), ("ATAN2(v)", "ATAN2"), ("POWER(i)", "POWER"),
                                      ("MOD(i, i, i)", "MOD"), ("ROUND(v, 1, 2)", "ROUND"), ("LN()", "LN"),
                                      ("SQRT(b)", "SQRT"), ("EXP(ts)", "EXP"), ("POWER(i, b)", "POWER"),
                                      ("FLOOR(ts)", "FLOOR"), ("ROUND(v, 1.5)", "ROUND"), ("ROUND(v, 'a')", "ROUND"),
                                      ("COS(v > 1)", "COS")])
def test_wrong_arity_or_argument_type_names_the_function(sql, name):
    from dask_sql_b200.utils import ParsingException
    with pytest.raises(ParsingException, match=name):
        _ctx().sql(f"SELECT {sql} AS x FROM t")


def test_string_argument_is_refused():
    from dask_sql_b200 import Context
    from dask_sql_b200.utils import ParsingException
    c = Context()
    c.create_table("s", pd.DataFrame({"s": pd.Categorical(["a", "b"]), "v": [1.0, 2.0]}))
    with pytest.raises(ParsingException, match="LOG10"):
        c.sql("SELECT LOG10(s) AS x FROM s")


def test_round_with_column_digits_is_not_implemented():
    with pytest.raises(NotImplementedError, match="ROUND"):
        _ctx().sql("SELECT ROUND(v, i) AS x FROM t")


def test_floor_ceil_to_unit_keep_their_temporal_path():
    lf = _ctx().sql("SELECT FLOOR(ts TO HOUR) AS f, CEIL(ts TO SECOND) AS c FROM t")
    assert str(lf.dtypes["f"]) == "datetime64[us]" and str(lf.dtypes["c"]) == "datetime64[us]"
    with pytest.raises(NotImplementedError):
        _ctx().sql("SELECT FLOOR(ts TO YEAR) AS f FROM t")


def test_calls_on_literals_fold_on_the_host():
    lf = _ctx().sql("SELECT ROUND(2.5) AS a, POWER(2, 62) AS b, MOD(7, 0) AS c, ROUND(1234.5678, -2) AS d, "
                    "ROUND(2.675, 2) AS e, MOD(-7, 3) AS f, MOD(7.5, -2) AS g, POWER(2, -1) AS h, "
                    "POWER(3, 41) AS k, POWER(2.0, 0.5) AS l, SIGN(-0.0) AS m, LN(0.0) AS n, ATAN2(1, 0) AS o, "
                    "CEIL(NULL) AS p, TRUNCATE(-2.7) AS q, SQRT(16) AS r FROM t")
    got = {n: lf.exprs[n].value for n in lf.columns}
    assert got["a"] == 2.0 and isinstance(got["a"], float)
    assert got["b"] == 4611686018427387904 and isinstance(got["b"], int)
    assert got["c"] is None and got["h"] is None and got["p"] is None
    assert got["d"] == 1200.0 and got["e"] == np.round(2.675, 2)
    assert got["f"] == 2.0 and got["g"] == np.mod(7.5, -2.0)
    assert got["k"] == int(np.power(np.int64(3), np.int64(41)))          # wraps modulo 2^64
    assert got["l"] == math.sqrt(2.0) and got["m"] == 0.0 and math.copysign(1, got["m"]) == 1
    assert got["n"] == -math.inf and got["o"] == math.pi / 2 and got["q"] == -2.0 and got["r"] == 4.0
    assert str(lf.dtypes["b"]) == "int64" and str(lf.dtypes["c"]) == "float64"


def test_programs_compile_to_the_new_opcodes():
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import expr as E
    i, v = E.ColRef("i", E.I64), E.ColRef("v", E.F64)

    def code(e):
        p = E.compile_expr(e, ["i", "v"])
        return [(p.code[k].op, p.code[k].a, p.code[k].imm_i, p.code[k].imm_f) for k in range(p.n)]

    assert code(E.math("round", [v], -2)) == [(L.OP_LOAD, 1, 0, 0.0), (L.OP_MATH_F, L.FN_ROUND, 1, 100.0)]
    assert code(E.math("ln", [i])) == [(L.OP_LOAD, 0, 0, 0.0), (L.OP_I2F, 0, 0, 0.0), (L.OP_MATH_F, L.FN_LN, 0, 0.0)]
    assert code(E.math("power", [i, 2])) == [(L.OP_LOAD, 0, 0, 0.0), (L.OP_CONST_I, 0, 2, 0.0), (L.OP_POW_I, 0, 0, 0.0)]
    assert code(E.math("mod", [i, 4]))[-2:] == [(L.OP_MOD_I, 0, 0, 0.0), (L.OP_I2F, 0, 0, 0.0)]
    assert code(E.binop("mod", v, 2.5))[-1] == (L.OP_MATH2_F, L.FN_MOD, 0, 0.0)
    assert code(E.math("atan2", [v, i]))[-1] == (L.OP_MATH2_F, L.FN_ATAN2, 0, 0.0)
    assert code(E.math("sqrt", [v]))[-1][0] == L.OP_SQRT_F
    assert E.may_be_null(E.math("power", [i, i]), lambda n: False)
    assert E.may_be_null(E.math("mod", [i, i]), lambda n: False)
    assert not E.may_be_null(E.math("sin", [v]), lambda n: False)
