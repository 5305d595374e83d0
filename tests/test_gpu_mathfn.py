"""The numeric SQL functions of b2_expr_eval (B2_OP_MATH_F, B2_OP_MATH2_F, B2_OP_POW_I) against tests/mathfn_ref.py,
through the C-ABI: an edge pool and about 10^6 random values per function over many magnitudes, with NULL rows.
Exact functions match word for word, validity words included; the others stay within the CUDA Math API's bound
of the correctly rounded value, and equal NumPy on the edge pool wherever the result is NaN, +-inf or +-0."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import mathfn_ref as M
from tests import rowwise_ref as R
from tests.test_gpu_rowwise import LD, run_prog

pytestmark = pytest.mark.gpu

OP_MATH_F, OP_MATH2_F, OP_POW_I = 63, 64, 65
NRAND = 1 << 20
DMAX, TINY = 1.7976931348623157e308, 5e-324
EDGES = [0.0, -0.0, TINY, -TINY, DMAX, -DMAX, math.inf, -math.inf, math.nan, 1.0, -1.0,
         math.pi / 2, np.nextafter(math.pi / 2, 0), np.nextafter(math.pi / 2, 4), -math.pi / 2, math.pi,
         709.782712893384, 709.7827128933841, 709.79, -745.1332191019411, -745.1332191019412, -745.2, -708.4,
         1e22, -1e22, 1e300, -1e300, 0.5, -0.5, 2.5, 3.5, -2.5, 1e-300, 2.0 ** 52 + 0.5, 2.0 ** 53, 1e16,
         np.nextafter(1.0, 0), np.nextafter(1.0, 2), np.nextafter(-1.0, 0), 4.0, -4.0, 2.0, 0.1, 10.0, 1e-5]


def _random(rng, n):
    """magnitudes 1e-300 .. 1e300 plus dense uniform ranges where the functions are interesting"""
    k = n // 4
    mags = np.exp(rng.uniform(-690, 690, k)) * rng.choice([-1.0, 1.0], k)
    parts = [mags, rng.uniform(-1.0, 1.0, k), rng.uniform(-20.0, 20.0, k), rng.uniform(-760.0, 760.0, n - 3 * k)]
    return rng.permutation(np.concatenate(parts))


def _nulls(n, seed):
    return np.random.default_rng(seed).random(n) < 0.05


def _unary_prog(fn, digits=0):
    return [LD(0), (OP_MATH_F, fn, int(digits < 0), M.pow10(abs(digits)) if fn == M.FN_ROUND else 0.0)]


def _binary_prog(fn):
    return [LD(0), LD(1), (OP_MATH2_F, fn, 0, 0.0)]


def _check_validity(got_valid, null, what):
    words = R.pack_valid(~null)
    bad = np.flatnonzero(got_valid != words)
    assert not len(bad), f"{what}: validity word {bad[0]} is {got_valid[bad[0]]:#x}, expected {words[bad[0]]:#x}"


def _check_exact(got_bits, exp, null, what):
    exp = np.where(null, 0.0, exp).view(np.int64)
    bad = (got_bits != exp) & ~(np.isnan(got_bits.view(np.float64)) & np.isnan(exp.view(np.float64)))
    assert not bad.any(), f"{what}: {int(bad.sum())} rows differ, first {np.flatnonzero(bad)[0]}"


def _check_bounded(fn, got, args, null, edge_rows, what):
    """every row within the bound; NumPy's NaN / inf / zero exactly on the edge rows"""
    with np.errstate(all="ignore"):
        ref = M.NUMPY[fn](*args)
    live = ~null
    g, r = got[live], ref[live]
    a = [x[live] for x in args]
    special = ~np.isfinite(r) | (r == 0)
    edge = edge_rows[live]
    # specials: equal to NumPy on the edge pool (NaN with NaN, signed infinities and zeros bit for bit)
    se = special & edge
    same = (g[se].view(np.int64) == r[se].view(np.int64)) | (np.isnan(g[se]) & np.isnan(r[se]))
    assert same.all(), f"{what}: edge {[x[se][~same][:3] for x in a]} gave {g[se][~same][:3]}, NumPy {r[se][~same][:3]}"
    # a domain error is NaN on every row, as in NumPy
    nan_diff = np.isnan(g) != np.isnan(r)
    assert not nan_diff.any(), f"{what}: NaN differs at {[x[nan_diff][:3] for x in a]}: {g[nan_diff][:3]}"
    # every other row is within the bound of the correctly rounded value.  NumPy (glibc, under 1 ulp) is the
    # sieve: a row fewer than `bound` ulps from NumPy is within the bound; the rest (for a 1-ulp function that
    # is every row where the two differ at all), rows where only one side is +-inf / 0, the edge rows and a
    # sample go to mpmath
    bound = M.ULP_BOUND[fn]
    g_special = ~np.isfinite(g) | (g == 0)
    d = M.ulp_distance(g, r)
    rng = np.random.default_rng(fn)
    sample = np.zeros(len(g), bool)
    sample[rng.choice(len(g), min(len(g), 300), replace=False)] = True
    check = np.flatnonzero(~np.isnan(r) & ((special != g_special) | (~special & ((d >= bound) | edge | sample))))
    assert len(check) < len(g) // 5, f"{what}: {len(check)} rows are {bound}+ ulp away from NumPy"
    for i in check:
        ex = M.exact_mp(fn, *[float(x[i]) for x in a])
        err = M.ulp_error(float(g[i]), ex)
        assert err <= bound, f"{what}: at {[float(x[i]) for x in a]} got {g[i]!r}, {err:.2f} ulp from {ex}"


@pytest.mark.parametrize("fn", M.UNARY, ids=[M.NAMES[f] for f in M.UNARY])
def test_unary_function(fn):
    rng = np.random.default_rng(100 + fn)
    x = np.concatenate([np.array(EDGES, np.float64), _random(rng, NRAND)])
    edge = np.zeros(len(x), bool)
    edge[: len(EDGES)] = True
    null = _nulls(len(x), fn)
    null[: len(EDGES)] = False
    col = R.Column(x, null, R.F64)
    for digits in ([0, 2, -1, 3, 16, -20, 309] if fn == M.FN_ROUND else [0]):
        what = f"{M.NAMES[fn]}({digits})"
        got, got_valid = run_prog(_unary_prog(fn, digits), R.F64, [col], len(x))
        _check_validity(got_valid, null, what)
        if fn in M.EXACT:
            _check_exact(got, M.exact(fn, x, digits=digits), null, what)
        else:
            _check_bounded(fn, got.view(np.float64), [x], null, edge, what)


@pytest.mark.parametrize("fn", M.BINARY, ids=[M.NAMES[f] for f in M.BINARY])
def test_binary_function(fn):
    rng = np.random.default_rng(200 + fn)
    e = np.array(EDGES, np.float64)
    ex, ey = [a.ravel() for a in np.meshgrid(e, e)]
    n = NRAND
    if fn == M.FN_POW:      # bases of all magnitudes, exponents where the result stays mostly finite
        rx = np.abs(_random(rng, n)) * np.where(rng.random(n) < 0.2, -1, 1)
        ry = np.where(rng.random(n) < 0.3, rng.integers(-30, 30, n).astype(float), rng.uniform(-4, 4, n))
    else:
        rx, ry = _random(rng, n), rng.permutation(_random(rng, n))
    x, y = np.concatenate([ex, rx]), np.concatenate([ey, ry])
    edge = np.zeros(len(x), bool)
    edge[: len(ex)] = True
    nx, ny = _nulls(len(x), fn), _nulls(len(x), fn + 50)
    nx[: len(ex)] = ny[: len(ex)] = False
    got, got_valid = run_prog(_binary_prog(fn), R.F64, [R.Column(x, nx, R.F64), R.Column(y, ny, R.F64)], len(x))
    null = nx | ny
    _check_validity(got_valid, null, M.NAMES[fn])
    if fn in M.EXACT:
        _check_exact(got, M.exact(fn, x, y), null, M.NAMES[fn])
        with np.errstate(all="ignore"):
            _check_exact(got, np.mod(x, y), null, "np.mod")
    else:
        _check_bounded(fn, got.view(np.float64), [x, y], null, edge, M.NAMES[fn])


def test_integer_power_and_integer_mod():
    rng = np.random.default_rng(9)
    pool = [0, 1, -1, 2, -2, 3, -3, 10, 2 ** 31, -(2 ** 62), 2 ** 63 - 1, -(2 ** 63), 1_234_567]
    exps = [0, 1, 2, 3, 5, 62, 63, 64, 65, 1000, 2 ** 40, -1, -2, -(2 ** 63)]
    a, b = [v.ravel() for v in np.meshgrid(np.array(pool, np.int64), np.array(exps, np.int64))]
    n = 1 << 18
    x = np.concatenate([a, rng.integers(-(2 ** 63), 2 ** 63 - 1, n, dtype=np.int64)])
    y = np.concatenate([b, rng.integers(-3, 70, n, dtype=np.int64)])
    nx, ny = _nulls(len(x), 1), _nulls(len(x), 2)
    cols = [R.Column(x, nx, R.I64), R.Column(y, ny, R.I64)]
    got, got_valid = run_prog([LD(0), LD(1), (OP_POW_I, 0, 0, 0.0)], R.I64, cols, len(x))
    exp, neg = M.pow_i(x, y)
    null = nx | ny | neg
    _check_validity(got_valid, null, "pow_i")
    assert (got == np.where(null, 0, exp)).all()
    # MOD of two integers: the floored B2_OP_MOD_I, then to double; a zero divisor is NULL
    y2 = np.where(np.arange(len(y)) % 11 == 0, 0, y)
    cols = [R.Column(x, nx, R.I64), R.Column(y2, ny, R.I64)]
    got, got_valid = run_prog([LD(0), LD(1), (R.OP_MOD_I, 0, 0, 0.0), (R.OP_I2F, 0, 0, 0.0)], R.F64, cols, len(x))
    null = nx | ny | (y2 == 0)
    _check_validity(got_valid, null, "mod_i")
    with np.errstate(all="ignore"):
        exp = np.mod(x, np.where(y2 == 0, 1, y2)).astype(np.float64)
    _check_exact(got, exp, null, "mod_i")


def test_unknown_function_is_an_error_before_any_launch():
    import torch
    from dask_sql_b200 import _lib as L
    from tests.test_gpu_rowwise import Dev, _ptr, _stream
    col = Dev(R.Column(np.array([1.0, 2.0, 3.0]), None, R.F64))
    arr = (L.Col * 2)()
    arr[0] = arr[1] = col.struct()
    out = torch.full((3,), 0x5A, dtype=torch.int64, device="cuda")
    for code in ([LD(0), (OP_MATH_F, M.FN_ATAN2, 0, 0.0)], [LD(0), (OP_MATH_F, -1, 0, 0.0)],
                 [LD(0), (OP_MATH_F, M.FN_ROUND, 2, 1.0)], [LD(0), LD(1), (OP_MATH2_F, M.FN_ATAN, 0, 0.0)],
                 [LD(0), LD(1), (OP_MATH2_F, 21, 0, 0.0)], [LD(0), (OP_MATH2_F, M.FN_POW, 0, 0.0)]):
        p = L.Prog()
        p.n, p.out_dtype = len(code), R.F64
        for i, (op, a, ii, ff) in enumerate(code):
            p.code[i].op, p.code[i].a, p.code[i].imm_i, p.code[i].imm_f = op, a, ii, ff
        with pytest.raises(L.B200SqlError):
            L.expr_eval(C.byref(p), arr, 2, 3, _ptr(out), C.c_void_p(0), _stream())
    torch.cuda.synchronize()
    assert (out.cpu() == 0x5A).all()
