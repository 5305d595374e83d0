"""NumPy reference of the numeric SQL functions of b2_expr_eval (B2_OP_MATH_F, B2_OP_MATH2_F, B2_OP_POW_I), one
entry per function id of include/b200sql.h, and the yardsticks the tests hold the device to.

The rule of each function is the NumPy call the reference makes for it (dask_sql/physical/rex/core/call.py:
1091-1113).  Two kinds of function:
  * exact: CEIL, FLOOR, TRUNCATE, ROUND, SIGN, DEGREES, RADIANS, MOD and the integer POWER are determined bit for
    bit (IEEE operations without contraction), so the device must match the restatements below word for word;
  * bounded: EXP, LN, LOG10, CBRT, SIN, COS, TAN, COT, ASIN, ACOS, ATAN, ATAN2 and the double POWER come from the
    CUDA Math API, whose documented maximum error is ULP_BOUND ulps of the correctly rounded result.  `exact_mp`
    gives that result through mpmath.
No GPU and no package import: NumPy and mpmath only."""
import mpmath
import numpy as np

# function ids: the numbers of include/b200sql.h (B2_FN_*)
(FN_CEIL, FN_FLOOR, FN_TRUNC, FN_ROUND, FN_SIGN, FN_DEGREES, FN_RADIANS, FN_EXP, FN_LN, FN_LOG10, FN_CBRT, FN_SIN,
 FN_COS, FN_TAN, FN_COT, FN_ASIN, FN_ACOS, FN_ATAN, FN_ATAN2, FN_POW, FN_MOD) = range(21)
UNARY = list(range(FN_CEIL, FN_ATAN2))
BINARY = [FN_ATAN2, FN_POW, FN_MOD]
NAMES = ["ceil", "floor", "truncate", "round", "sign", "degrees", "radians", "exp", "ln", "log10", "cbrt", "sin",
         "cos", "tan", "cot", "asin", "acos", "atan", "atan2", "power", "mod"]
EXACT = {FN_CEIL, FN_FLOOR, FN_TRUNC, FN_ROUND, FN_SIGN, FN_DEGREES, FN_RADIANS, FN_MOD}

# Maximum ulp error of the CUDA Math API's double-precision functions: CUDA C++ Programming Guide (CUDA 12.9),
# appendix "Mathematical Functions", table "Double-Precision Mathematical Standard Library Functions with Maximum
# ULP Error" (the library is built without fast-math, so these are the functions that run).  COT is 1 / tan(x):
# tan's 2 ulp plus the half ulp of the division's rounding, counted as 3.  LOG10 is held to 2 ulp: on an H100
# log10(0.11027725308110115) gives -0.9575140603625814, 1.10 ulp from the exact value.
ULP_BOUND = {FN_EXP: 1, FN_LN: 1, FN_LOG10: 2, FN_CBRT: 1, FN_SIN: 2, FN_COS: 2, FN_TAN: 2, FN_COT: 3,
             FN_ASIN: 2, FN_ACOS: 2, FN_ATAN: 2, FN_ATAN2: 2, FN_POW: 2}

NUMPY = {FN_CEIL: np.ceil, FN_FLOOR: np.floor, FN_TRUNC: np.trunc, FN_SIGN: np.sign, FN_DEGREES: np.degrees,
         FN_RADIANS: np.radians, FN_EXP: np.exp, FN_LN: np.log, FN_LOG10: np.log10, FN_CBRT: np.cbrt,
         FN_SIN: np.sin, FN_COS: np.cos, FN_TAN: np.tan, FN_COT: lambda x: 1 / np.tan(x), FN_ASIN: np.arcsin,
         FN_ACOS: np.arccos, FN_ATAN: np.arctan, FN_ATAN2: np.arctan2, FN_POW: np.power, FN_MOD: np.mod}


# ---- exact functions ----------------------------------------------------------------------------------------
def pow10(d: int) -> float:
    """NumPy's power of ten for np.round (multiarray/calculation.c, power_of_ten): 1e0 .. 1e8 from a table, then
    1e9 multiplied by 10.0 once per further digit.  inf from d = 309 on."""
    if d < 9:
        return [1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8][d]
    r = 1e9
    for _ in range(d - 9):
        r *= 10.0
    return r


def round_(x, d: int):
    """np.round(x, d) on float64: rint(x * f) / f, or rint(x / f) * f for d < 0."""
    x = np.asarray(x, np.float64)
    f = pow10(abs(d))
    with np.errstate(all="ignore"):
        return np.rint(x / f) * f if d < 0 else np.rint(x * f) / f


def sign(x):
    """np.sign on float64: +-1.0, +0.0 for +-0.0 and NaN for NaN"""
    x = np.asarray(x, np.float64)
    return np.where(x > 0, 1.0, np.where(x < 0, -1.0, np.where(x == 0, 0.0, x)))


def degrees(x):
    return np.asarray(x, np.float64) * (180.0 / np.pi)


def radians(x):
    return np.asarray(x, np.float64) * (np.pi / 180.0)


def mod(x, y):
    """np.mod on float64 (npymath npy_divmod's remainder): fmod, moved onto y's sign; a zero result takes y's
    sign; x mod 0 is fmod's NaN"""
    x, y = np.broadcast_arrays(np.asarray(x, np.float64), np.asarray(y, np.float64))
    with np.errstate(all="ignore"):
        r = np.fmod(x, y)
        move = (y != 0) & (r != 0) & ((y < 0) != (r < 0))
        r = np.where(move, r + y, r)
        return np.where((y != 0) & (r == 0), np.copysign(0.0, y), r)


def pow_i(x, y):
    """np.power on int64 for y >= 0: x ** y modulo 2^64.  Returns (values, null): y < 0 is NULL (NumPy raises)."""
    x, y = np.broadcast_arrays(np.asarray(x, np.int64), np.asarray(y, np.int64))
    base, e = x.astype(np.uint64), np.where(y < 0, 0, y).astype(np.uint64)
    r = np.ones(x.shape, np.uint64)
    with np.errstate(all="ignore"):
        while e.any():
            r = np.where(e & np.uint64(1), r * base, r)
            base = base * base
            e = e >> np.uint64(1)
    return np.where(y < 0, 0, r.view(np.int64)), y < 0


def exact(fn: int, x, y=None, digits: int = 0):
    """the exact functions on float64 arrays"""
    if fn == FN_ROUND:
        return round_(x, digits)
    if fn == FN_SIGN:
        return sign(x)
    if fn == FN_DEGREES:
        return degrees(x)
    if fn == FN_RADIANS:
        return radians(x)
    if fn == FN_MOD:
        return mod(x, y)
    return NUMPY[fn](np.asarray(x, np.float64))


# ---- bounded functions ----------------------------------------------------------------------------------
def ulp_distance(a, b):
    """number of doubles between a and b (0 when equal; +0.0 and -0.0 are 0 apart), as float64"""
    a, b = np.atleast_1d(np.asarray(a, np.float64)), np.atleast_1d(np.asarray(b, np.float64))
    ia, ib = a.view(np.int64), b.view(np.int64)
    oa = np.where(ia < 0, -(ia & np.int64((1 << 63) - 1)), ia)
    ob = np.where(ib < 0, -(ib & np.int64((1 << 63) - 1)), ib)
    far = np.abs(oa.astype(np.float64) - ob.astype(np.float64))
    with np.errstate(all="ignore"):
        near = np.abs(oa - ob).astype(np.float64)       # exact unless the int64 difference overflows
    return np.where(far > 2.0 ** 62, far, near)


_MP = {FN_EXP: mpmath.exp, FN_LN: mpmath.log, FN_LOG10: lambda v: mpmath.log(v, 10), FN_CBRT: mpmath.cbrt,
       FN_SIN: mpmath.sin, FN_COS: mpmath.cos, FN_TAN: mpmath.tan, FN_COT: mpmath.cot, FN_ASIN: mpmath.asin,
       FN_ACOS: mpmath.acos, FN_ATAN: mpmath.atan, FN_ATAN2: mpmath.atan2, FN_POW: mpmath.power}


def exact_mp(fn: int, x: float, y: float = None):
    """the real value of a bounded function at finite arguments with a finite real result, as an mpf; the
    working precision covers the exponent of x so that sin / cos / tan of 1e300 reduce correctly.  At an
    infinite argument, and at a zero argument of ATAN2 / POWER, the value is C99's special case (atan(inf) =
    pi/2 rounded, atan2(-0, -1) = -pi rounded, pow(x, 0) = 1), taken from NumPy, which follows C99 there."""
    args = [x] if y is None else [x, y]
    if not all(np.isfinite(args)) or (fn in (FN_ATAN2, FN_POW) and 0.0 in args):
        with np.errstate(all="ignore"):
            return mpmath.mpf(float(NUMPY[fn](*args)))
    e = max(abs(mpmath.mpf(v).exp) if v else 0 for v in ([x] if y is None else [x, y]))
    with mpmath.workprec(200 + e):
        if fn == FN_CBRT:
            r = mpmath.cbrt(abs(x)) * (1 if x >= 0 else -1)
        elif fn == FN_ATAN2:
            r = mpmath.atan2(x, y)
        elif fn == FN_POW:
            r = mpmath.power(x, y)
        else:
            r = _MP[fn](x)
        return +r


def ulp_error(got: float, real) -> float:
    """|got - real| in ulps of the double nearest to `real` (subnormal spacing near 0)"""
    near = abs(float(real))
    unit = float(np.spacing(np.float64(near))) if near < 2.0 ** 1023 else 2.0 ** 971    # top binade's spacing
    with mpmath.workprec(300):
        return float(abs(mpmath.mpf(got) - real) / unit)
