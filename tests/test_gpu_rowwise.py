"""The row-wise kernels bit for bit against the NumPy reference of tests/rowwise_ref.py, through the C-ABI:
the postfix interpreter b2_expr_eval (every opcode), the predicate terms every fused scan shares
(b2_eval_terms, checked through b2_select_count/write and b2_scan_agg), b2_sort_by, b2_gather and
b2_col_stats.  Operands are the int64 / float64 edges where kernels go wrong (INT64_MIN, 2^53 + 1, ±0.0,
±inf, NaN, subnormals), and row counts straddle the warp (32), the per-lane batch (512), the selection
tile (4096) and the sort chunk (16384)."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import rowwise_ref as R

pytestmark = pytest.mark.gpu

MIN, MAX = R.INT64_MIN, R.INT64_MAX
SIZES = [1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 4095, 4096, 4097, 16383, 16384, 16385, 100_003]
INT_POOL = [0, 1, -1, 2, -2, 3, -3, 7, -7, MIN, MIN + 1, MAX, 2 ** 31, -2 ** 31, 2 ** 32, -2 ** 32,
            2 ** 53, -2 ** 53, 2 ** 53 + 1, 1_234_567_890_123, -987_654_321, 6_917_529_027_641_081_856]
FLOAT_POOL = [0.0, -0.0, 1.5, -1.5, math.inf, -math.inf, math.nan, 5e-324, -5e-324, 1.7976931348623157e308,
              -1.7976931348623157e308, 2.0 ** 53, -2.0 ** 53, 2.0 ** 63, 3.0, -7.0, 0.1, -2.5e-300, 123456.789,
              -9.87e15]


# ---- plumbing --------------------------------------------------------------------------------------------
def _L():
    from dask_sql_b200 import _lib as L
    return L


def _dev():
    import torch
    return torch.device("cuda", torch.cuda.current_device())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


_NP = {R.I64: np.int64, R.F64: np.float64, R.U8: np.uint8}


class Dev:
    """a R.Column on the device: values + LSB-packed validity words (None = no bitmap)"""

    def __init__(self, col: R.Column):
        import torch
        self.col = col
        self.data = torch.from_numpy(np.ascontiguousarray(col.values)).to(_dev())
        self.valid = None
        if col.null is not None:
            self.valid = torch.from_numpy(R.pack_valid(~col.null).view(np.int32)).to(_dev())

    def struct(self):
        c = _L().Col()
        c.data = self.data.data_ptr() if self.data.numel() else 0
        c.valid = self.valid.data_ptr() if self.valid is not None and self.valid.numel() else 0
        c.dtype = self.col.dtype
        return c


def _pairs(pool, n, rng):
    """two columns of length n that run through the cartesian product of `pool` (shuffled, tiled)"""
    p = len(pool)
    k = rng.permutation(p * p)
    k = np.resize(k, n) if n else k[:0]
    return [pool[i] for i in k // p], [pool[i] for i in k % p]


def _column(vals, dtype, null=None):
    return R.Column(np.array(vals, dtype=_NP[dtype]), null, dtype)


def _null_pattern(n, mod, rem):
    return (np.arange(n) % mod) == rem


def _assert_words(got, exp, what, f64=False):
    """int64 words equal; for float64 words any NaN matches any NaN (the sign of zero counts)"""
    got, exp = np.asarray(got), np.asarray(exp)
    bad = got != exp
    if f64:
        bad &= ~(np.isnan(got.view(np.float64)) & np.isnan(exp.view(np.float64)))
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {len(bad)} rows differ; first at row {i}: "
                             f"got {got[i]!r}, expected {exp[i]!r}")


# ---- b2_expr_eval ------------------------------------------------------------------------------------------
def run_prog(code, out_dtype, cols, n):
    """the kernel's (out, valid words) for `code`; the outputs start as garbage so every written bit counts"""
    import torch
    L = _L()
    p = L.Prog()
    p.n, p.out_dtype = len(code), out_dtype
    for i, (op, a, ii, ff) in enumerate(code):
        p.code[i].op, p.code[i].a, p.code[i].imm_i, p.code[i].imm_f = op, a, ii, ff
    devs = [Dev(c) for c in cols]
    arr = (L.Col * max(1, len(devs)))()
    for i, d in enumerate(devs):
        arr[i] = d.struct()
    tdt = {R.I64: torch.int64, R.F64: torch.int64, R.U8: torch.uint8}[out_dtype]
    out = torch.full((max(n, 1),), 0x5A, dtype=tdt, device=_dev())
    valid = torch.full((max((n + 31) // 32, 1),), -1, dtype=torch.int32, device=_dev())
    L.expr_eval(C.byref(p), arr, len(devs), n, _ptr(out), _ptr(valid), _stream())
    torch.cuda.synchronize()
    return out.cpu().numpy()[:n], valid.cpu().numpy().view(np.uint32)[: (n + 31) // 32]


def check_prog(code, out_dtype, cols, n, what):
    got, got_valid = run_prog(code, out_dtype, cols, n)
    exp, exp_valid = R.eval_prog(code, out_dtype, cols, n)
    _assert_words(got, exp, what, f64=out_dtype == R.F64)
    words = R.pack_valid(exp_valid)
    bad = np.flatnonzero(got_valid != words)
    assert not len(bad), f"{what}: validity word {bad[0]} is {got_valid[bad[0]]:#x}, expected {words[bad[0]]:#x}"


def LD(i):
    return (R.OP_LOAD, i, 0, 0.0)


def OP(op):
    return (op, 0, 0, 0.0)


def CI(v):
    return (R.OP_CONST_I, 0, v, 0.0)


def CF(v):
    return (R.OP_CONST_F, 0, 0, v)


CN = (R.OP_CONST_NULL, 0, 0, 0.0)

INT_BINARY = [R.OP_ADD_I, R.OP_SUB_I, R.OP_MUL_I, R.OP_DIV_I, R.OP_MOD_I] + [R.OP_EQ_I + k for k in range(6)]
FLOAT_BINARY = [R.OP_ADD_F, R.OP_SUB_F, R.OP_MUL_F, R.OP_DIV_F] + [R.OP_EQ_F + k for k in range(6)]


@pytest.mark.parametrize("nulls", [False, True], ids=["valid", "nulls"])
@pytest.mark.parametrize("kind", ["int", "float"])
def test_expr_binary_ops_over_the_operand_product(kind, nulls):
    """every binary arithmetic / comparison opcode on every pair of the pool; with NULLs each operand is
    nulled in its own pattern (and both together on some rows)"""
    rng = np.random.default_rng(1 if kind == "int" else 2)
    pool = INT_POOL if kind == "int" else FLOAT_POOL
    dt = R.I64 if kind == "int" else R.F64
    n = len(pool) ** 2 + 37
    a, b = _pairs(pool, n, rng)
    ca = _column(a, dt, _null_pattern(n, 3, 0) if nulls else None)
    cb = _column(b, dt, _null_pattern(n, 5, 1) if nulls else None)
    for op in (INT_BINARY if kind == "int" else FLOAT_BINARY):
        out = R.U8 if (R.OP_EQ_I <= op <= R.OP_EQ_I + 5 or R.OP_EQ_F <= op <= R.OP_EQ_F + 5) else dt
        check_prog([LD(0), LD(1), OP(op)], out, [ca, cb], n, f"op {op}")
        check_prog([LD(1), LD(0), OP(op)], out, [ca, cb], n, f"op {op} swapped")
    if kind == "int":   # the literal forms the host compiler emits (a % 3, a % -3, a / -1 ...)
        for op in (R.OP_MOD_I, R.OP_DIV_I):
            for k in (3, -3, 1, -1, 0, MIN, MAX):
                check_prog([LD(0), CI(k), OP(op)], R.I64, [ca], n, f"op {op} by {k}")


def test_expr_modulo_is_floored():
    """the case the reference and the scalar fold agree on: -7 % 3 = 2, 7 % -3 = -2, x % 0 NULL"""
    a = _column([-7, 7, 7, -7, 6, -6, 5, MIN, MIN, MAX], R.I64)
    b = _column([3, -3, 3, -3, 3, 3, 0, -1, 3, -2], R.I64)
    got, valid = run_prog([LD(0), LD(1), OP(R.OP_MOD_I)], R.I64, [a, b], 10)
    assert got.tolist() == [2, -2, 1, -1, 0, 0, 0, 0, 1, -1]
    assert valid[0] == 0x3FF & ~(1 << 6)


@pytest.mark.parametrize("nulls", [False, True], ids=["valid", "nulls"])
def test_expr_unary_ops_at_the_edges(nulls):
    rng = np.random.default_rng(3)
    n = 4097
    ints = list(np.resize(INT_POOL, n))
    floats = list(np.resize(FLOAT_POOL, n))
    rng.shuffle(ints)
    rng.shuffle(floats)
    ci = _column(ints, R.I64, _null_pattern(n, 4, 1) if nulls else None)
    cf = _column(floats, R.F64, _null_pattern(n, 7, 2) if nulls else None)
    cases = [
        ([LD(0), OP(R.OP_NEG_I)], R.I64), ([LD(0), OP(R.OP_ABS_I)], R.I64), ([LD(0), OP(R.OP_I2F)], R.F64),
        ([LD(0), OP(R.OP_NOT)], R.U8), ([LD(0), OP(R.OP_ISNULL_I)], R.U8), ([LD(0), OP(R.OP_ORD2F)], R.F64),
        ([LD(1), OP(R.OP_NEG_F)], R.F64), ([LD(1), OP(R.OP_ABS_F)], R.F64), ([LD(1), OP(R.OP_SQRT_F)], R.F64),
        ([LD(1), OP(R.OP_F2I)], R.I64), ([LD(1), OP(R.OP_ISNULL_F)], R.U8), ([LD(1), OP(R.OP_ORD2F)], R.F64),
        ([LD(1), OP(R.OP_F2I), OP(R.OP_I2F)], R.F64),                       # LazySeries.trunc
        ([LD(0), CI(-5), OP(R.OP_FILLNA)], R.I64), ([LD(0), CN, OP(R.OP_FILLNA)], R.I64),
        ([LD(1), CF(-0.0), OP(R.OP_FILLNA)], R.F64), ([CN, CI(1), OP(R.OP_ADD_I)], R.I64),
        ([LD(1), CF(math.nan), OP(R.OP_EQ_F + R.NE)], R.U8), ([LD(0), OP(R.OP_I2F), CF(2.0 ** 53), OP(R.OP_EQ_F)], R.U8),
    ]
    for code, out in cases:
        check_prog(code, out, [ci, cf], n, f"program {code}")


@pytest.mark.parametrize("nulls", [False, True], ids=["valid", "nulls"])
def test_expr_kleene_logic_case_and_not(nulls):
    """AND / OR over all 3x3 (true, false, NULL) pairs, NOT, and CASE whose condition is NULL"""
    n = 9 * 61
    k = np.arange(n) % 9
    a_null, b_null = k // 3 == 2, k % 3 == 2
    a = _column(k // 3 == 0, R.U8, a_null)
    b = _column(k % 3 == 0, R.U8, b_null)
    x = _column(np.arange(n) * 7 - 100, R.I64, _null_pattern(n, 5, 3) if nulls else None)
    y = _column(np.linspace(-3, 3, n), R.F64, _null_pattern(n, 6, 0) if nulls else None)
    cols = [a, b, x, y]
    for code, out in [
        ([LD(0), LD(1), OP(R.OP_AND)], R.U8), ([LD(0), LD(1), OP(R.OP_OR)], R.U8),
        ([LD(0), OP(R.OP_NOT)], R.U8), ([LD(0), LD(1), OP(R.OP_AND), OP(R.OP_NOT)], R.U8),
        ([LD(0), LD(2), LD(2), OP(R.OP_NEG_I), OP(R.OP_CASE)], R.I64),
        ([LD(0), LD(3), CF(-0.0), OP(R.OP_CASE)], R.F64),
        ([LD(1), CN, LD(2), OP(R.OP_CASE)], R.I64),
        ([LD(0), LD(1), OP(R.OP_OR), LD(3), CN, OP(R.OP_CASE)], R.F64),
        ([CN, CI(1), CI(2), OP(R.OP_CASE)], R.I64),
        ([LD(3), OP(R.OP_ISNULL_F), LD(2), OP(R.OP_ISNULL_I), OP(R.OP_OR)], R.U8),
    ]:
        check_prog(code, out, cols, n, f"program {code}")


@pytest.mark.parametrize("n", [0] + SIZES)
def test_expr_shapes_and_a_depth_16_program(n):
    """row counts around every warp / batch / tile boundary; a program that fills the 16-deep stack"""
    rng = np.random.default_rng(n)
    cols = [_column(rng.choice(INT_POOL, n) if n else [], R.I64, rng.random(n) < 0.1),
            _column(rng.integers(-1000, 1000, n), R.I64),
            _column(rng.choice(FLOAT_POOL, n) if n else [], R.F64, rng.random(n) < 0.1)]
    deep = [LD(0), LD(1), CI(3), LD(1), CI(-7), LD(0), LD(1), CI(11), LD(0), LD(1), CI(5), LD(1), CI(-2),
            LD(0), LD(1), CI(13)]
    ops = [R.OP_ADD_I, R.OP_MUL_I, R.OP_SUB_I, R.OP_MOD_I, R.OP_DIV_I] * 3
    deep += [OP(o) for o in ops]
    assert len(deep) == 31
    check_prog(deep, R.I64, cols, n, "depth 16")
    check_prog([LD(2), LD(0), OP(R.OP_I2F), OP(R.OP_MUL_F), LD(1), OP(R.OP_I2F), OP(R.OP_ADD_F)], R.F64, cols, n,
               "mixed")
    check_prog([LD(0), LD(1), OP(R.OP_EQ_I + R.GT), LD(2), CF(0.0), OP(R.OP_EQ_F + R.LE), OP(R.OP_OR)], R.U8,
               cols, n, "predicate")


def test_expr_programs_of_the_host_compiler():
    """programs built by expr.compile_expr: casts to U8, fillna on floats through CASE, int % literal, an
    int column compared with a float literal, trunc (F2I then I2F)"""
    from dask_sql_b200 import expr as E
    rng = np.random.default_rng(5)
    n = 4099
    ci = _column(rng.choice(INT_POOL, n), R.I64, rng.random(n) < 0.15)
    cf = _column(rng.choice(FLOAT_POOL, n), R.F64, rng.random(n) < 0.15)
    cb = _column(rng.integers(0, 2, n), R.U8, rng.random(n) < 0.15)
    i, f, b = E.ColRef("i", R.I64), E.ColRef("f", R.F64), E.ColRef("b", R.U8)
    exprs = [E.cast(i, R.U8), E.cast(f, R.U8), E.fillna(f, 2.5), E.fillna(i, -1), E.binop("mod", i, 3),
             E.binop("mod", i, -3), E.binop("mod", -7, i), E.binop("eq", i, 2.0 ** 53), E.binop("lt", i, 0.5),
             E.cast(E.cast(f, R.I64), R.F64), E.case(E.binop("gt", f, 0), i, None), E.unop("isnull", f),
             E.binop("or", b, E.binop("ge", f, 1.5)), E.binop("and", b, E.unop("isnull", i)),
             E.binop("divt", i, -2), E.binop("truediv", i, f), E.unop("abs", f), E.unop("neg", i)]
    for e in exprs:
        p = E.compile_expr(e, ["i", "f", "b"])
        check_prog(R.prog_code(p), p.out_dtype, [ci, cf, cb], n, repr(e))


def test_expr_rejects_malformed_programs():
    L = _L()
    col = _column([1, 2, 3], R.I64)
    for code in ([OP(R.OP_ADD_I)], [LD(0), LD(0)], [LD(1)], [LD(0)] * 17 + [OP(R.OP_ADD_I)] * 16):
        with pytest.raises(L.B200SqlError):
            run_prog(code, R.I64, [col], 3)


# ---- predicate terms -------------------------------------------------------------------------------------
def make_scan(devs, terms, n):
    """terms: [(col, op, as_f64, lit_i, lit_f)] as in R.eval_terms"""
    L = _L()
    s = L.Scan()
    s.ncols, s.nterms, s.n = len(devs), len(terms), n
    for i, d in enumerate(devs):
        s.cols[i] = d.struct()
    for i, (c, op, as_f64, lit_i, lit_f) in enumerate(terms):
        t = s.terms[i]
        t.col, t.op, t.as_f64, t.lit_i, t.lit_f = c, op, as_f64, lit_i, lit_f
    return s


def check_select(devs, terms, n, what):
    """b2_select_count + b2_select_write (row ids, every column gathered with its validity)"""
    import torch
    L = _L()
    cols = [d.col for d in devs]
    exp_rows = np.flatnonzero(R.eval_terms(cols, terms, n))
    scan = make_scan(devs, terms, n)
    ntiles = L.num_tiles(n)
    off = torch.empty(ntiles + 1, dtype=torch.int64, device=_dev())
    L.select_count(C.byref(scan), _ptr(off), _stream())
    off_h = off.cpu().numpy()
    total = int(off_h[-1])
    assert total == len(exp_rows), f"{what}: {total} rows pass, expected {len(exp_rows)}"
    k = len(devs)
    out_idx = torch.full((max(total, 1),), -7, dtype=torch.int32, device=_dev())
    outs = [torch.full((max(total, 1),), 0x5A, dtype=d.data.dtype, device=_dev()) for d in devs]
    vals = [torch.zeros(max((total + 31) // 32, 1), dtype=torch.int32, device=_dev()) for _ in devs]
    gcols = (C.c_int32 * k)(*range(k))
    odata = (C.c_void_p * k)(*[o.data_ptr() for o in outs])
    ovalid = (C.c_void_p * k)(*[v.data_ptr() for v in vals])
    L.select_write(C.byref(scan), _ptr(off), _ptr(out_idx), k, gcols, odata, ovalid, _stream())
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out_idx.cpu().numpy()[:total], exp_rows, err_msg=f"{what}: row ids")
    for d, o, v in zip(devs, outs, vals):
        got = o.cpu().numpy()[:total]
        exp = d.col.values[exp_rows]
        _assert_words(got.view(np.int64) if d.col.dtype != R.U8 else got,
                      exp.view(np.int64) if d.col.dtype != R.U8 else exp, f"{what}: gathered values")
        words = R.pack_valid(~d.col.null_mask()[exp_rows])
        np.testing.assert_array_equal(v.cpu().numpy().view(np.uint32)[: len(words)], words,
                                      err_msg=f"{what}: gathered validity")


def _agg_ops(dtype):
    L = _L()
    return (L.AGG_MIN, L.AGG_MAX) if dtype == R.F64 else (L.AGG_SUM, L.AGG_MAX)


def check_scan_agg(devs, terms, n, agg_cols, what):
    """b2_scan_agg: COUNT(*), then two exact aggregates (SUM / MIN / MAX) over each column of `agg_cols`"""
    import torch
    L = _L()
    cols = [d.col for d in devs]
    passing = R.eval_terms(cols, terms, n)
    specs = [(-1, L.AGG_COUNT)] + [(c, op) for c in agg_cols for op in _agg_ops(cols[c].dtype)]
    aggs = (L.Agg * len(specs))()
    for i, (c, op) in enumerate(specs):
        aggs[i].col, aggs[i].op = c, op
    acc = torch.full((len(specs),), 0x5A, dtype=torch.int64, device=_dev())
    cnt = torch.full((len(specs),), 0x5A, dtype=torch.int64, device=_dev())
    ws = torch.empty(L.scan_agg_ws_bytes(), dtype=torch.uint8, device=_dev())
    scan = make_scan(devs, terms, n)
    L.scan_agg(C.byref(scan), aggs, len(specs), _ptr(acc), _ptr(cnt), 0, _ptr(ws), _stream())
    got_acc, got_cnt = acc.cpu().numpy(), cnt.cpu().numpy()
    assert got_cnt[0] == passing.sum(), f"{what}: COUNT(*) {got_cnt[0]} vs {passing.sum()}"
    for i, (c, op) in enumerate(specs[1:], 1):
        col = cols[c]
        keep = passing & ~col.null_mask()[:n]
        raw = col.raw()[:n]
        if col.dtype == R.F64:
            keep &= ~np.isnan(col.values[:n])
            raw = R.ordered(raw)
        v = raw[keep]
        if op == L.AGG_SUM:
            exp = int(v.view(np.uint64).sum(dtype=np.uint64).view(np.int64))
        elif op == L.AGG_MIN:
            exp = int(v.min()) if len(v) else MAX
        else:
            exp = int(v.max()) if len(v) else MIN
        assert got_cnt[i] == keep.sum(), f"{what}: count of aggregate {i} (col {c})"
        assert got_acc[i] == exp, f"{what}: aggregate {i} (col {c}, op {op}) = {got_acc[i]}, expected {exp}"


def _term_column(dtype, nullable, n, rng):
    if dtype == R.I64:
        vals = np.resize(np.array(INT_POOL, np.int64), n)
        vals[len(INT_POOL):] = np.where(rng.random(n - len(INT_POOL)) < 0.5, vals[len(INT_POOL):],
                                        rng.integers(-2 ** 40, 2 ** 40, n - len(INT_POOL)))
    elif dtype == R.F64:
        vals = np.resize(np.array(FLOAT_POOL), n)
        vals[len(FLOAT_POOL):] = np.where(rng.random(n - len(FLOAT_POOL)) < 0.5, vals[len(FLOAT_POOL):],
                                          rng.normal(0, 1e6, n - len(FLOAT_POOL)))
    else:
        vals = rng.integers(0, 2, n)
    rng.shuffle(vals)
    return _column(vals, dtype, (rng.random(n) < 0.2) if nullable else None)


@pytest.mark.parametrize("nullable", [False, True], ids=["valid", "nulls"])
@pytest.mark.parametrize("dtype", [R.I64, R.F64, R.U8], ids=["i64", "f64", "u8"])
def test_terms_every_op_and_literal(dtype, nullable):
    """one term at a time: every operator x every literal of the pool x as_f64, checked through the
    selection and, with the term's column aggregated, through b2_scan_agg (n >= 4 x 2048: the staged
    instance takes its TMA path, plus a 37-row tail)"""
    rng = np.random.default_rng(10 * dtype + nullable)
    n = 8229
    other = _column(rng.integers(-100, 100, n), R.I64, (rng.random(n) < 0.3) if nullable else None)
    devs = [Dev(_term_column(dtype, nullable, n, rng)), Dev(other)]
    terms = [(0, R.IS_NULL, 0, 0, 0.0), (0, R.IS_NOT_NULL, 0, 0, 0.0)]
    if dtype == R.U8:
        terms.append((0, R.IS_TRUE, 0, 0, 0.0))
    for op in (R.EQ, R.NE, R.LT, R.LE, R.GT, R.GE):
        for as_f64 in (0, 1):
            if as_f64 or dtype == R.F64:
                terms += [(0, op, as_f64, 0, lit) for lit in FLOAT_POOL]
            else:
                terms += [(0, op, 0, lit, 0.0) for lit in INT_POOL]
    for t in terms:
        check_select(devs, [t], n, f"term {t}")
        check_scan_agg(devs, [t], n, [0, 1], f"term {t}")


def _random_terms(cols, k, rng):
    """k terms over the columns, literals drawn from the pools and from the columns' own values"""
    out = []
    for _ in range(k):
        c = int(rng.integers(0, len(cols)))
        col = cols[c]
        op = int(rng.choice([R.EQ, R.NE, R.LT, R.LE, R.GT, R.GE, R.NE, R.IS_NOT_NULL, R.IS_NULL]))
        if col.dtype == R.U8 and rng.random() < 0.5:
            op = R.IS_TRUE
        pick = col.values[int(rng.integers(0, col.n))] if col.n else 0
        if col.dtype == R.F64:
            lit = float(pick) if rng.random() < 0.6 else float(rng.choice(FLOAT_POOL))
            out.append((c, op, 0, 0, lit))
        elif rng.random() < 0.3:
            out.append((c, op, 1, 0, float(rng.choice(FLOAT_POOL)) if rng.random() < 0.5 else float(pick) + 0.5))
        else:
            out.append((c, op, 0, int(pick) if rng.random() < 0.7 else int(rng.choice(INT_POOL)), 0.0))
    return out


def _scan_columns(n, rng):
    return [_column(rng.integers(-50, 50, n), R.I64, rng.random(n) < 0.1),
            _column(np.where(rng.random(n) < 0.1, rng.choice(FLOAT_POOL, n), rng.normal(0, 30, n)), R.F64,
                    rng.random(n) < 0.05),
            _column(rng.integers(0, 2, n), R.U8, rng.random(n) < 0.1),
            _column(rng.integers(-50, 50, n), R.I64)]


@pytest.mark.parametrize("nterms", [0, 1, 2, 5, 8])
@pytest.mark.parametrize("n", [0] + SIZES)
def test_terms_conjunctions_select(n, nterms):
    rng = np.random.default_rng(1000 * nterms + n)
    cols = _scan_columns(n, rng)
    devs = [Dev(c) for c in cols]
    for rep in range(3):
        terms = _random_terms(cols, nterms, rng)
        check_select(devs, terms, n, f"n={n} terms={terms}")


@pytest.mark.parametrize("nterms", [1, 2, 5, 8])
@pytest.mark.parametrize("n", [0] + SIZES)
def test_terms_conjunctions_scan_agg(n, nterms):
    """COUNT(*) and exact aggregates over the LAST term's column (whose values b2_scan_agg_body reuses from
    the predicate's registers) and over an EARLIER term's column (re-loaded).  At n >= 8192 the staged
    instance (B200SQL_PIPELINE=1, tests/test_gpu_pipeline.py) takes its TMA path."""
    rng = np.random.default_rng(2000 * nterms + n)
    cols = _scan_columns(n, rng)
    devs = [Dev(c) for c in cols]
    for rep in range(3):
        terms = _random_terms(cols, nterms, rng)
        last = terms[-1][0]
        earlier = terms[0][0] if terms[0][0] != last else (last + 1) % len(cols)
        check_scan_agg(devs, terms, n, [last, earlier], f"n={n} terms={terms}")


# ---- b2_sort_by --------------------------------------------------------------------------------------------
def _sort_column(dtype, n, rng):
    null = rng.random(n) < 0.07
    if dtype == R.I64:   # few distinct values: stability decides most of the order
        vals = rng.choice(np.array([MIN, MIN + 1, -2 ** 53, -1, 0, 1, 2 ** 53, 2 ** 53 + 1, MAX - 1, MAX], np.int64), n)
    elif dtype == R.U8:
        vals = rng.integers(0, 2, n)
    else:                # ±0.0 interleaved (they tie), ±inf, subnormals, NaN next to bitmap NULLs
        vals = rng.choice(np.array([0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, math.nan, 1.5, -1.5,
                                    1.7976931348623157e308, -2.5]), n)
    return _column(vals, dtype, null)


def run_sort(col, idx, descending, nulls_first):
    import torch
    L = _L()
    n = len(idx)
    d = Dev(col)
    t = torch.from_numpy(np.asarray(idx, np.int32).copy()).to(_dev())
    ws = torch.empty(max(L.sort_ws_bytes(n), 1), dtype=torch.uint8, device=_dev())
    st = d.struct()
    L.sort_by(C.byref(st), n, descending, nulls_first, _ptr(t) if n else C.c_void_p(ws.data_ptr()), _ptr(ws),
              _stream())
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.mark.parametrize("direction", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["asc_nl", "asc_nf", "desc_nl", "desc_nf"])
@pytest.mark.parametrize("dtype", [R.I64, R.U8, R.F64], ids=["i64", "u8", "f64"])
@pytest.mark.parametrize("n", [0, 1, 2, 33, 513, 4097, 16383, 16384, 16385, 100_003])
def test_sort_by_is_the_stable_permutation(n, dtype, direction):
    desc, nf = direction
    rng = np.random.default_rng(n + 7 * dtype)
    col = _sort_column(dtype, n, rng)
    for idx in (np.arange(n), rng.permutation(n)):      # identity and a non-identity input permutation
        got = run_sort(col, idx, desc, nf)
        exp = R.sort_perm(col, idx, desc, nf)
        bad = np.flatnonzero(got != exp)
        assert not len(bad), f"first difference at {bad[0]}: row {got[bad[0]]} vs {exp[bad[0]]}"


@pytest.mark.parametrize("n", [33, 16385, 100_003])
def test_sort_by_two_keys(n):
    """ORDER BY a DESC NULLS LAST, f ASC NULLS FIRST: the last key first, then the first key"""
    rng = np.random.default_rng(n)
    a, f = _sort_column(R.I64, n, rng), _sort_column(R.F64, n, rng)
    idx = rng.permutation(n).astype(np.int32)
    got = run_sort(a, run_sort(f, idx, 0, 1), 1, 0)
    exp = R.sort_perm(a, R.sort_perm(f, idx, 0, 1), 1, 0)
    np.testing.assert_array_equal(got, exp)


# ---- b2_gather ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [R.I64, R.F64, R.U8], ids=["i64", "f64", "u8"])
@pytest.mark.parametrize("n", [0, 1, 31, 33, 4097, 100_003])
def test_gather(dtype, n):
    """indices that are -1, repeated and out of order; the F64 fill is NaN; validity words exact"""
    import torch
    L = _L()
    rng = np.random.default_rng(n + dtype)
    m = 777
    src = _column(rng.choice(INT_POOL, m) if dtype == R.I64 else
                  (rng.choice(FLOAT_POOL, m) if dtype == R.F64 else rng.integers(0, 2, m)), dtype, rng.random(m) < 0.2)
    idx = rng.integers(-1, m, n).astype(np.int32)
    idx[rng.random(n) < 0.1] = -1
    d = Dev(src)
    t = torch.from_numpy(idx).to(_dev())
    out = torch.full((max(n, 1),), 0x5A, dtype=d.data.dtype, device=_dev())
    valid = torch.full((max((n + 31) // 32, 1),), -1, dtype=torch.int32, device=_dev())
    st = d.struct()
    L.gather(C.byref(st), _ptr(t), n, _ptr(out), _ptr(valid), _stream())
    torch.cuda.synchronize()
    exp, exp_valid = R.gather(src, idx)
    got = out.cpu().numpy()[:n]
    if dtype == R.U8:
        np.testing.assert_array_equal(got, exp)
    else:
        np.testing.assert_array_equal(got.view(np.int64), exp.view(np.int64))   # exact bits, NaN fill included
    words = R.pack_valid(exp_valid)
    np.testing.assert_array_equal(valid.cpu().numpy().view(np.uint32)[: len(words)], words)


# ---- b2_col_stats ------------------------------------------------------------------------------------------
def _stats_cases():
    rng = np.random.default_rng(9)
    yield "all_null_i64", _column([5, 6, 7], R.I64, np.ones(3, bool))
    yield "all_null_f64", _column([1.0, math.nan], R.F64, np.ones(2, bool))
    yield "all_nan", _column([math.nan] * 40, R.F64)
    yield "single_row", _column([-3], R.I64)
    yield "single_nan", _column([math.nan], R.F64)
    yield "zeros_only", _column([0.0, -0.0] * 20, R.F64)
    yield "neg_zero_only", _column([-0.0] * 33, R.F64)
    yield "pos_zero_and_null", _column([0.0, -0.0, 0.0], R.F64, np.array([False, True, False]))
    yield "infinities", _column([math.inf, -math.inf, 1.0, math.nan], R.F64)
    yield "subnormals", _column([5e-324, -5e-324, 0.0], R.F64)
    yield "int64_extremes", _column([MIN, MAX, 0, MIN + 1], R.I64)
    yield "int64_max_only", _column([MAX] * 5, R.I64)
    yield "int64_min_only", _column([MIN] * 5, R.I64, np.array([True, False, False, False, True]))
    yield "bool", _column([1, 0, 1], R.U8, np.array([False, True, False]))
    yield "empty_i64", _column([], R.I64)
    yield "empty_f64", _column([], R.F64)
    for n in (31, 32, 33, 511, 513, 4097, 16385, 100_003):
        yield f"i64_{n}", _column(rng.choice(INT_POOL, n), R.I64, rng.random(n) < 0.1)
        yield f"f64_{n}", _column(rng.choice(FLOAT_POOL, n), R.F64, rng.random(n) < 0.1)


@pytest.mark.parametrize("case", list(_stats_cases()), ids=lambda c: c[0])
def test_col_stats(case):
    import torch
    L = _L()
    name, col = case
    d = Dev(col)
    out = torch.full((6,), 0x5A, dtype=torch.int64, device=_dev())
    ws = torch.empty(L.stats_ws_bytes(), dtype=torch.uint8, device=_dev())
    st = d.struct()
    L.col_stats(C.byref(st), col.n, _ptr(out), _ptr(ws), _stream())
    mn, mx, nulls, nans, rep, sampled = out.cpu().tolist()
    exp = R.col_stats(col)
    assert {"min": mn, "max": mx, "null_count": nulls, "n_nan": nans} == exp, name
    assert 0 <= rep <= sampled <= col.n, (rep, sampled)
