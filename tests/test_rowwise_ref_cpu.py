"""The NumPy reference of the row-wise kernels (tests/rowwise_ref.py) against hand-computed rows, so that
the oracle of tests/test_gpu_rowwise.py is itself checked on a machine without a GPU."""
import numpy as np

from tests import rowwise_ref as R

MIN, MAX = R.INT64_MIN, R.INT64_MAX
NAN = float("nan")


def _i64(*v):
    return R.Column(np.array(v, np.int64), None, R.I64)


def _binary(op, a, b):
    """op on two int64 columns -> list of python ints, None for NULL"""
    out, valid = R.eval_prog([(R.OP_LOAD, 0, 0, 0.0), (R.OP_LOAD, 1, 0, 0.0), (op, 0, 0, 0.0)], R.I64,
                             [_i64(*a), _i64(*b)], len(a))
    return [int(v) if ok else None for v, ok in zip(out, valid)]


def test_modulo_is_floored_and_zero_divisor_is_null():
    a = [-7, 7, 7, -7, 6, -6, 5, MIN, MIN, MAX, MIN, 0]
    b = [3, -3, 3, -3, 3, 3, 0, -1, 3, -2, MAX, -5]
    assert _binary(R.OP_MOD_I, a, b) == [2, -2, 1, -1, 0, 0, None, 0, 1, -1, MAX - 1, 0]
    assert [x % y if y else None for x, y in zip(a, b)] == _binary(R.OP_MOD_I, a, b)   # Python's % agrees


def test_division_truncates_and_wraps():
    a = [-7, 7, -7, 7, MIN, MIN, 5, MAX, MIN]
    b = [2, -2, -2, 2, -1, 1, 0, -1, 3]
    assert _binary(R.OP_DIV_I, a, b) == [-3, -3, 3, 3, MIN, MIN, None, -MAX, -3074457345618258602]


def test_int_arithmetic_wraps():
    assert _binary(R.OP_ADD_I, [MAX, MIN], [1, -1]) == [MIN, MAX]
    assert _binary(R.OP_SUB_I, [MIN], [1]) == [MAX]
    assert _binary(R.OP_MUL_I, [1 << 62, MIN, 3], [4, -1, -5]) == [0, MIN, -15]


def test_kleene_truth_tables():
    vals = [True, False, None]
    a = [x for x in vals for _ in vals]
    b = [y for _ in vals for y in vals]
    cols = [R.Column(np.array([bool(v) for v in c], np.uint8), np.array([v is None for v in c]), R.U8)
            for c in (a, b)]
    for op, expect in ((R.OP_AND, [True, False, None, False, False, False, None, False, None]),
                       (R.OP_OR, [True, True, True, True, False, None, True, None, None])):
        out, valid = R.eval_prog([(R.OP_LOAD, 0, 0, 0.0), (R.OP_LOAD, 1, 0, 0.0), (op, 0, 0, 0.0)], R.U8, cols, 9)
        assert [bool(v) if ok else None for v, ok in zip(out, valid)] == expect, op


def test_case_with_null_condition_takes_else_and_fillna():
    cond = R.Column(np.array([1, 0, 1], np.uint8), np.array([False, False, True]), R.U8)
    code = [(R.OP_LOAD, 0, 0, 0.0), (R.OP_CONST_I, 0, 10, 0.0), (R.OP_CONST_I, 0, 20, 0.0), (R.OP_CASE, 0, 0, 0.0)]
    out, valid = R.eval_prog(code, R.I64, [cond], 3)
    assert out.tolist() == [10, 20, 20] and valid.all()
    x = R.Column(np.array([5, 6], np.int64), np.array([True, False]), R.I64)
    out, valid = R.eval_prog([(R.OP_LOAD, 0, 0, 0.0), (R.OP_CONST_NULL, 0, 0, 0.0), (R.OP_FILLNA, 0, 0, 0.0)],
                             R.I64, [x], 2)
    assert out.tolist() == [0, 6] and valid.tolist() == [False, True]      # NULL rows are written as 0


def test_float_to_int_saturates_and_nan_is_null():
    x = R.Column(np.array([1.9, -1.9, np.inf, -np.inf, NAN, 2.0 ** 63, -(2.0 ** 63), 1e300, -0.0]), None, R.F64)
    out, valid = R.eval_prog([(R.OP_LOAD, 0, 0, 0.0), (R.OP_F2I, 0, 0, 0.0)], R.I64, [x], 9)
    assert out.tolist() == [1, -1, MAX, MIN, 0, MAX, MIN, MAX, 0]
    assert valid.tolist() == [True] * 4 + [False] + [True] * 4


def test_negative_zero_and_nan_handling():
    z = R.Column(np.array([0.0, -0.0, NAN, 1.5]), None, R.F64)
    out, _ = R.eval_prog([(R.OP_LOAD, 0, 0, 0.0), (R.OP_NEG_F, 0, 0, 0.0)], R.F64, [z], 4)
    assert np.signbit(R.bits2f(out)).tolist()[:2] == [True, False]
    out, valid = R.eval_prog([(R.OP_LOAD, 0, 0, 0.0), (R.OP_ISNULL_F, 0, 0, 0.0)], R.U8, [z], 4)
    assert out.tolist() == [0, 0, 1, 0] and valid.all()
    # ORD2F is the order-preserving image, an involution that puts -0.0 just below +0.0
    assert R.ordered(R.f2bits(-0.0)) == -1 and R.ordered(R.f2bits(0.0)) == 0
    assert R.ordered(R.ordered(R.f2bits(-2.5))) == R.f2bits(-2.5)
    st = R.col_stats(R.Column(np.array([0.0, -0.0, NAN, 0.0]), np.array([False, False, False, True]), R.F64))
    assert st == {"min": int(R.f2bits(-0.0)), "max": 0, "null_count": 1, "n_nan": 1}
    # -0.0 ties with 0.0 and keeps its place; NaN sorts with the NULLs
    col = R.Column(np.array([0.0, -0.0, NAN, -1.0, 0.0, -0.0]), np.array([False] * 5 + [True]), R.F64)
    assert R.sort_perm(col, np.arange(6), 0, 0).tolist() == [3, 0, 1, 4, 2, 5]
    assert R.sort_perm(col, np.arange(6), 1, 1).tolist() == [2, 5, 0, 1, 4, 3]


def test_terms_compare_like_numpy():
    f = R.Column(np.array([NAN, 1.0, -np.inf]), None, R.F64)
    assert [R.eval_term(f, op, lit_f=1.0).tolist() for op in (R.EQ, R.NE, R.LT, R.GE)] == \
        [[False, True, False], [True, False, True], [False, False, True], [False, True, False]]
    assert R.eval_term(f, R.IS_NULL).tolist() == [True, False, False]
    # an int64 column against 2^53 in float64: 2^53 + 1 rounds to 2^53 and is equal
    x = R.Column(np.array([2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1], np.int64), np.array([False, False, True]), R.I64)
    assert R.eval_term(x, R.EQ, as_f64=1, lit_f=2.0 ** 53).tolist() == [False, True, False]   # NULL fails
    assert R.eval_term(x, R.EQ, lit_i=2 ** 53).tolist() == [False, True, False]
    assert R.eval_term(x, R.IS_NULL).tolist() == [False, False, True]


def test_gather_and_bitmaps():
    col = R.Column(np.array([1.5, 2.5, 3.5]), np.array([False, True, False]), R.F64)
    out, valid = R.gather(col, [2, -1, 1, 2])
    assert R.f2bits(out).tolist()[0] == R.f2bits(3.5) and np.isnan(out[1]) and valid.tolist() == [True, False, False, True]
    w = R.pack_valid(np.array([True] * 33))
    assert w.tolist() == [0xFFFFFFFF, 1]


# ---- the host side of the same semantics: scalar folding and how a literal becomes a kernel term -------
def test_scalar_modulo_fold_is_floored_and_null_on_zero():
    from dask_sql_b200.physical.rex.core.call import OPERATORS
    mod = OPERATORS["%"]
    assert [mod([a, b], None) for a, b in ((-7, 3), (7, -3), (7, 3), (-7, -3))] == [2, -2, 1, -1]
    assert mod([7, 0], None) is None and mod([None, 3], None) is None


def test_int_column_vs_float_literal_term_is_exact_only_below_2_53():
    import torch
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    from dask_sql_b200 import expr as E

    x = E.ColRef("x", R.I64)
    col = D.DeviceColumn(torch.zeros(4, dtype=torch.int64), None, R.I64)
    for lit, exact in ((2.0 ** 53 - 1, True), (-(2.0 ** 53 - 1), True), (2.0 ** 53, False), (-(2.0 ** 53), False),
                       (2.0 ** 62, False), (2.0 ** 63, False), (0.5, False), (float("inf"), False)):
        name, op, v = E.as_term(E.binop("eq", x, lit))
        assert name == "x" and op == L.EQ and isinstance(v, int) == exact, lit
        tm = D.make_scan([col], [D.TermSpec(0, op, v)]).terms[0]
        assert tm.as_f64 == (0 if exact else 1), lit
        assert (tm.lit_i == int(lit)) if exact else (tm.lit_f == lit), lit
    # an int literal against an int column stays an exact int64 comparison at any magnitude
    tm = D.make_scan([col], [D.TermSpec(0, L.EQ, 2 ** 53 + 1)]).terms[0]
    assert tm.as_f64 == 0 and tm.lit_i == 2 ** 53 + 1


def test_parquet_pruning_compares_int_statistics_in_float64(tmp_path):
    """row-group pruning must not drop a group that the kernel's float64 comparison would pass"""
    import pyarrow as pa
    import pyarrow.parquet as pq
    from dask_sql_b200 import _lib as L
    from dask_sql_b200.table import ParquetTable

    path = str(tmp_path / "x.parquet")
    x = pa.array([2 ** 53 + 1, 2 ** 53 + 1, 5, 6], pa.int64())
    pq.write_table(pa.table({"x": x}), path, row_group_size=2)
    t = ParquetTable(path)
    assert t.surviving_groups([("x", L.EQ, 2.0 ** 53)]) == [0]       # float(2^53 + 1) == 2^53
    assert t.surviving_groups([("x", L.EQ, 2 ** 53)]) == []          # an int literal compares exactly
    assert t.surviving_groups([("x", L.LT, 2.0 ** 53)]) == [1]
