"""b2_sample_mask and the B2_OP_RAND_F / B2_OP_RAND_I opcodes of b2_expr_eval, word for word against the NumPy
restatement of the contract (tests/rand_ref.py), at row numbers that start anywhere in a group of four and near
the 2^32 carry of the Philox counter."""
import ctypes as C

import numpy as np
import pytest

from tests import rand_ref as RR

pytestmark = pytest.mark.gpu

OP_RAND_F, OP_RAND_I = 66, 67


def _lib():
    from dask_sql_b200 import _lib as L
    return L


def _run(code, out_dtype, cols, n, row_base):
    """(out, valid words) of the program `code` over the int64 / float64 numpy `cols`"""
    import torch
    from dask_sql_b200 import device as D
    L = _lib()
    p = L.Prog()
    p.n, p.out_dtype = len(code), out_dtype
    for i, (op, a, ii, ff) in enumerate(code):
        p.code[i].op, p.code[i].a, p.code[i].imm_i, p.code[i].imm_f = op, a, ii, ff
    keep = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in cols]
    arr = (L.Col * max(1, len(keep)))()
    for i, t in enumerate(keep):
        arr[i].data, arr[i].valid = t.data_ptr(), None
        arr[i].dtype = L.F64 if t.dtype == torch.float64 else L.I64
    out = torch.full((max(n, 1),), 0x5A5A, dtype=torch.int64, device="cuda")
    valid = torch.full((max((n + 31) // 32, 1),), -1, dtype=torch.int32, device="cuda")
    L.expr_eval_rows(C.byref(p), arr, len(keep), n, row_base, out.data_ptr(), valid.data_ptr(), D.stream_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy()[:n], valid.cpu().numpy().view(np.uint32)[: (n + 31) // 32]


def _mask(n, row_base, key, site, p, off=None):
    """the mask written `off` bytes into a guarded buffer (default: 1 for odd row_base, else 0)"""
    import torch
    from dask_sql_b200 import device as D
    L = _lib()
    off = (1 if row_base % 2 else 0) if off is None else off
    buf = torch.full((n + 8,), 0xEE, dtype=torch.uint8, device="cuda")
    L.sample_mask(n, row_base, key, site, RR.threshold(p), buf.data_ptr() + off, D.stream_ptr())
    torch.cuda.synchronize()
    h = buf.cpu().numpy()
    assert (h[:off] == 0xEE).all() and (h[off + n:] == 0xEE).all(), "b2_sample_mask wrote outside [0, n)"
    return h[off:off + n]


BASES = [0, 1, 2, 3, 4097, 2 ** 32 - 5, 2 ** 32 - 2, 2 ** 40 + 3]


@pytest.mark.parametrize("row_base", BASES)
@pytest.mark.parametrize("n", [1, 3, 5, 1023, 100_003])
@pytest.mark.parametrize("p", [0, 0.001, 10, 50, 99.9999, 100])
def test_sample_mask_matches_reference(n, row_base, p):
    key, site = RR.key_of(-7), 3
    got = _mask(n, row_base, key, site, p)
    assert set(np.unique(got)) <= {0, 1}
    want = RR.bernoulli_mask(np.arange(n, dtype=np.int64) + row_base, key, site, p)
    np.testing.assert_array_equal(got.astype(bool), want)


@pytest.mark.parametrize("off", [1, 2, 3])
@pytest.mark.parametrize("row_base", [0, 4, 2 ** 32])
def test_sample_mask_misaligned_output(row_base, off):
    """row_base on a group boundary but `out` not 4-byte aligned: the byte stores, not the 32-bit one"""
    n, key = 10_007, RR.key_of(5)
    got = _mask(n, row_base, key, 2, 40, off)
    want = RR.bernoulli_mask(np.arange(n, dtype=np.int64) + row_base, key, 2, 40)
    np.testing.assert_array_equal(got.astype(bool), want)


def test_sample_mask_is_independent_of_the_split():
    """one table cut into pieces at arbitrary offsets gives the same rows as one piece"""
    n, key = 200_001, 12345
    whole = _mask(n, 0, key, 1, 30)
    cuts = [0, 1, 6, 4099, 77_777, 150_002, n]
    pieces = np.concatenate([_mask(b - a, a, key, 1, 30) for a, b in zip(cuts, cuts[1:])])
    np.testing.assert_array_equal(whole, pieces)


def test_sample_mask_rejects_bad_arguments():
    L = _lib()
    with pytest.raises(L.B200SqlError):
        L.sample_mask(-1, 0, 1, 1, 5, None, None)
    with pytest.raises(L.B200SqlError):
        L.sample_mask(10, -4, 1, 1, 5, None, None)


def test_known_answer_vectors_on_the_device():
    """row r at call site s draws Philox(r lo, r hi, s, 0): the counters of two of Random123's vectors"""
    # counter (0, 0, 0, 0), key 0: w0 | w1 << 32 of the first vector
    got, _ = _run([(OP_RAND_F, 0, 0, 0.0)], _lib().F64, [], 1, 0)
    u = 0x6627e8d5 | 0xe169c58d << 32
    assert got.view(np.float64)[0] == (u >> 11) * 2.0 ** -53
    # the third vector's key, at rows across the 2^32 carry of the counter, against the NumPy restatement
    key = 0x299f31d0a4093822
    rows = np.arange(4, dtype=np.int64) + 2 ** 32 - 2
    got, _ = _run([(OP_RAND_F, 7, key, 0.0)], _lib().F64, [], 4, int(rows[0]))
    np.testing.assert_array_equal(got.view(np.float64), RR.rand(rows, key, 7))


@pytest.mark.parametrize("row_base", [0, 3, 2 ** 32 - 100, 2 ** 45])
def test_rand_inside_a_larger_program(row_base):
    """RAND(1) * 10 + x over an int64 column"""
    L = _lib()
    n = 5000
    x = np.random.default_rng(1).integers(-100, 100, n)
    key = RR.key_of(1)
    code = [(OP_RAND_F, 2, key, 0.0), (L.OP_CONST_F, 0, 0, 10.0), (L.OP_MUL_F, 0, 0, 0.0),
            (L.OP_LOAD, 0, 0, 0.0), (L.OP_I2F, 0, 0, 0.0), (L.OP_ADD_F, 0, 0, 0.0)]
    got, valid = _run(code, L.F64, [x], n, row_base)
    want = RR.rand(np.arange(n) + row_base, key, 2) * 10.0 + x.astype(np.float64)
    np.testing.assert_array_equal(got.view(np.float64), want)
    assert (valid[: n // 32] == 0xFFFFFFFF).all()


@pytest.mark.parametrize("h", [1, 3, 10, 1000, 2 ** 63 - 1])
def test_rand_integer_inside_a_larger_program(h):
    """RAND_INTEGER(h) = 3, and the plain value, at row numbers across the 2^32 carry"""
    L = _lib()
    n, row_base, key = 10_000, 2 ** 32 - 5000, RR.key_of(-3)
    got, _ = _run([(L.OP_CONST_I, 0, h, 0.0), (OP_RAND_I, 4, key, 0.0)], L.I64, [], n, row_base)
    want = RR.rand_integer(np.arange(n) + row_base, key, 4, h)
    np.testing.assert_array_equal(got, want)
    code = [(L.OP_CONST_I, 0, h, 0.0), (OP_RAND_I, 4, key, 0.0), (L.OP_CONST_I, 0, 3, 0.0), (L.OP_EQ_I, 0, 0, 0.0)]
    got, _ = _run(code, L.I64, [], n, row_base)
    np.testing.assert_array_equal(got != 0, want == 3)


def test_rand_integer_of_a_non_positive_bound_is_null():
    L = _lib()
    got, valid = _run([(L.OP_CONST_I, 0, 0, 0.0), (OP_RAND_I, 1, 5, 0.0)], L.I64, [], 40, 0)
    assert (got == 0).all() and valid[0] == 0 and valid[1] & 0xFF == 0


def test_programs_without_rand_ignore_row_base():
    L = _lib()
    x = np.arange(100, dtype=np.int64)
    a, _ = _run([(L.OP_LOAD, 0, 0, 0.0)], L.I64, [x], 100, 0)
    b, _ = _run([(L.OP_LOAD, 0, 0, 0.0)], L.I64, [x], 100, 12345)
    np.testing.assert_array_equal(a, b)
