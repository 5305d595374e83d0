"""b2_join_mark through the C-ABI against tests/mark_ref.py, row for row and validity bit for validity bit:
chained, direct-address and key-ordered (presence bitmap) tables; NULL and NaN keys and an empty build; one key
with 10^5 candidates; all six comparisons on int64 extremes and on +-0.0 / +-inf; row counts that are not
multiples of 32; rows that fail the scan's terms; and the B2_ERR_ARG cases."""
import ctypes as C

import numpy as np
import pytest

from tests import mark_ref as M

pytestmark = pytest.mark.gpu

MIN, MAX = -(1 << 63), (1 << 63) - 1
SIZES = [0, 1, 31, 33, 4097, 70_001]


def _mods():
    import torch
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    return torch, L, D


def _col(vals, valid=None):
    torch, L, D = _mods()
    vals = np.ascontiguousarray(vals)
    dt = L.F64 if vals.dtype.kind == "f" else L.I64
    data = torch.from_numpy(vals).to("cuda")
    words = None
    if valid is not None:
        b = np.packbits(np.asarray(valid, bool), bitorder="little")
        b = np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)])
        words = torch.from_numpy(b.view(np.int32).copy()).to("cuda")
    return D.DeviceColumn(data, words, dt)


def _table(bkeys, kind):
    """kind: chained | direct | bitmap"""
    torch, L, D = _mods()
    jt = D.JoinTable(bkeys, allow_dense=kind != "chained")
    if kind != "chained":
        assert jt.dense, "the test's keys must be unique and dense for a direct-address table"
        if kind == "bitmap":
            jt.key_layout([])
    return jt


def _run(pkeys, bkeys, kind="chained", terms=(), null_aware=False, passes=None):
    """pkeys / bkeys / terms as mark_ref takes them; passes: a scan term `filter column != 0`."""
    torch, L, D = _mods()
    pcols = [_col(v, ok) for v, ok in pkeys]
    bcols = [_col(v, ok) for v, ok in bkeys]
    jt = _table(bcols, kind)
    cols = list(pcols)
    mt = []
    for t in terms:
        cols.append(_col(*t[0]))
        cmp = M.CMP_CODE[t[2]] | (L.MARK_WHERE if len(t) > 3 and t[3] else 0)
        mt.append((len(cols) - 1, _col(*t[1]), cmp))
    scan_terms = []
    if passes is not None:
        cols.append(_col(np.asarray(passes, np.int64)))
        scan_terms.append(D.TermSpec(len(cols) - 1, L.NE, 0))
    n = len(pkeys[0][0])
    flags = 0
    if null_aware:
        m = len(bkeys[0][0])
        flags = L.MARK_NULL_AWARE | (L.MARK_BUILD_NONEMPTY if m else 0)
        if m and not M._valid(bkeys[0]).all():
            flags |= L.MARK_BUILD_HAS_NULL
    scan = D.make_scan(cols, scan_terms, n)
    got = D.join_mark(scan, list(range(len(pcols))), jt, mt, flags, torch.device("cuda"))
    torch.cuda.synchronize()
    out = got.data.cpu().numpy()
    words = got.valid.cpu().numpy().view(np.uint32)
    valid = np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)
    # bits past the last row are zero
    assert not np.unpackbits(words.view(np.uint8), bitorder="little")[n:].any()
    want_out, want_valid = M.mark(pkeys, bkeys, terms, null_aware, passes)
    np.testing.assert_array_equal(valid, want_valid)
    np.testing.assert_array_equal(out, want_out)
    return want_out, want_valid


def _ints(rng, n, lo, hi, nulls):
    return rng.integers(lo, hi, n).astype(np.int64), rng.random(n) >= nulls


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("null_aware", [False, True])
def test_chained_keys_with_nulls(n, null_aware):
    rng = np.random.default_rng(n)
    p = _ints(rng, n, 0, 50, 0.1)
    b = _ints(rng, 300, 0, 40, 0.05)
    _run([p], [b], "chained", null_aware=null_aware)


@pytest.mark.parametrize("kind", ["direct", "bitmap"])
@pytest.mark.parametrize("n", SIZES)
def test_direct_and_bitmap_tables(kind, n):
    rng = np.random.default_rng(7 + n)
    b = (rng.permutation(1000).astype(np.int64)[:600], None)
    p = _ints(rng, n, -10, 1010, 0.1)
    _run([p], [b], kind, null_aware=True)
    _run([p], [b], kind)


def test_duplicate_build_keys_without_terms_and_multi_keys():
    rng = np.random.default_rng(3)
    p = [_ints(rng, 5000, 0, 30, 0.05), _ints(rng, 5000, 0, 4, 0.05)]
    b = [_ints(rng, 2000, 0, 30, 0.05), _ints(rng, 2000, 0, 4, 0.05)]
    _run(p, b, "chained")
    _run(p, b, "chained", terms=[(_ints(rng, 5000, 0, 9, 0.1), _ints(rng, 2000, 0, 9, 0.1), "<", True)])


def test_float_keys_nan_signed_zero_and_empty_build():
    p = (np.array([0.0, -0.0, np.nan, 2.0, np.inf, -np.inf, 3.0] * 9), None)
    b = (np.array([-0.0, np.nan, np.inf, 2.0]), None)
    _run([p], [b], null_aware=True)
    _run([p], [b])
    empty = (np.zeros(0), None)
    _run([p], [empty], null_aware=True)
    _run([p], [empty], terms=[(p, empty, "=")])


def test_one_key_with_many_candidates():
    n, m = 777, 100_000
    rng = np.random.default_rng(11)
    p = (np.zeros(n, np.int64), rng.random(n) > 0.05)
    b = (np.zeros(m, np.int64), None)
    pv = _ints(rng, n, 0, 2 * m, 0.0)
    bv = (np.arange(m, dtype=np.int64) * 2, rng.random(m) > 0.001)
    _run([p], [b], terms=[(pv, bv, "=")])                  # TRUE found late in the chain, or NULL / FALSE
    _run([p], [b], terms=[(pv, bv, ">", True)])


@pytest.mark.parametrize("cmp", list(M.CMPS))
@pytest.mark.parametrize("where", [False, True])
def test_comparisons_at_int64_and_ieee_edges(cmp, where):
    ints = np.array([MIN, MAX, MIN + 1, MAX - 1, 0, -1, 1], np.int64)
    floats = np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -2.25, np.nan])
    for vals in (ints, floats):
        k = len(vals)
        pv, bv = np.repeat(vals, k), np.tile(vals, k)
        pvalid = np.ones(k * k, bool)
        pvalid[::5] = False
        key = (np.repeat(np.arange(k * k, dtype=np.int64), 1), None)
        _run([key], [key], "direct", terms=[((pv, pvalid), (bv, None), cmp, where)])
        _run([key], [key], "chained", terms=[((pv, None), (bv, pvalid), cmp, where)])


def test_rows_that_fail_the_scan_terms_are_false():
    rng = np.random.default_rng(5)
    n = 1000
    p = _ints(rng, n, 0, 20, 0.1)
    b = _ints(rng, 50, 0, 20, 0.1)
    passes = rng.random(n) > 0.3
    out, valid = _run([p], [b], null_aware=True, passes=passes)
    assert not out[~passes].any() and valid[~passes].all()


def test_argument_errors():
    torch, L, D = _mods()
    k = _col(np.arange(64, dtype=np.int64))
    f = _col(np.arange(64, dtype=np.float64))
    jt = _table([k], "direct")
    bitmap = _table([k], "bitmap")
    chained = _table([k, k], "chained")
    out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    valid = torch.zeros(2, dtype=torch.int32, device="cuda")
    scan = D.make_scan([k, f], [], 64)

    def call(table, terms=(), flags=0, keys=(0,), ntrms=None):
        mt = (L.MarkTerm * max(1, len(terms)))()
        for i, (slot, col, cmp) in enumerate(terms):
            mt[i].probe_col, mt[i].build, mt[i].cmp = slot, col.as_struct(), cmp
        pk = (C.c_int32 * len(keys))(*keys)
        return L._lib.b2_join_mark(C.byref(scan), pk, C.byref(table.struct), mt,
                                   len(terms) if ntrms is None else ntrms, flags, D.ptr(out), D.ptr(valid),
                                   D.stream_ptr())

    assert call(jt) == 0
    assert call(bitmap, [(0, k, L.EQ)]) == -2             # pair terms need every candidate
    assert call(jt, [(1, k, L.EQ)]) == -2                 # float64 probe side, int64 build side
    assert call(jt, [(0, k, 6)]) == -2                    # no such comparison
    assert call(jt, [(2, k, L.EQ)]) == -2                 # probe column out of range
    assert call(jt, [(0, k, L.EQ)] * 5) == -2             # more than B2_MARK_MAX_TERMS
    assert call(jt, ntrms=-1) == -2
    assert call(jt, flags=16) == -2                       # unknown flag
    assert call(chained, flags=L.MARK_NULL_AWARE, keys=(0, 0)) == -2   # a NULL-aware mark has one key
    assert call(jt, keys=(1,)) == -2                      # key types differ
    torch.cuda.synchronize()
