"""b2_select_hist bin for bin against the NumPy reference of tests/select_ref.py, through the C-ABI: the edge
sets (INT64_MIN / MAX, +-inf, +-0.0, subnormals, NaN, all-equal, n = 1), NULL bitmaps, lengths that are not
multiples of 32, partition slices on bitmap word boundaries, nsel 1..8, bits 1..11 and the compacting pass;
then the driver's order statistics (executor.order_statistics) against np.partition."""
import ctypes as C

import numpy as np
import pytest

from tests import select_ref as R

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
SIZES = [1, 31, 33, 255, 1023, 1025, 4099, 100_003]


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


def _pack(valid):
    n = valid.shape[0]
    bits = np.packbits(valid, bitorder="little")
    out = np.zeros(-(-n // 32) * 4, np.uint8)
    out[:bits.shape[0]] = bits
    return out.view(np.int32)


class Col:
    def __init__(self, values, valid=None):
        import torch
        self.values, self.valid_np = values, valid
        self.data = torch.from_numpy(np.ascontiguousarray(values)).to(_dev())
        self.valid = None if valid is None else torch.from_numpy(_pack(valid)).to(_dev())

    def struct(self, lo=0, hi=None):
        L = _L()
        c = L.Col()
        c.data = self.data.data_ptr() + 8 * lo
        c.valid = 0 if self.valid is None else self.valid.data_ptr() + lo // 8
        c.dtype = L.F64 if self.values.dtype == np.float64 else L.I64
        return c


def _hist(col, prefixes, shift, bits, lo=0, hi=None, compact=False):
    import torch
    L = _L()
    hi = col.values.shape[0] if hi is None else hi
    sel = L.Select()
    sel.nsel, sel.shift, sel.bits = len(prefixes), shift, bits
    for k, p in enumerate(prefixes):
        sel.prefix[k] = int(p)
    h = torch.zeros(len(prefixes) << bits, dtype=torch.int64, device=_dev())
    out = torch.empty(max(hi - lo, 1), dtype=torch.int64, device=_dev()) if compact else None
    cnt = torch.zeros(1, dtype=torch.int64, device=_dev()) if compact else None
    cs = col.struct(lo, hi)
    L.select_hist(C.byref(cs), hi - lo, C.byref(sel), _ptr(h), _ptr(out), _ptr(cnt), _stream())
    res = h.cpu().numpy().view(np.uint64)
    if compact:
        return res, out[:int(cnt.item())].cpu().numpy()
    return res


def _ref_images(col, lo=0, hi=None):
    hi = col.values.shape[0] if hi is None else hi
    return R.images(col.values[lo:hi], None if col.valid_np is None else col.valid_np[lo:hi])


def _edge_columns():
    """(name, values, valid or None): numpy only, so that collecting the tests needs no device"""
    rng = np.random.default_rng(11)
    ints = np.array([I64_MIN, I64_MAX, 0, -1, 1, I64_MIN + 1, I64_MAX - 1, 1 << 40, -(1 << 40)], np.int64)
    flts = np.array([-np.inf, np.inf, -0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308, np.nan, 1.0, -1.0,
                     1e308, -1e308], np.float64)
    for n in SIZES:
        vi = rng.choice(ints, n)
        vf = rng.choice(flts, n)
        valid = rng.random(n) < 0.8
        yield f"i{n}", vi, None
        yield f"i{n}_null", vi, valid
        yield f"f{n}", vf, None
        yield f"f{n}_null", vf, valid
    yield "equal", np.full(777, 5, np.int64), None
    yield "sub", rng.random(999) * 1e-310, None


@pytest.mark.parametrize("name,values,valid", list(_edge_columns()), ids=[e[0] for e in _edge_columns()])
def test_first_pass_bin_for_bin(name, values, valid):
    col = Col(values, valid)
    u = _ref_images(col)
    # the whole image: 11 top bits over every row, then a prefix that keeps only some rows
    assert np.array_equal(_hist(col, [0], 53, 11), R.hist_pass(u, [0], 53, 11))
    prefixes = sorted({int(x) >> 40 for x in u[:3]}) or [0]
    assert np.array_equal(_hist(col, prefixes, 29, 11), R.hist_pass(u, prefixes, 29, 11))


@pytest.mark.parametrize("nsel", range(1, 9))
@pytest.mark.parametrize("bits", range(1, 12))
def test_nsel_and_bits(nsel, bits):
    rng = np.random.default_rng(nsel * 16 + bits)
    n = 20_011
    v = rng.integers(-(1 << 20), 1 << 20, n).astype(np.int64)
    valid = rng.random(n) < 0.9
    col = Col(v, valid)
    u = _ref_images(col)
    shift = 20 - bits if bits < 20 else 0
    hs = shift + bits
    pool = sorted({int(x) >> hs for x in u})
    prefixes = [pool[i % len(pool)] for i in rng.permutation(max(nsel, len(pool)))[:nsel]]
    prefixes = sorted(set(prefixes)) + [pool[0] ^ 1] * (nsel - len(set(prefixes)))   # unmatched extras
    assert np.array_equal(_hist(col, prefixes, shift, bits), R.hist_pass(u, prefixes, shift, bits))


def test_partition_slices_on_word_boundaries():
    rng = np.random.default_rng(3)
    n = 10_000
    col = Col(rng.standard_normal(n), rng.random(n) < 0.7)
    for lo, hi in [(0, 32), (32, 4096), (4096, 9999), (64, 65), (9984, 10_000)]:
        u = _ref_images(col, lo, hi)
        assert np.array_equal(_hist(col, [0], 53, 11, lo, hi), R.hist_pass(u, [0], 53, 11)), (lo, hi)


def test_compacting_pass_writes_exactly_the_matching_rows():
    rng = np.random.default_rng(5)
    n = 50_001
    for values in (rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64), rng.standard_normal(n)):
        values[::97] = values[1]            # a value that repeats, so a bucket holds duplicates
        valid = rng.random(n) < 0.85
        col = Col(values, valid)
        u = _ref_images(col)
        prefixes = sorted({int(u[0]) >> 53, int(u[-1]) >> 53})
        h, out = _hist(col, prefixes, 42, 11, compact=True)
        assert np.array_equal(h, R.hist_pass(u, prefixes, 42, 11))
        keep = np.isin(u >> np.uint64(53), np.array(prefixes, np.uint64))
        assert out.shape[0] == int(keep.sum())
        got = np.sort(R.images(out.view(values.dtype)))
        assert np.array_equal(got, np.sort(u[keep]))


def test_bad_arguments_are_refused():
    L = _L()
    col = Col(np.arange(10, dtype=np.int64))
    for nsel, shift, bits, prefix in ((0, 0, 8, 0), (9, 0, 8, 0), (1, 0, 12, 0), (1, 0, 0, 0), (1, 60, 8, 0),
                                      (1, 0, 8, 1 << 56)):
        with pytest.raises(L.B200SqlError):
            sel = L.Select()
            sel.nsel, sel.shift, sel.bits = nsel, shift, bits
            sel.prefix[0] = prefix
            cs = col.struct()
            L.select_hist(C.byref(cs), 10, C.byref(sel), _ptr(col.data), None, None, _stream())
    b = L.Col()
    b.data, b.dtype = col.data.data_ptr(), L.U8
    sel = L.Select()
    sel.nsel, sel.shift, sel.bits = 1, 53, 11
    with pytest.raises(L.B200SqlError):
        L.select_hist(C.byref(b), 10, C.byref(sel), _ptr(col.data), None, None, _stream())


def _driver(parts, ranks):
    """executor.order_statistics over device partitions of (values, valid) against the sorted images and
    np.partition; returns the number of compacting passes it ran"""
    from dask_sql_b200 import executor as X
    from dask_sql_b200.device import DeviceColumn
    L = _L()
    dt = L.F64 if parts[0][0].dtype == np.float64 else L.I64
    cols, imgs = [], []
    for values, valid in parts:
        c = Col(values, valid)
        cols.append(DeviceColumn(c.data, c.valid, dt))
        imgs.append(_ref_images(c))
    u = np.concatenate(imgs)
    before = {k: X.stats.get(k, 0) for k in ("select_passes", "select_compactions")}
    got = X.order_statistics(cols, dt, ranks, int(u.min()), int(u.max()), u.shape[0])
    assert X.stats["select_passes"] - before["select_passes"] == R.passes(int(u.min()), int(u.max()))
    want = np.sort(u)
    assert [got[k] for k in ranks] == [int(want[k]) for k in ranks]
    clean = np.concatenate([v if m is None else v[m] for v, m in parts])
    if clean.dtype == np.float64:
        clean = clean[~np.isnan(clean)]
    part = np.partition(clean, ranks)
    assert [X.select_value(got[k], dt) for k in ranks] == [part[k] for k in ranks]
    return X.stats.get("select_compactions", 0) - before["select_compactions"]


def _cases(rng, n):
    return {
        "uniform_i64": rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64),
        "20_bits": rng.integers(0, 1 << 20, n).astype(np.int64),
        "uniform_f64": rng.random(n),
        "mostly_one_value": np.where(rng.random(n) < 0.9, 7.0, rng.standard_normal(n)),
        "six_values": rng.integers(-3, 3, n).astype(np.int64),
    }


@pytest.mark.parametrize("seed", range(3))
def test_driver_matches_np_partition(seed):
    rng = np.random.default_rng(100 + seed)
    n = 300_000
    for name, values in _cases(rng, n).items():
        valid = rng.random(n) < 0.95
        if values.dtype == np.float64:
            values[rng.random(n) < 0.01] = np.nan
        bounds = [0, 32 * 1000, 32 * 4000, n]
        parts = [(values[a:b], valid[a:b]) for a, b in zip(bounds, bounds[1:])]
        m = int(sum(((~np.isnan(v)) if v.dtype == np.float64 else np.ones(v.shape, bool))[k].sum() for v, k in parts))
        ranks = sorted({0, m - 1, m // 4, m // 4 + 1, m // 2, (3 * m) // 4} | set(rng.integers(0, m, 2).tolist()))
        compactions = _driver(parts, ranks)
        if name in ("uniform_i64", "uniform_f64"):
            assert compactions == 1, name
        if name in ("mostly_one_value", "six_values", "20_bits"):
            assert compactions == 0, name


@pytest.mark.parametrize("n", [1, 2, 3, 31, 33])
def test_driver_small_columns(n):
    rng = np.random.default_rng(n)
    values = rng.standard_normal(n)
    _driver([(values, None)], sorted({0, n - 1, n // 2}))
    _driver([(np.full(n, -0.0), None)], [0, n - 1])
