"""B2_OP_DATEPART / B2_OP_ADDMONTHS through the C-ABI, bit for bit against tests/temporal_ref.py, on pools
of calendar edges in every unit, with NULL rows, at row counts around the warp / block / tile sizes."""
import numpy as np
import pytest

from tests import temporal_ref as R

pytestmark = pytest.mark.gpu

SIZES = [1, 31, 32, 33, 511, 512, 513, 4095, 4096, 4097]


def _pool(unit):
    per_day = R.tpd(unit)
    days = [np.datetime64(s, "D").astype(np.int64) for s in (
        "1970-01-01", "1969-12-31", "1600-02-28", "1600-02-29", "1900-02-28", "2000-02-28", "2000-02-29",
        "2100-02-28", "2400-02-28", "2400-02-29", "1999-12-31", "2000-01-01", "2004-12-31", "2005-01-01",
        "2010-01-03", "2015-12-31", "2016-01-03", "2020-12-31", "2021-01-03", "2000-01-31", "1996-02-29")]
    vals = [0, 1, -1]
    for d in days:
        t = int(d) * per_day
        vals += [t, t - 1, t + 1, t + per_day // 2 + (per_day // 7)]
    if unit == "D":
        vals += [-(2 ** 31), 2 ** 31 - 1, -(2 ** 31) + 1, 2 ** 31 - 2]
    lim = {"D": 2 ** 31, "s": 10 ** 12, "ms": 10 ** 15, "us": 10 ** 18, "ns": 9 * 10 ** 18}[unit]
    rng = np.random.default_rng(11)
    vals += rng.integers(-lim, lim, 3000).tolist()
    return np.array([v for v in vals if -(2 ** 63) <= v < 2 ** 63], dtype=np.int64)


def _run(prog_code, cols, n, out_nullable=True):
    import torch
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    from dask_sql_b200.device import DeviceColumn
    p = L.Prog()
    p.n = len(prog_code)
    p.out_dtype = L.I64
    for i, (op, a, imm) in enumerate(prog_code):
        p.code[i].op, p.code[i].a, p.code[i].imm_i, p.code[i].imm_f = op, a, imm, 0.0
    dev = torch.device("cuda", 0)
    dcols = []
    for vals, nulls in cols:
        valid = None
        if nulls is not None:
            valid = torch.from_numpy(D._pack_valid(nulls)).to(dev)
        dcols.append(DeviceColumn(torch.from_numpy(np.ascontiguousarray(vals)).to(dev), valid, L.I64))
    out = D.expr_eval(p, dcols, n, out_nullable)
    torch.cuda.synchronize()
    vals = out.data.cpu().numpy()
    isnull = np.zeros(n, bool)
    if out.valid is not None:
        bits = out.valid.cpu().numpy().view(np.uint8)
        isnull = ~np.unpackbits(bits, bitorder="little")[:n].astype(bool)
    return vals, isnull


@pytest.mark.parametrize("unit", ["D", "s", "ms", "us", "ns"])
def test_datepart_every_field_matches_reference(unit):
    from dask_sql_b200 import _lib as L
    x = _pool(unit)
    nulls = np.zeros(len(x), bool)
    nulls[::17] = True
    for fi, field in enumerate(R.FIELDS):
        got, isnull = _run([(L.OP_LOAD, 0, 0), (L.OP_DATEPART, fi, R.TPS[unit])], [(x, nulls)], len(x))
        np.testing.assert_array_equal(isnull, nulls)
        want = R.datepart(x, field, unit)
        np.testing.assert_array_equal(got[~nulls], want[~nulls], err_msg=f"{field} {unit}")


@pytest.mark.parametrize("unit", ["D", "s", "ms", "us", "ns"])
@pytest.mark.parametrize("to_last", [0, 1])
def test_addmonths_matches_reference(unit, to_last):
    from dask_sql_b200 import _lib as L
    x = _pool(unit)
    rng = np.random.default_rng(5)
    n = rng.integers(-30, 30, len(x)).astype(np.int64)
    n[:8] = [0, 1, -1, 12, -12, 13, -13, 1200]
    nn = np.zeros(len(x), bool)
    nn[5::23] = True
    keep = np.abs(x // R.tpd(unit)) < 2 ** 31 - 40000          # the target stays inside int64 ticks
    x, n, nn = x[keep], n[keep], nn[keep]
    got, isnull = _run([(L.OP_LOAD, 0, 0), (L.OP_LOAD, 1, 0), (L.OP_ADDMONTHS, to_last, R.TPS[unit])],
                       [(x, None), (n, nn)], len(x))
    np.testing.assert_array_equal(isnull, nn)
    want = R.add_months(x, n, unit, bool(to_last))
    np.testing.assert_array_equal(got[~nn], want[~nn])


@pytest.mark.parametrize("n", SIZES)
def test_row_counts_around_warp_block_and_tile(n):
    from dask_sql_b200 import _lib as L
    x = np.resize(_pool("us"), n)
    nulls = (np.arange(n) % 5) == 3
    got, isnull = _run([(L.OP_LOAD, 0, 0), (L.OP_DATEPART, L.DP_ISOWEEK, 10 ** 6)], [(x, nulls)], n)
    np.testing.assert_array_equal(isnull, nulls)
    np.testing.assert_array_equal(got[~nulls], R.datepart(x, "ISOWEEK", "us")[~nulls])


def test_bad_programs_are_refused():
    from dask_sql_b200 import _lib as L
    x = np.zeros(4, np.int64)
    with pytest.raises(Exception):
        _run([(L.OP_LOAD, 0, 0), (L.OP_DATEPART, 13, 1)], [(x, None)], 4)
    with pytest.raises(Exception):
        _run([(L.OP_LOAD, 0, 0), (L.OP_DATEPART, 1, 7)], [(x, None)], 4)
    with pytest.raises(Exception):
        _run([(L.OP_LOAD, 0, 0), (L.OP_ADDMONTHS, 0, 1)], [(x, None)], 4)
