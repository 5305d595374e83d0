"""GroupTable.reset(): every array a group table allocates -- accumulators, counts, rows, presence bitmap --
goes back to the value an empty table holds, on CPU tensors.  A prepared star plan refills its tables
this way run after run, including the two in symmetric memory that it allocates through `new=`."""
import pytest
import torch

from dask_sql_b200 import _lib as L
from dask_sql_b200 import device as D
from dask_sql_b200.device import F64, I64

INT64_MIN = -(1 << 63)
# (input column, op), dtype, count kept next to it
AGGS = [((0, L.AGG_SUM), I64, False), ((1, L.AGG_SUM), F64, True), ((2, L.AGG_MIN), I64, False),
        ((3, L.AGG_MAX), I64, False), ((4, L.AGG_AND), I64, False), ((5, L.AGG_COUNT), I64, False)]


def _carving(nbytes):
    """a `new=` allocator that hands out filled views of one buffer, as the symmetric-memory arena does"""
    buf = torch.empty(nbytes, dtype=torch.uint8)
    used = [0]

    def new(n, dtype, fill):
        width = torch.empty((), dtype=dtype).element_size()
        t = buf[used[0]: used[0] + n * width].view(dtype)
        used[0] += (n * width + 255) // 256 * 256
        t.fill_(fill)
        return t
    return new


def _table(aggs, rows, present, indicator, new):
    specs, dtypes, need_cnt = zip(*aggs)
    return D.GroupTable(torch.device("cpu"), 1000, list(specs), list(dtypes), list(need_cnt), rows, present,
                        indicator=indicator, alloc=1024, new=new)


def _bits(t):
    return t.view(torch.int64) if t.dtype == torch.float64 else t.to(torch.int64)


def _check_empty(t, aggs, indicator):
    for a, (((_, op), dt, _), acc) in enumerate(zip(aggs, t.acc)):
        if op == L.AGG_COUNT:
            assert acc is None
            continue
        want = INT64_MIN if a == indicator else 0 if dt == F64 else L.agg_identity(op)
        assert (_bits(acc) == want).all(), (a, op)
    for a, cnt in enumerate(t.cnt):
        assert cnt is None or (cnt == 0).all(), a
    for arr in (t.rows, t.present):
        assert arr is None or (arr == 0).all()


@pytest.mark.parametrize("carve", [False, True])
@pytest.mark.parametrize("rows,present,indicator", [(True, True, None), (False, False, 1)])
def test_reset_restores_every_array(rows, present, indicator, carve):
    new = _carving(1 << 20) if carve else None
    t = _table(AGGS, rows, present, indicator, new)
    arrays = [x for x in t.acc + t.cnt + [t.rows, t.present] if x is not None]
    assert sorted(x.data_ptr() for x in arrays) == sorted(x.data_ptr() for x, _ in t.fills)
    assert (t.rows is not None) == rows and (t.present is not None) == present
    _check_empty(t, AGGS, indicator)
    for x in arrays:
        if x.dtype == torch.float64:
            x.fill_(3.5)
        else:
            x.fill_(0x5A5A5A5A)
    t.reset()
    _check_empty(t, AGGS, indicator)
