"""The 32-bit images that prepared star plans stream in place of int64 columns (DeviceColumn.star_image,
b2_narrow_image, the B2_U32 branch of b2_load_batch).  Star queries through Context.sql() with and without
images (B200SQL_NO_NARROW=1) against the exact reference of tests/query_ref.py, at the edges of the 2^32 span
and of int64, with NULL keys, DATE keys and an imaged int64 SUM input; an in-place write to a registered column
between two runs; the image kernel word for word; and the entry points that must refuse an image."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
import torch

from tests import query_ref as Q
from tests.test_sql_paths_gpu import I64_MAX, I64_MIN, run

pytestmark = pytest.mark.gpu

SQL = ("SELECT d.g AS g, SUM(f.v) AS s, SUM(f.w) AS sw, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
       "WHERE f.x > {x} AND d.flag < 5 GROUP BY d.g")
ND, NF = 3000, 120_000


def _partitions(c, name):
    return c.schema[c.schema_name].tables[name].df.source.table.partitions


def _imaged(c, table, col):
    """per partition: does the column carry a 32-bit image (made by the last star run)?"""
    from dask_sql_b200 import _lib as L
    out = []
    for p in _partitions(c, table):
        img = p[col]._image
        out.append(img is not None and img[1].dtype == L.U32)
    return out


def _span(rng, n, lo, width):
    """n int64 values in [lo, lo + width] (Python ints, so the ends of int64 are exact), both ends in every run of
    1000 rows: an image belongs to one partition and is decided over its rows alone"""
    v = np.array([lo + int(o) for o in rng.integers(0, width + 1, n, dtype=np.uint64)], dtype=object)
    v[0::1000], v[1::1000] = lo, lo + width
    return v.astype(np.int64)


def _tables(rng, pk_lo=0, x_lo=-(2 ** 31), x_width=2 ** 32 - 1, w_lo=2 ** 40, w_width=2 ** 32 - 1, fk_nulls=False):
    pk = (rng.permutation(ND) + pk_lo).astype(np.int64)
    dim = pd.DataFrame({"pk": pk, "flag": rng.integers(0, 10, ND), "g": rng.integers(-20, 30, ND)})
    fk = (rng.integers(-5, ND + 5, NF) + pk_lo).astype(np.int64)
    fact = pd.DataFrame({"fk": fk, "x": _span(rng, NF, x_lo, x_width),
                         "v": rng.integers(-2 ** 20, 2 ** 20, NF) * 2.0 ** -10,     # dyadic: sums are exact
                         "w": _span(rng, NF, w_lo, w_width)})
    if fk_nulls:
        fact["fk"] = pd.array(fk, dtype="Int64")
        fact.loc[rng.random(NF) < 0.1, "fk"] = pd.NA
    return dim, fact


def _ref(dim, fact, x):
    j = Q.join(Q.table(fact), Q.table(dim), ["fk"], ["pk"], "inner")
    mask = Q.cmp(j["x"], ">", x) & Q.cmp(j["flag"], "<", 5)
    return Q.aggregate(j, ["g"], [("s", "sum", "v"), ("sw", "sum", "w"), ("n", "count_star")], mask=mask)


def _bits(got):
    """result rows in group order, floats as their bit patterns"""
    order = np.argsort(np.array(got["g"], dtype=np.int64), kind="stable")
    return {k: [np.float64(v[i]).view(np.int64).item() if isinstance(v[i], float) else v[i] for i in order]
            for k, v in got.items()}


CASES = {
    # case: (table arguments, x literal, fact columns that must be imaged, ... that must not)
    "span_2^32-1": (dict(), 0, ("fk", "x", "w"), ()),
    "span_2^32": (dict(x_width=2 ** 32, w_width=2 ** 32), 0, ("fk",), ("x", "w")),
    "int64_min": (dict(x_lo=I64_MIN, w_lo=I64_MIN), I64_MIN + 2 ** 31, ("fk", "x", "w"), ()),
    "int64_max": (dict(x_lo=I64_MAX - (2 ** 32 - 1), w_lo=I64_MAX - (2 ** 32 - 1)), I64_MAX - 2 ** 31,
                  ("fk", "x", "w"), ()),
    "negative": (dict(pk_lo=-10 ** 12, x_lo=-(2 ** 40), w_lo=-(2 ** 50)), -(2 ** 40) + 2 ** 31,
                 ("fk", "x", "w"), ()),
    "nullable_fk": (dict(fk_nulls=True), 0, ("fk", "x", "w"), ()),
}


@pytest.mark.parametrize("case", list(CASES))
def test_star_images(monkeypatch, case):
    from dask_sql_b200 import Context
    kw, x, imaged, wide = CASES[case]
    dim, fact = _tables(np.random.default_rng(len(case)), **kw)
    exp = _ref(dim, fact, x)
    got = {}
    for arm in ("images", "int64"):
        if arm == "int64":
            monkeypatch.setenv("B200SQL_NO_NARROW", "1")
        c = Context()
        c.create_table("fact", fact, npartitions=3, persist=True)
        c.create_table("dim", dim, persist=True)
        for _ in range(2):                       # the second run re-uses the prepared plan and its images
            got[arm] = run(c, SQL.format(x=x), "star_fused")
            Q.assert_result(got[arm], exp, what=f"{case}, {arm}")
        for col in imaged:
            assert all(_imaged(c, "fact", col)) == (arm == "images"), f"{col} of {case}, {arm}"
        for col in wide:
            assert not any(_imaged(c, "fact", col)), f"{col} spans 2^32 or more: no image"
        if arm == "images":
            assert all(_imaged(c, "dim", "pk")) and all(_imaged(c, "dim", "g"))
    assert _bits(got["images"]) == _bits(got["int64"])


def test_star_images_date_keys(monkeypatch):
    """DATE join keys and a DATE predicate column: day numbers, imaged like any int64 column"""
    from dask_sql_b200 import Context
    rng = np.random.default_rng(3)
    dim, fact = _tables(rng, pk_lo=18000)
    day = lambda v: np.asarray(v, dtype=np.int64).astype("datetime64[D]")
    lit = 18000 + ND // 2
    sql = ("SELECT d.g AS g, SUM(f.v) AS s, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
           f"WHERE f.t > DATE '{np.datetime64(lit, 'D')}' AND d.flag < 5 GROUP BY d.g")
    j = Q.join(Q.table(fact.assign(t=fact["fk"])), Q.table(dim), ["fk"], ["pk"], "inner")
    exp = Q.aggregate(j, ["g"], [("s", "sum", "v"), ("n", "count_star")],
                      mask=Q.cmp(j["t"], ">", lit) & Q.cmp(j["flag"], "<", 5))
    got = {}
    for arm in ("images", "int64"):
        if arm == "int64":
            monkeypatch.setenv("B200SQL_NO_NARROW", "1")
        c = Context()
        c.create_table("fact", {"fk": day(fact["fk"]), "t": day(fact["fk"]), "v": fact["v"].to_numpy()},
                       npartitions=3, persist=True)
        c.create_table("dim", {"pk": day(dim["pk"]), "flag": dim["flag"].to_numpy(), "g": dim["g"].to_numpy()},
                       persist=True)
        got[arm] = run(c, sql, "star_fused")
        Q.assert_result(got[arm], exp, what=arm)
        assert all(_imaged(c, "fact", "fk")) == (arm == "images") and all(_imaged(c, "fact", "t")) == (arm == "images")
    assert _bits(got["images"]) == _bits(got["int64"])


def test_star_image_follows_in_place_write():
    """a write to a registered column between two runs of one prepared plan: the next run makes the image
    again, from fresh statistics, and answers over the new values"""
    from dask_sql_b200 import Context
    dim, fact = _tables(np.random.default_rng(5))
    c = Context()
    c.create_table("fact", fact, npartitions=3, persist=True)
    c.create_table("dim", dim, persist=True)
    Q.assert_result(run(c, SQL.format(x=0), "star_fused"), _ref(dim, fact, 0), what="before the write")
    before = [p["x"]._image[1] for p in _partitions(c, "fact")]
    for p in _partitions(c, "fact"):
        p["x"].data.neg_()                       # in place: new values, a new range, the same tensor
        p["w"].data.sub_(2 ** 35)
    fact2 = fact.assign(x=-fact["x"], w=fact["w"] - 2 ** 35)
    Q.assert_result(run(c, SQL.format(x=0), "star_fused"), _ref(dim, fact2, 0), what="after the write")
    after = [p["x"]._image[1] for p in _partitions(c, "fact")]
    assert all(a is not b for a, b in zip(after, before)) and all(_imaged(c, "fact", "x"))


def test_narrow_image_kernel_words():
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    rng = np.random.default_rng(7)
    n = 10_001
    for lo in (I64_MIN, -12345, I64_MAX - (2 ** 32 - 1)):
        vals = _span(rng, n, lo, 2 ** 32 - 1)
        null = rng.random(n) < 0.2
        null[0::1000] = null[1::1000] = False     # the ends are values, so the base is lo
        col = D.column_from_host(pd.Series(pd.arrays.IntegerArray(vals, null)), D.cur_device())
        img = col.star_image()
        assert img.dtype == L.U32 and img.base == lo and img.valid is col.valid
        got = img.data.cpu().numpy().view(np.uint32)
        exp = np.where(null, 0, (vals.view(np.uint64) - np.uint64(lo & (2 ** 64 - 1))) & np.uint64(0xFFFFFFFF))
        assert np.array_equal(got.astype(np.uint64), exp.astype(np.uint64))
        assert col.star_image() is img            # kept while the values are unchanged


def test_other_entry_points_refuse_images():
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    col = D.column_from_host(np.arange(1000, dtype=np.int64) - 7, D.cur_device())
    img = col.star_image()
    assert img.dtype == L.U32
    scan = D.make_scan([img], [D.TermSpec(0, L.GT, 3)])
    aggs = D.make_aggs([(0, L.AGG_SUM)])
    acc = torch.zeros(1, dtype=torch.int64, device=col.device)
    cnt = torch.zeros(1, dtype=torch.int64, device=col.device)
    ws = torch.empty(L.scan_agg_ws_bytes(), dtype=torch.uint8, device=col.device)
    with pytest.raises(L.B200SqlError, match=r"\(-2\)"):
        L.scan_agg(C.byref(scan), aggs, 1, D.ptr(acc), D.ptr(cnt), 0, D.ptr(ws), D.stream_ptr())
    tile_off = torch.empty(L.num_tiles(1000) + 1, dtype=torch.int64, device=col.device)
    with pytest.raises(L.B200SqlError, match=r"\(-2\)"):
        L.select_count(C.byref(scan), D.ptr(tile_off), D.stream_ptr())
