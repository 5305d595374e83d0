"""The ranked-bitmap lookup of the fused star pipeline (b2_star_build_mark / _rank / _fill, probed by
b2_star_agg): dimension shapes that exercise the directory's rank and the slot array, against pandas."""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu
RTOL = 1e-9


def _table(df, npartitions=1):
    import torch
    from dask_sql_b200.frame import LazyFrame, TableSource
    from dask_sql_b200.table import DeviceTable

    dev = torch.device("cuda", torch.cuda.current_device())
    return LazyFrame(TableSource(DeviceTable.from_pandas(df, npartitions, dev, True)))


def _dim_fact(case, rng):
    nd, nf, ng = 40_000, 600_000, 700
    pk = rng.permutation(nd).astype(np.int64)
    if case == "holes":
        pk = pk * 3 + 11                     # key range about 3x the row count: two in three keys unused
    dim = pd.DataFrame({"pk": pk, "flag": rng.integers(0, 10, nd), "grp": rng.integers(0, ng, nd)})
    fk = pk[rng.integers(0, nd, nf)]
    if case == "outside":
        out = rng.random(nf) < 0.3
        fk = np.where(out, np.where(rng.random(nf) < 0.5, pk.min() - 1 - rng.integers(0, 100, nf),
                                    pk.max() + 1 + rng.integers(0, 100, nf)), fk)
    if case == "nulls":
        dim["pk"] = pd.array(dim["pk"], dtype="Int64")
        dim["grp"] = pd.array(dim["grp"], dtype="Int64")
        dim.loc[rng.random(nd) < 0.05, "pk"] = pd.NA
        dim.loc[rng.random(nd) < 0.05, "grp"] = pd.NA
    if case == "dup_passing":
        i, k = np.flatnonzero(dim["flag"].to_numpy() < 5)[:2]
        dim.loc[k, "pk"] = dim.loc[i, "pk"]
    if case == "dup_filtered":
        i, k = np.flatnonzero(dim["flag"].to_numpy() >= 5)[:2]
        dim.loc[k, "pk"] = dim.loc[i, "pk"]
    fact = pd.DataFrame({"fk": fk, "x": rng.integers(-2**31, 2**31, nf), "val": rng.random(nf)})
    return dim, fact


def _expected(fact, dim, dim_pred):
    f = fact[fact["x"] > 0]
    d = dim[dim["flag"] < 5] if dim_pred else dim
    d = d[d["pk"].notna()]                   # NULL keys never join
    j = f.merge(d.astype({"pk": "int64"}), left_on="fk", right_on="pk", how="inner")
    return j.groupby("grp", dropna=False).agg(rev=("val", "sum"), n=("val", "size")).reset_index()


CASES = [  # (case, dim partitions, dim predicate, fused path taken)
    ("multi_partition", 3, True, True),
    ("holes", 2, True, True),
    ("no_predicate", 3, False, True),
    ("nulls", 2, True, True),
    ("outside", 1, True, True),
    ("dup_passing", 2, True, False),
    ("dup_filtered", 2, True, True),
]


@pytest.mark.parametrize("case,dparts,dim_pred,fused", CASES, ids=[c[0] for c in CASES])
def test_star_bitmap_lookup(case, dparts, dim_pred, fused):
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import AggSource, LazyFrame
    rng = np.random.default_rng(sum(map(ord, case)))
    dim, fact = _dim_fact(case, rng)
    f, d = _table(fact, 4), _table(dim, dparts)
    dd = d[d["flag"] < 5] if dim_pred else d
    j = f[f["x"] > 0].merge(dd, left_on=["fk"], right_on=["pk"], how="inner")
    before = executor.stats["star_fused"]
    got = LazyFrame(AggSource(j, ["grp"], [("val", "rev", "sum"), (None, "n", "size")])).compute()
    assert executor.stats["star_fused"] == before + (1 if fused else 0)
    exp = _expected(fact, dim, dim_pred)
    got = got.sort_values("grp", na_position="last").reset_index(drop=True)
    exp = exp.sort_values("grp", na_position="last").reset_index(drop=True)
    assert len(got) == len(exp), f"{len(got)} groups vs {len(exp)}"
    np.testing.assert_array_equal(got["grp"].to_numpy(dtype=float, na_value=np.nan),
                                  exp["grp"].to_numpy(dtype=float, na_value=np.nan))
    np.testing.assert_array_equal(got["n"].to_numpy(dtype=np.int64), exp["n"].to_numpy(dtype=np.int64))
    np.testing.assert_allclose(got["rev"].to_numpy(dtype=float), exp["rev"].to_numpy(dtype=float), rtol=RTOL)


def test_star_bitmap_lookup_twice_on_prepared_plan():
    """A repeated query rebuilds the lookup into the same buffer: the second run must not see the first
    run's bits or ranks."""
    from dask_sql_b200 import Context
    rng = np.random.default_rng(21)
    dim, fact = _dim_fact("multi_partition", rng)
    c = Context()
    c.create_table("fact", fact, npartitions=4)
    c.create_table("dim", dim, npartitions=3)
    q = ("SELECT d.grp, SUM(f.val) AS rev, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
         "WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp")
    exp = _expected(fact, dim, True).sort_values("grp").reset_index(drop=True)
    for _ in range(2):
        got = c.sql(q).compute().sort_values("grp").reset_index(drop=True)
        np.testing.assert_array_equal(got["grp"].to_numpy(), exp["grp"].to_numpy())
        np.testing.assert_array_equal(got["n"].to_numpy(), exp["n"].to_numpy())
        np.testing.assert_allclose(got["rev"].to_numpy(), exp["rev"].to_numpy(), rtol=RTOL)
