"""GPU parity of the execution layer below the SQL surface: LazyFrame ops (the calls the plugins
make) against the pandas oracle on the same seeded inputs.  Integers bit-exact; float SUM/AVG
within 1e-9 relative (BASELINE.json north_star)."""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-9


def _table(df, npartitions=1, persist=True):
    import torch
    from dask_sql_b200.frame import LazyFrame, TableSource
    from dask_sql_b200.table import DeviceTable

    dev = torch.device("cuda", torch.cuda.current_device())
    return LazyFrame(TableSource(DeviceTable.from_pandas(df, npartitions, dev, persist)))


def _sorted(df, cols=None):
    cols = cols or list(df.columns)
    return df.sort_values(cols, na_position="last").reset_index(drop=True)


def assert_frames(got, exp, float_cols=(), sort_by=None):
    got, exp = _sorted(got, sort_by), _sorted(exp, sort_by)
    assert list(got.columns) == list(exp.columns)
    assert len(got) == len(exp), f"{len(got)} rows vs {len(exp)}"
    for c in got.columns:
        g, e = got[c].to_numpy(dtype=float, na_value=np.nan), exp[c].to_numpy(dtype=float, na_value=np.nan)
        if c in float_cols:
            np.testing.assert_allclose(g, e, rtol=RTOL, atol=0, equal_nan=True)
        else:
            np.testing.assert_array_equal(g, e)


def agg(frame, by, spec):
    from dask_sql_b200.frame import AggSource, LazyFrame
    return LazyFrame(AggSource(frame, by, spec)).compute()


@pytest.mark.parametrize("n,nparts", [(1, 1), (31, 1), (4096, 1), (100_003, 3), (1_000_000, 8)])
def test_filter_select(n, nparts):
    rng = np.random.default_rng(n)
    df = pd.DataFrame({"x": rng.integers(-1000, 1000, n), "y": rng.random(n), "z": rng.integers(0, 5, n)})
    f = _table(df, nparts)
    got = f[(f["x"] > 0) & (f["y"] < 0.5)].compute()
    exp = df[(df["x"] > 0) & (df["y"] < 0.5)]
    # selection is order preserving: compare without sorting
    pd.testing.assert_frame_equal(got.reset_index(drop=True), exp.reset_index(drop=True))


def test_filter_complex_predicate_and_projection():
    rng = np.random.default_rng(5)
    n = 50_000
    df = pd.DataFrame({"a": rng.integers(-50, 50, n), "b": rng.random(n) * 10, "c": rng.integers(0, 3, n)})
    f = _table(df, 2)
    cond = ((f["a"] < 3) | (f["b"] > 7.5)) & ~(f["c"] == 1)
    out = f[cond].assign(s=f["a"] * 2 + f["c"], q=f["b"] / 4)[["s", "q", "a"]].compute()
    m = ((df["a"] < 3) | (df["b"] > 7.5)) & ~(df["c"] == 1)
    exp = df[m].assign(s=df["a"] * 2 + df["c"], q=df["b"] / 4)[["s", "q", "a"]]
    pd.testing.assert_frame_equal(out.reset_index(drop=True), exp.reset_index(drop=True))


def test_filter_nulls_are_false():
    df = pd.DataFrame({"c": pd.array([1, 2, None, 3, None, 3], dtype="Int64"),
                       "f": [1.0, np.nan, 3.0, np.nan, 5.0, 6.0]})
    f = _table(df)
    got = f[f["c"] == 3].compute()
    assert got["c"].tolist() == [3, 3]
    got = f[f["c"].isna()].compute()
    assert len(got) == 2
    # IEEE: NaN != x is True for plain float columns (numpy semantics the reference inherits)
    got = f[f["f"] != 1.0].compute()
    assert len(got) == 5
    got = f[f["f"].isna()].compute()
    assert len(got) == 2


@pytest.mark.parametrize("n,nparts", [(10, 1), (100_000, 1), (1_000_003, 8)])
def test_global_aggregates(n, nparts):
    from oracle import pandas_oracle as O
    rng = np.random.default_rng(1)
    df = pd.DataFrame({"x": rng.integers(-2**31, 2**31, n), "v": rng.random(n)})
    f = _table(df, nparts)
    g = f[f["x"] > 0]
    got = agg(g, [], [("x", "s", "sum"), ("v", "sv", "sum"), ("v", "av", "mean"), ("x", "mn", "min"),
                      ("x", "mx", "max"), ("v", "vmn", "min"), ("v", "vmx", "max"), (None, "n", "size")])
    e = df[df["x"] > 0]
    assert int(got["s"][0]) == int(e["x"].sum())
    assert int(got["n"][0]) == len(e)
    assert int(got["mn"][0]) == int(e["x"].min()) and int(got["mx"][0]) == int(e["x"].max())
    assert got["vmn"][0] == e["v"].min() and got["vmx"][0] == e["v"].max()
    np.testing.assert_allclose(got["sv"][0], e["v"].sum(), rtol=RTOL)
    np.testing.assert_allclose(got["av"][0], e["v"].mean(), rtol=RTOL)
    # oracle path (partitioned restatement) agrees too
    o = O.c1_filter_sum(O.split(df[["x"]], nparts))
    assert int(o.iloc[0, 0]) == int(got["s"][0])


def test_int64_sum_wraps_like_numpy():
    df = pd.DataFrame({"x": np.array([2**62, 2**62, 2**62, 5], dtype=np.int64)})
    got = agg(_table(df), [], [("x", "s", "sum")])
    with np.errstate(over="ignore"):
        assert int(got["s"][0]) == int(df["x"].to_numpy().sum())


@pytest.mark.parametrize("nkeys,n,nparts", [(10, 1000, 1), (1000, 200_000, 4), (100_000, 1_000_000, 8)])
@pytest.mark.parametrize("vtype", ["int", "float"])
def test_groupby_dense(nkeys, n, nparts, vtype):
    from oracle import pandas_oracle as O
    from dask_sql_b200 import executor
    rng = np.random.default_rng(2)
    val = rng.integers(-1000, 1001, n) if vtype == "int" else rng.random(n)
    df = pd.DataFrame({"key": rng.integers(0, nkeys, n), "val": val})
    before = executor.stats["dense_groupby"]
    got = agg(_table(df, nparts), ["key"], [("val", "s", "sum"), ("val", "a", "mean"), ("val", "c", "count"),
                                            ("val", "lo", "min"), ("val", "hi", "max")])
    assert executor.stats["dense_groupby"] == before + 1
    exp = O.groupby_agg(O.split(df, nparts), ["key"], [("val", "s", "sum"), ("val", "a", "mean"),
                                                       ("val", "c", "count"), ("val", "lo", "min"),
                                                       ("val", "hi", "max")])
    fc = ("a",) if vtype == "int" else ("s", "a")
    assert_frames(got, exp, float_cols=fc, sort_by=["key"])


def test_groupby_hash_sparse_keys_and_sentinels():
    from dask_sql_b200 import executor
    rng = np.random.default_rng(3)
    n = 300_000
    keys = rng.integers(-2**62, 2**62, 5000)
    keys[0], keys[1] = -(2**63), 2**63 - 1        # the table's EMPTY sentinel is a legal key
    df = pd.DataFrame({"key": keys[rng.integers(0, 5000, n)], "val": rng.integers(-5, 6, n)})
    before = executor.stats["hash_groupby"]
    got = agg(_table(df, 3), ["key"], [("val", "s", "sum"), (None, "n", "size")])
    assert executor.stats["hash_groupby"] == before + 1
    exp = df.groupby("key", dropna=False).agg(s=("val", "sum"), n=("val", "size")).reset_index()
    assert_frames(got, exp, sort_by=["key"])


def test_groupby_hash_grows_on_overflow():
    rng = np.random.default_rng(4)
    n = 3_000_000
    df = pd.DataFrame({"key": rng.integers(0, 2**40, n) * 1000003, "val": np.ones(n, dtype=np.int64)})
    got = agg(_table(df, 2), ["key"], [("val", "s", "sum")])
    exp = df.groupby("key").agg(s=("val", "sum")).reset_index()
    assert_frames(got, exp, sort_by=["key"])


def test_groupby_null_keys_and_null_values():
    # reference pins: NULL key forms its own group (tests/integration/test_groupby.py:174-186),
    # SUM over an all-NULL group is NULL (test_groupby.py:133-141)
    df = pd.DataFrame({
        "k": pd.array([1, None, 2, None, 1, 3], dtype="Int64"),
        "v": pd.array([10, 20, None, 40, 50, None], dtype="Int64"),
        "f": [1.5, np.nan, 2.5, 3.5, np.nan, np.nan],
    })
    got = agg(_table(df), ["k"], [("v", "sv", "sum"), ("v", "cv", "count"), ("f", "sf", "sum"), ("f", "af", "mean"),
                                  (None, "n", "size")])
    got = got.sort_values("k", na_position="last").reset_index(drop=True)
    assert got["k"].isna().tolist() == [False, False, False, True]
    assert got["n"].tolist() == [2, 1, 1, 2]
    assert got["cv"].tolist() == [2, 0, 0, 2]
    sv = got["sv"].to_numpy(dtype=float, na_value=np.nan)
    np.testing.assert_array_equal(sv, [60, np.nan, np.nan, 60])
    np.testing.assert_array_equal(got["sf"].to_numpy(dtype=float), [1.5, 2.5, np.nan, 3.5])
    np.testing.assert_array_equal(got["af"].to_numpy(dtype=float), [1.5, 2.5, np.nan, 3.5])


def test_groupby_two_keys_and_float_key():
    rng = np.random.default_rng(6)
    n = 200_000
    df = pd.DataFrame({"a": rng.integers(0, 50, n), "b": rng.integers(-3, 4, n).astype(float), "v": rng.random(n)})
    df.loc[rng.integers(0, n, 500), "b"] = np.nan
    got = agg(_table(df, 4), ["a", "b"], [("v", "s", "sum"), (None, "n", "size")])
    exp = df.groupby(["a", "b"], dropna=False).agg(s=("v", "sum"), n=("v", "size")).reset_index()
    assert_frames(got, exp, float_cols=("s",), sort_by=["a", "b"])
    got = agg(_table(df, 4), ["b"], [("v", "s", "sum")])
    exp = df.groupby(["b"], dropna=False).agg(s=("v", "sum")).reset_index()
    assert_frames(got, exp, float_cols=("s",), sort_by=["b"])


def test_distinct():
    rng = np.random.default_rng(7)
    df = pd.DataFrame({"a": rng.integers(0, 7, 10_000), "b": rng.integers(0, 3, 10_000)})
    got = _table(df, 2).drop_duplicates().compute()
    assert_frames(got, df.drop_duplicates(), sort_by=["a", "b"])


@pytest.mark.parametrize("how", ["inner", "left", "right", "outer", "leftsemi", "leftanti"])
def test_join_types_small_with_duplicates_and_nulls(how):
    from oracle import pandas_oracle as O
    lhs = pd.DataFrame({"lk": pd.array([2, 1, 2, 3, None, 7], dtype="Int64"), "b": [3, 3, 1, 3, 9, 8]})
    rhs = pd.DataFrame({"rk": pd.array([1, 1, 2, 4, None], dtype="Int64"), "c": [1, 2, 3, 4, 5]})
    if how == "outer":
        # pandas.merge matches NA keys with NA keys and the reference only drops them for the
        # other join types (join.py:202-213); SQL never matches NULL keys and neither do we
        # (DESIGN.md "Known divergences"), so keep NULL keys to one side here.
        rhs = rhs.iloc[:4]
    got = _table(lhs).merge(_table(rhs), left_on=["lk"], right_on=["rk"], how=how).compute()
    exp = O.join_on_columns(lhs, rhs, ["lk"], ["rk"], how)
    if how in ("leftsemi", "leftanti"):
        exp = exp[["lk", "b"]]
    assert_frames(got, exp, sort_by=list(exp.columns))


@pytest.mark.parametrize("dense", [True, False])
def test_join_inner_large(dense):
    from oracle import pandas_oracle as O
    from dask_sql_b200 import executor
    rng = np.random.default_rng(8)
    nd, nf = 100_000, 1_000_000
    pk = rng.permutation(nd).astype(np.int64)
    if not dense:
        pk = pk * 1_000_003 + 17
    dim = pd.DataFrame({"pk": pk, "w": rng.integers(0, 100, nd)})
    fk = pk[rng.integers(0, nd, nf)]
    miss = rng.random(nf) < 0.2
    fk = np.where(miss, -5 - rng.integers(0, 1000, nf), fk)
    fact = pd.DataFrame({"fk": fk, "v": rng.random(nf)})
    key = "dense_join" if dense else "chain_join"
    before = executor.stats[key]
    got = _table(fact, 8).merge(_table(dim), left_on=["fk"], right_on=["pk"], how="inner")[["fk", "v", "w"]].compute()
    assert executor.stats[key] == before + 1
    exp = pd.concat(O.c3_join(O.split(fact, 8), dim))
    assert len(got) == len(exp)
    assert_frames(got, exp, sort_by=["fk", "v", "w"])


def test_join_duplicate_build_keys_many_to_many():
    rng = np.random.default_rng(9)
    lhs = pd.DataFrame({"k": rng.integers(0, 50, 5000), "a": np.arange(5000)})
    rhs = pd.DataFrame({"k2": rng.integers(0, 60, 700), "b": np.arange(700)})
    got = _table(lhs, 2).merge(_table(rhs), left_on=["k"], right_on=["k2"], how="inner").compute()
    exp = lhs.merge(rhs, left_on="k", right_on="k2", how="inner")
    assert_frames(got, exp, sort_by=["a", "b"])


def test_join_two_keys():
    rng = np.random.default_rng(10)
    lhs = pd.DataFrame({"a": rng.integers(0, 20, 3000), "b": rng.integers(0, 20, 3000), "x": np.arange(3000)})
    rhs = pd.DataFrame({"c": rng.integers(0, 20, 300), "d": rng.integers(0, 20, 300), "y": np.arange(300)})
    got = _table(lhs).merge(_table(rhs), left_on=["a", "b"], right_on=["c", "d"], how="inner").compute()
    exp = lhs.merge(rhs, left_on=["a", "b"], right_on=["c", "d"], how="inner")
    assert_frames(got, exp, sort_by=["x", "y"])


@pytest.mark.parametrize("sparse_pk,sparse_grp", [(False, False), (True, False), (False, True)])
def test_star_fused_q3(sparse_pk, sparse_grp):
    """filter -> join -> group-by in one pass; equals the oracle's Q3 restatement."""
    from oracle import pandas_oracle as O
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import AggSource, LazyFrame
    rng = np.random.default_rng(11)
    nd, nf, ng = 50_000, 800_000, 1000
    pk = rng.permutation(nd).astype(np.int64)
    if sparse_pk:
        pk = pk * 999_983 + 5
    grp = rng.integers(0, ng, nd)
    if sparse_grp:
        grp = grp * 1_000_000_007 - 3
    dim = pd.DataFrame({"pk": pk, "flag": rng.integers(0, 10, nd), "grp": grp})
    fact = pd.DataFrame({"fk": pk[rng.integers(0, nd, nf)], "x": rng.integers(-2**31, 2**31, nf), "val": rng.random(nf)})
    f, d = _table(fact, 8), _table(dim)
    ff = f[f["x"] > 0]
    dd = d[d["flag"] < 5]
    j = ff.merge(dd, left_on=["fk"], right_on=["pk"], how="inner")
    before = executor.stats["star_fused"]
    got = LazyFrame(AggSource(j, ["grp"], [("val", "rev", "sum")])).compute()
    assert executor.stats["star_fused"] == before + 1, "fused star pipeline was not taken"
    exp = O.c4_q3(O.split(fact, 8), dim)
    assert_frames(got, exp, float_cols=("rev",), sort_by=["grp"])


def test_star_falls_back_on_duplicate_build_keys():
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import AggSource, LazyFrame
    dim = pd.DataFrame({"pk": [1, 1, 2, 3], "grp": [10, 20, 10, 30]})
    fact = pd.DataFrame({"fk": [1, 2, 2, 3, 4], "val": [1.0, 2.0, 3.0, 4.0, 5.0]})
    j = _table(fact).merge(_table(dim), left_on=["fk"], right_on=["pk"], how="inner")
    before = executor.stats["star_fused"]
    got = LazyFrame(AggSource(j, ["grp"], [("val", "rev", "sum")])).compute()
    assert executor.stats["star_fused"] == before
    exp = fact.merge(dim, left_on="fk", right_on="pk").groupby("grp").agg(rev=("val", "sum")).reset_index()
    assert_frames(got, exp, float_cols=("rev",), sort_by=["grp"])


def test_host_resident_table_streams_per_query():
    rng = np.random.default_rng(12)
    df = pd.DataFrame({"key": rng.integers(0, 100, 100_000), "val": rng.random(100_000)})
    got = agg(_table(df, 4, persist=False), ["key"], [("val", "s", "sum")])
    exp = df.groupby("key").agg(s=("val", "sum")).reset_index()
    assert_frames(got, exp, float_cols=("s",), sort_by=["key"])


def test_float_sum_accumulator_doubles_as_group_flag():
    """Dense group-by over a NULL-free float column keeps no presence bitmap: the SUM accumulator
    starts at -0.0 and an untouched slot is an absent group.  Groups whose values are all -0.0 /
    +0.0 / cancel to 0 must still exist (pandas: running sum from +0.0 -> +0.0), absent keys must not."""
    from dask_sql_b200 import executor
    key = np.array([0, 0, 2, 2, 5, 5, 7, 9, 9, 9], dtype=np.int64)          # 1,3,4,6,8 absent
    val = np.array([-0.0, -0.0, 0.0, -0.0, 1.5, -1.5, -0.0, 1e-300, -1e-300, 0.0])
    df = pd.DataFrame({"key": key, "val": val})
    before = executor.stats["dense_groupby"]
    got = agg(_table(df, 2), ["key"], [("val", "s", "sum")])
    assert executor.stats["dense_groupby"] == before + 1
    exp = df.groupby("key").agg(s=("val", "sum")).reset_index()
    assert_frames(got, exp, float_cols=("s",), sort_by=["key"])
    g = _sorted(got, ["key"])
    assert not np.signbit(g["s"].to_numpy()).any(), "sum of zeros must be +0.0 like pandas"


@pytest.mark.parametrize("env", ["B200SQL_NO_INDICATOR", "B200SQL_NO_DEFER"])
def test_dense_groupby_same_result_without_shortcuts(env, monkeypatch):
    rng = np.random.default_rng(21)
    n = 200_000
    df = pd.DataFrame({"key": rng.integers(0, 5000, n) * 2, "val": rng.random(n), "w": rng.integers(-9, 9, n)})
    spec = [("val", "s", "sum"), ("w", "sw", "sum"), ("val", "mx", "max")]
    a = agg(_table(df, 4), ["key"], spec)
    monkeypatch.setenv(env, "1")
    b = agg(_table(df, 4), ["key"], spec)
    assert_frames(a, b, float_cols=("s",), sort_by=["key"])     # float atomics: order varies run to run
    exp = df.groupby("key").agg(s=("val", "sum"), sw=("w", "sum"), mx=("val", "max")).reset_index()
    assert_frames(a, exp, float_cols=("s",), sort_by=["key"])


def test_dense_result_is_pending_until_used():
    """The compaction of a dense group table is enqueued without waiting for its row count."""
    from dask_sql_b200 import executor
    from dask_sql_b200.frame import AggSource, LazyFrame
    rng = np.random.default_rng(22)
    n = 100_000
    df = pd.DataFrame({"key": rng.integers(0, 1000, n), "val": rng.random(n)})
    frame = LazyFrame(AggSource(_table(df, 2), ["key"], [("val", "s", "sum")]))
    parts = executor.execute(frame)
    assert isinstance(parts[0], executor.PendingPart) and not parts[0].resolved
    assert parts[0].n == df["key"].nunique() and parts[0].resolved
    assert set(parts[0].keys()) == {"key", "s"} and parts[0]["s"].n == parts[0].n
    exp = df.groupby("key").agg(s=("val", "sum")).reset_index()
    assert_frames(frame.compute(), exp, float_cols=("s",), sort_by=["key"])
    # an empty selection resolves to an empty partition
    f = _table(df, 2)
    empty = LazyFrame(AggSource(f[f["val"] > 2.0], ["key"], [("val", "s", "sum")])).compute()
    assert len(empty) == 0 and list(empty.columns) == ["key", "s"]


@pytest.mark.parametrize("how", ["inner", "left", "leftsemi", "leftanti"])
@pytest.mark.parametrize("fk_nulls", [True, False])
def test_join_key_ordered_payload_layout(how, fk_nulls, monkeypatch):
    """Unique dense build keys: build columns are re-laid in key order (narrow uint32 offsets for
    small-range ints, 8 bytes otherwise, bool, nullable) and probed by key offset, with and without NULL
    probe keys.  The result must hold the rows of the row-lookup table's and the oracle's; row order across
    output batches is unspecified, so they are compared sorted."""
    from dask_sql_b200 import executor
    rng = np.random.default_rng(31)
    nd, nf = 20_000, 150_003
    pk = rng.permutation(nd * 2)[:nd].astype(np.int64) - 777           # unique, with holes, negative kmin
    dim = pd.DataFrame({
        "pk": pk,
        "w": rng.integers(-500, 500, nd),                                # narrow int
        "big": rng.integers(-2**62, 2**62, nd),                          # wide int stays 8 bytes
        "f": rng.random(nd),
        "b": rng.integers(0, 2, nd).astype(bool),
        "ni": pd.array(np.where(rng.random(nd) < 0.2, None, rng.integers(0, 9, nd)), dtype="Int64"),
    })
    fk = rng.integers(-2000, nd * 2 + 500, nf).astype(np.int64)         # some outside [kmin, kmax], some in holes
    nulls = rng.random(nf) < 0.05
    fact = pd.DataFrame({"fk": pd.array(np.where(nulls, None, fk), dtype="Int64") if fk_nulls else fk,
                         "v": rng.random(nf)})
    f, d = _table(fact, 3), _table(dim)
    before = executor.stats["keyed_join"]
    got = f.merge(d, left_on=["fk"], right_on=["pk"], how=how).compute()
    assert executor.stats["keyed_join"] == before + 1
    monkeypatch.setenv("B200SQL_NO_KEY_LAYOUT", "1")
    plain = f.merge(d, left_on=["fk"], right_on=["pk"], how=how).compute()
    assert executor.stats["keyed_join"] == before + 1
    pd.testing.assert_frame_equal(_sorted(got), _sorted(plain))          # same rows, same dtypes
    from oracle import pandas_oracle as O
    exp = O.join_on_columns(fact, dim, ["fk"], ["pk"], how)
    assert_frames(got[list(exp.columns)], exp, sort_by=["fk", "v"])


@pytest.mark.parametrize("how", ["inner", "left", "leftsemi", "leftanti"])
@pytest.mark.parametrize("match", [0.03, 0.8])
def test_join_single_pass_equals_two_pass(how, match, monkeypatch):
    """b2_join_onepass (output ranges reserved atomically, count left on the device) must emit
    exactly the rows of the count + write protocol -- across many tiles, with tiles that emit
    nothing and with a pushed-down probe filter.  Row order across batches is unspecified."""
    from dask_sql_b200 import executor
    rng = np.random.default_rng(int(match * 100) + 41)
    nd, nf = 50_000, 700_003
    dim = pd.DataFrame({"pk": rng.permutation(nd).astype(np.int64), "w": rng.integers(0, 1000, nd), "g": rng.random(nd)})
    hit = rng.random(nf) < match
    fk = np.where(hit, rng.integers(0, nd, nf), rng.integers(nd, 2 * nd, nf)).astype(np.int64)
    fk[200_000:420_000] = nd + 7                                   # a long run of tiles without matches
    fact = pd.DataFrame({"fk": fk, "v": rng.random(nf), "x": rng.integers(-5, 5, nf)})
    f, d = _table(fact, 3), _table(dim)

    def run():
        j = f[f["x"] > -3].merge(d, left_on=["fk"], right_on=["pk"], how=how)
        parts = executor.execute(j)
        return parts, j.compute()

    from oracle import pandas_oracle as O
    exp = O.join_on_columns(fact[fact["x"] > -3], dim, ["fk"], ["pk"], how)
    parts, streamed = run()
    assert all(isinstance(p, executor.PendingPart) for p in parts)
    monkeypatch.setenv("B200SQL_NO_ONEPASS", "1")
    parts2, two_pass = run()
    assert not any(isinstance(p, executor.PendingPart) for p in parts2)
    pd.testing.assert_frame_equal(_sorted(streamed), _sorted(two_pass))
    assert len(streamed) == len(exp)
    assert_frames(streamed[list(exp.columns)], exp, sort_by=["fk", "v"])


@pytest.mark.parametrize("nullable_key", [False, True])
def test_groupby_range_partitioned_matches_direct(nullable_key, monkeypatch):
    """Group tables far beyond L2 are fed by b2_range_partition (rows reordered by key range, then the
    same dense kernel).  Forced here on a small table: many buckets, a pushed-down predicate, NULL
    keys, several aggregates sharing inputs, float NaNs as NULL inputs."""
    from dask_sql_b200 import executor
    rng = np.random.default_rng(51)
    n, nkeys = 300_007, 5_000
    key = rng.integers(100, 100 + nkeys, n)
    df = pd.DataFrame({
        "key": pd.array(np.where(rng.random(n) < 0.02, None, key), dtype="Int64") if nullable_key else key,
        "v": rng.random(n),
        "w": rng.integers(-100, 100, n),
        "g": np.where(rng.random(n) < 0.1, np.nan, rng.random(n)),
        "x": rng.integers(0, 10, n),
    })
    spec = [("v", "sv", "sum"), ("w", "sw", "sum"), ("v", "av", "mean"), ("g", "cg", "count"), ("g", "sg", "sum"),
            ("w", "mn", "min"), ("v", "mx", "max"), (None, "n", "size")]

    def run():
        f = _table(df, 3)
        return agg(f[f["x"] > 2], ["key"], spec)

    direct = run()
    monkeypatch.setenv("B200SQL_PARTITION_MIN_BYTES", "1")
    monkeypatch.setenv("B200SQL_PARTITION_BUCKET_BYTES", "8192")
    before = executor.stats["partitioned_groupby"]
    parted = run()
    assert executor.stats["partitioned_groupby"] == before + 1
    fl = ("sv", "av", "sg")
    assert_frames(parted, direct, float_cols=fl, sort_by=["key"])
    d = df[df["x"] > 2]
    exp = d.groupby("key", dropna=False).agg(sv=("v", "sum"), sw=("w", "sum"), av=("v", "mean"), cg=("g", "count"),
                                             sg=("g", lambda s: s.sum(min_count=1)), mn=("w", "min"),
                                             mx=("v", "max"), n=("v", "size")).reset_index()
    assert_frames(parted, exp, float_cols=fl, sort_by=["key"])


@pytest.mark.parametrize("ncarry", [1, 3])
def test_range_partition_scatter_variants(ncarry, monkeypatch):
    """The range-partition scatter with one and with three carried columns must produce the same groups
    as pandas.  Many buckets, a ragged tail, a predicate, NULL keys."""
    from dask_sql_b200 import executor
    rng = np.random.default_rng(77)
    n, nkeys = 250_013, 40_000
    key = rng.integers(-500, -500 + nkeys, n)
    df = pd.DataFrame({"key": pd.array(np.where(rng.random(n) < 0.01, None, key), dtype="Int64"),
                       "v": rng.random(n), "w": rng.integers(-100, 100, n), "u": rng.random(n) * 3,
                       "x": rng.integers(0, 10, n)})
    spec = [("v", "sv", "sum"), ("v", "av", "mean")]
    if ncarry == 3:
        spec += [("w", "sw", "sum"), ("u", "mu", "max")]
    monkeypatch.setenv("B200SQL_PARTITION_MIN_BYTES", "1")
    monkeypatch.setenv("B200SQL_PARTITION_BUCKET_BYTES", "4096")
    before = executor.stats["partitioned_groupby"]
    f = _table(df, 4)
    got = agg(f[f["x"] > 1], ["key"], spec)
    assert executor.stats["partitioned_groupby"] == before + 1
    d = df[df["x"] > 1]
    named = dict(sv=("v", "sum"), av=("v", "mean"))
    if ncarry == 3:
        named.update(sw=("w", "sum"), mu=("u", "max"))
    exp = d.groupby("key", dropna=False).agg(**named).reset_index()
    assert_frames(got, exp, float_cols=("sv", "av"), sort_by=["key"])


def test_join_agg_fused_global_aggregates():
    """Aggregate(no GROUP BY) <- Inner Join on a unique dense key runs as ONE pass over the probe side
    (b2_join_agg): mixed-side products / sums / differences, single-sided inputs, COUNT(*), NULLs on
    both sides, predicates on both sides, int and float payloads; against pandas on the merged frame."""
    from dask_sql_b200 import Context, executor
    rng = np.random.default_rng(12)
    nd, nf = 20_000, 400_003
    dim = pd.DataFrame({"pk": rng.permutation(nd) + 1000, "w": rng.integers(0, 1000, nd),
                        "r": np.where(rng.random(nd) < 0.05, np.nan, rng.random(nd) * 10),
                        "flag": rng.integers(0, 10, nd)})
    fact = pd.DataFrame({"fk": pd.array(np.where(rng.random(nf) < 0.01, None, rng.integers(1000, 1000 + int(nd * 1.25), nf)),
                                        dtype="Int64"),
                         "v": np.where(rng.random(nf) < 0.03, np.nan, rng.random(nf)),
                         "q": rng.integers(-50, 50, nf), "x": rng.integers(-100, 100, nf)})
    c = Context()
    c.create_table("fact", fact, npartitions=3, persist=True)
    c.create_table("dim", dim, persist=True)
    before = executor.stats.get("join_agg", 0)
    where = "FROM fact f JOIN dim d ON f.fk = d.pk WHERE f.x > -50 AND d.flag < 7"
    got1 = c.sql(f"SELECT SUM(f.v * d.w) AS s_vw, SUM(f.q * d.w) AS s_qw, SUM(d.r - f.v) AS s_rv, AVG(d.w) AS a_w, "
                 f"COUNT(*) AS n {where}", return_futures=False)
    got2 = c.sql(f"SELECT COUNT(f.v) AS n_v, MIN(f.q + d.w) AS mn, MAX(f.v * d.r) AS mx, SUM(f.q) AS s_q {where}",
                 return_futures=False)
    assert executor.stats.get("join_agg", 0) == before + 2
    got = pd.concat([got1, got2], axis=1)
    j = fact[fact.x > -50].dropna(subset=["fk"]).astype({"fk": "int64"}).merge(dim[dim.flag < 7], left_on="fk", right_on="pk")
    exp = {"s_vw": (j.v * j.w).sum(), "s_qw": int((j.q * j.w).sum()), "s_rv": (j.r - j.v).sum(), "a_w": j.w.mean(),
           "n": len(j), "n_v": int(j.v.count()), "mn": int((j.q + j.w).min()), "mx": (j.v * j.r).max(),
           "s_q": int(j.q.sum())}
    assert len(got) == 1
    for k in ("s_qw", "n", "n_v", "mn", "s_q"):
        assert int(got[k][0]) == exp[k], k
    for k in ("s_vw", "s_rv", "a_w", "mx"):
        np.testing.assert_allclose(float(got[k][0]), exp[k], rtol=RTOL, err_msg=k)
    # no match at all -> zero rows, like the reference's groupby over an empty frame
    got = c.sql("SELECT SUM(f.v * d.w) AS s FROM fact f JOIN dim d ON f.fk = d.pk WHERE d.flag > 100",
                return_futures=False)
    assert len(got) == 0


def test_join_agg_falls_back_on_duplicate_build_keys():
    from dask_sql_b200 import Context
    dim = pd.DataFrame({"pk": [1, 2, 2, 3], "w": [10, 20, 30, 40]})
    fact = pd.DataFrame({"fk": [1, 2, 3, 3, 9], "v": [1.0, 2.0, 3.0, 4.0, 5.0]})
    c = Context()
    c.create_table("fact", fact, persist=True)
    c.create_table("dim", dim, persist=True)
    got = c.sql("SELECT SUM(f.v * d.w) AS s, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk", return_futures=False)
    j = fact.merge(dim, left_on="fk", right_on="pk")
    assert int(got.n[0]) == len(j)
    np.testing.assert_allclose(float(got.s[0]), (j.v * j.w).sum(), rtol=RTOL)


@pytest.mark.parametrize("mode", ["hot", "warp", "warp_only"])
@pytest.mark.parametrize("nullable_key", [False, True])
def test_groupby_skewed_keys_preaggregate(mode, nullable_key, monkeypatch):
    """Keys that repeat inside a warp (Zipf-like) do not take one global atomic per row: "hot" = the
    sampled heavy hitters accumulate in thread-private shared-memory partials (b2_hot_slots +
    b2_groupby_dense_hot); "warp" = per-warp match/shuffle pre-aggregation + a per-CTA table of claimed
    slots (b2_groupby_dense_grouped), "warp_only" without that table.  Every accumulator kind, NULL
    inputs, a predicate, NULL keys, zero-valued rows, a ragged tail; against pandas."""
    from dask_sql_b200 import executor
    monkeypatch.setenv("B200SQL_SKEW", "hot" if mode == "hot" else "warp")
    if mode == "warp_only":
        monkeypatch.setenv("B200SQL_NO_HOT_TABLE", "1")
    rng = np.random.default_rng(91)
    n, nkeys = 400_037, 3_000
    w = 1.0 / np.arange(1, nkeys + 1) ** 1.1
    key = rng.permutation(nkeys)[rng.choice(nkeys, size=n, p=w / w.sum())] + 50
    df = pd.DataFrame({
        "key": pd.array(np.where(rng.random(n) < 0.03, None, key), dtype="Int64") if nullable_key else key,
        "v": rng.random(n), "w": rng.integers(-100, 100, n),
        "g": np.where(rng.random(n) < 0.2, np.nan, rng.random(n)), "x": rng.integers(0, 10, n),
        "z": np.where(key % 2 == 0, 0.0, -0.0)})          # sums of +-0.0 only: existence must not hinge on the value
    spec = [("v", "sv", "sum"), ("w", "sw", "sum"), ("w", "aw", "mean"), ("g", "cg", "count"), ("g", "sg", "sum"),
            ("w", "mn", "min"), ("g", "mx", "max"), (None, "n", "size")]
    before = executor.stats.get("grouped_groupby", 0)
    f = _table(df, 3)
    got = agg(f[f["x"] > 1], ["key"], spec)
    assert executor.stats.get("grouped_groupby", 0) == before + 1
    d = df[df["x"] > 1]
    exp = d.groupby("key", dropna=False).agg(sv=("v", "sum"), sw=("w", "sum"), aw=("w", "mean"), cg=("g", "count"),
                                             sg=("g", lambda s: s.sum(min_count=1)), mn=("w", "min"),
                                             mx=("g", "max"), n=("v", "size")).reset_index()
    assert_frames(got, exp, float_cols=("sv", "aw", "sg"), sort_by=["key"])
    # a single float SUM over a never-NULL column: the accumulator doubles as the existence flag
    got = agg(f, ["key"], [("v", "sv", "sum")])
    exp = df.groupby("key", dropna=False).agg(sv=("v", "sum")).reset_index()
    assert_frames(got, exp, float_cols=("sv",), sort_by=["key"])
    got = agg(f, ["key"], [("z", "sz", "sum")])             # every group exists although every sum is 0.0
    exp = df.groupby("key", dropna=False).agg(sz=("z", "sum")).reset_index()
    assert_frames(got, exp, float_cols=("sz",), sort_by=["key"])


def test_uniform_keys_keep_the_per_row_atomic_kernel():
    from dask_sql_b200 import executor
    rng = np.random.default_rng(92)
    df = pd.DataFrame({"key": rng.integers(0, 1_000_000, 300_000), "v": rng.random(300_000)})
    before = executor.stats.get("grouped_groupby", 0)
    got = agg(_table(df, 2), ["key"], [("v", "sv", "sum")])
    assert executor.stats.get("grouped_groupby", 0) == before
    assert_frames(got, df.groupby("key").agg(sv=("v", "sum")).reset_index(), float_cols=("sv",), sort_by=["key"])


@pytest.mark.parametrize("pcol,bcol,op", [("v", "w", "*"), ("v", "big", "+"), ("q", "w", "*"), ("q", "r", "-"),
                                          ("v", "r", "*"), ("q", "big", "-")])
def test_join_agg_single_sum_fast_path(pcol, bcol, op, monkeypatch):
    """SUM(P o B) alone takes the specialised kernel: float / int probe column x payload stored as uint32
    with the absent-key sentinel, wide int64, float64; NaNs on either side are skipped; a probe filter."""
    from dask_sql_b200 import Context, executor
    rng = np.random.default_rng(33)
    nd, nf = 30_000, 300_017
    dim = pd.DataFrame({"pk": rng.permutation(nd * 2)[:nd] - 100, "w": rng.integers(0, 5000, nd),
                        "big": rng.integers(-2**40, 2**40, nd),
                        "r": np.where(rng.random(nd) < 0.05, np.nan, rng.random(nd) * 10)})
    fact = pd.DataFrame({"fk": rng.integers(-500, nd * 2 + 300, nf),
                         "v": np.where(rng.random(nf) < 0.03, np.nan, rng.random(nf)),
                         "q": rng.integers(-50, 50, nf), "x": rng.integers(-100, 100, nf)})
    c = Context()
    c.create_table("fact", fact, npartitions=3, persist=True)
    c.create_table("dim", dim, persist=True)
    lhs, rhs = (f"d.{bcol}", f"f.{pcol}") if (op == "-" and bcol == "big") else (f"f.{pcol}", f"d.{bcol}")
    q = f"SELECT SUM({lhs} {op} {rhs}) AS s FROM fact f JOIN dim d ON f.fk = d.pk WHERE f.x > -60"
    j = fact[fact.x > -60].merge(dim, left_on="fk", right_on="pk")
    a, b = (j[bcol], j[pcol]) if lhs.startswith("d.") else (j[pcol], j[bcol])
    exp = {"*": a * b, "+": a + b, "-": a - b}[op].sum()
    before = executor.stats.get("join_agg", 0)
    got = c.sql(q, return_futures=False)
    assert executor.stats.get("join_agg", 0) == before + 1
    monkeypatch.setenv("B200SQL_JA_GENERIC", "1")
    generic = c.sql(q, return_futures=False)
    if np.issubdtype(type(exp), np.integer) or isinstance(exp, (int, np.integer)):
        assert int(got.s[0]) == int(exp) == int(generic.s[0])
    else:
        np.testing.assert_allclose([float(got.s[0]), float(generic.s[0])], [exp, exp], rtol=RTOL)
