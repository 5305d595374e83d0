"""RAND / RANDOM / RAND_INTEGER and TABLESAMPLE through SQL, checked value for value against the NumPy restatement
of the contract (tests/rand_ref.py): the same column and the same sample at any partitioning and from Parquet,
BERNOULLI on each executor path against tests/query_ref.py over the rows the reference mask keeps, and SYSTEM's
choice of partitions and Parquet row groups."""
import numpy as np
import pandas as pd
import pytest

from tests import rand_ref as RR

pytestmark = pytest.mark.gpu

N = 20_011


@pytest.fixture()
def c():
    from dask_sql_b200 import Context
    return Context()


def _frame(n=N, seed=5):
    rng = np.random.default_rng(seed)
    return pd.DataFrame({"id": np.arange(n, dtype=np.int64), "k": rng.integers(0, 50, n),
                         "h": rng.integers(-2 ** 40, 2 ** 40, n), "x": rng.random(n)})


def _parquet(tmp_path, df, rows_per_group):
    import pyarrow as pa
    import pyarrow.parquet as pq
    path = str(tmp_path / "t.parquet")
    pq.write_table(pa.Table.from_pandas(df, preserve_index=False), path, row_group_size=rows_per_group)
    return path


def _stat(name):
    from dask_sql_b200 import executor
    return executor.stats.get(name, 0)


def test_random(c):
    """the reference's test_random (tests/integration/test_rex.py:143-180); RAND_INTEGER is int64 here"""
    q = 'SELECT RAND(0) AS "0", RAND_INTEGER(0, 10) AS "1"'
    a, b = c.sql(q).compute(), c.sql(q).compute()
    pd.testing.assert_frame_equal(a, b)
    assert a["0"].dtype == "float64" and a["1"].dtype == "int64"
    assert 0 <= a["0"][0] < 1 and 0 <= a["1"][0] < 10
    assert a["0"][0] == RR.rand([0], 0, 1)[0] and a["1"][0] == RR.rand_integer([0], 0, 2, 10)[0]
    r = c.sql('SELECT RAND() AS "0", RANDOM() AS "1", RAND_INTEGER(30) AS "2"').compute()
    assert r["0"].dtype == "float64" and r["1"].dtype == "float64" and r["2"].dtype == "int64"
    assert 0 <= r["0"][0] < 1 and 0 <= r["1"][0] < 1 and 0 <= r["2"][0] < 30


def _sources(c, tmp_path, df):
    """the same rows as tables of 1, 5 and 100 partitions and a Parquet file of many row groups"""
    names = []
    for k in (1, 5, 100):
        c.create_table(f"t{k}", df, npartitions=k)
        names.append(f"t{k}")
    c.create_table("tp", _parquet(tmp_path, df, 1500))
    names.append("tp")
    return names


def test_rand_column_and_sample_do_not_depend_on_partitioning(c, tmp_path):
    df = _frame()
    rows = df["id"].to_numpy()
    want_r = RR.rand(rows, RR.key_of(7), 1)
    want_i = RR.rand_integer(rows, RR.key_of(7), 2, 1000)
    keep = RR.bernoulli_mask(rows, RR.key_of(3), 1, 10)
    for t in _sources(c, tmp_path, df):
        got = c.sql(f"SELECT id, RAND(7) AS r, RAND_INTEGER(7, 1000) AS i FROM {t}").compute()
        np.testing.assert_array_equal(got["id"].to_numpy(), rows, err_msg=t)
        np.testing.assert_array_equal(got["r"].to_numpy(), want_r, err_msg=t)
        np.testing.assert_array_equal(got["i"].to_numpy(), want_i, err_msg=t)
        before = _stat("sample_masks")
        s = c.sql(f"SELECT id FROM {t} TABLESAMPLE BERNOULLI (10) REPEATABLE (3)").compute()
        np.testing.assert_array_equal(np.sort(s["id"].to_numpy()), rows[keep], err_msg=t)
        assert _stat("sample_masks") > before


COUNTERS = ("dense_groupby", "partitioned_groupby", "hash_groupby", "star_fused", "join_agg", "dense_join",
            "chain_join", "keyed_join")


def _path(c, sql, moved=(), unmoved=()):
    """run `sql` over a sampled table: the BERNOULLI mask was launched, every counter in `moved` moved and
    none in `unmoved` did"""
    before = {k: _stat(k) for k in COUNTERS + ("sample_masks",)}
    got = c.sql(sql).compute()
    after = {k: _stat(k) for k in COUNTERS + ("sample_masks",)}
    assert after["sample_masks"] > before["sample_masks"], sql
    for m in moved:
        assert after[m] > before[m], f"path {m} did not run: {before} -> {after}\n{sql}"
    for m in unmoved:
        assert after[m] == before[m], f"path {m} ran: {before} -> {after}\n{sql}"
    return got


@pytest.mark.parametrize("npart", [1, 7])
def test_bernoulli_on_each_path(c, monkeypatch, npart):
    """fused global aggregate, filtered select, dense, range-partitioned and hash group-by, join with the sampled
    side probing and building, join-aggregate, and the Q3 shape, each over a sampled table"""
    df = _frame().assign(r=lambda f: np.random.default_rng(8).integers(0, 3000, len(f)))
    c.create_table("t", df, npartitions=npart, persist=True)
    dim = pd.DataFrame({"pk": np.arange(50, dtype=np.int64), "g": np.arange(50, dtype=np.int64) % 7})
    dim["gf"] = dim["g"] * 0.5 - 1.0
    c.create_table("d", dim, persist=True)
    keep = RR.bernoulli_mask(df["id"].to_numpy(), RR.key_of(11), 1, 25)
    sub = df[keep]
    samp = "t TABLESAMPLE BERNOULLI (25) REPEATABLE (11)"

    got = _path(c, f"SELECT COUNT(*) AS n, SUM(h) AS s, MIN(x) AS m FROM {samp} WHERE k < 40", unmoved=COUNTERS)
    ref = sub[sub.k < 40]
    assert got["n"][0] == len(ref) and got["s"][0] == ref.h.sum() and got["m"][0] == ref.x.min()

    got = _path(c, f"SELECT id FROM {samp} WHERE x > 0.5", unmoved=COUNTERS)
    np.testing.assert_array_equal(np.sort(got["id"].to_numpy()), sub[sub.x > 0.5].id.to_numpy())

    got = _path(c, f"SELECT k, COUNT(*) AS n, SUM(h) AS s FROM {samp} GROUP BY k", ("dense_groupby",),
                ("partitioned_groupby", "hash_groupby")).sort_values("k")
    ref = sub.groupby("k").agg(n=("h", "size"), s=("h", "sum")).reset_index()
    np.testing.assert_array_equal(got[["k", "n", "s"]].to_numpy(), ref[["k", "n", "s"]].to_numpy())

    with monkeypatch.context() as m:
        m.setenv("B200SQL_PARTITION_MIN_BYTES", "0")
        m.setenv("B200SQL_PARTITION_BUCKET_BYTES", "512")
        got = _path(c, f"SELECT r, COUNT(*) AS n, SUM(h) AS s FROM {samp} GROUP BY r", ("partitioned_groupby",),
                    ("hash_groupby",)).sort_values("r")
    ref = sub.groupby("r").agg(n=("h", "size"), s=("h", "sum")).reset_index()
    np.testing.assert_array_equal(got[["r", "n", "s"]].to_numpy(), ref[["r", "n", "s"]].to_numpy())

    got = _path(c, f"SELECT h, COUNT(*) AS n FROM {samp} GROUP BY h", ("hash_groupby",))
    assert sorted(got["h"].tolist()) == sorted(sub.h.tolist()) and (got["n"] == 1).all()

    # the sampled side probes: d (50 unique dense keys) is the direct-address build side
    got = _path(c, f"SELECT t.id, d.g FROM {samp} JOIN d ON t.k = d.pk", ("dense_join",),
                ("chain_join",)).sort_values("id")
    np.testing.assert_array_equal(got["id"].to_numpy(), sub.id.to_numpy())
    np.testing.assert_array_equal(got["g"].to_numpy(), sub.k.to_numpy() % 7)

    # the sampled side builds: the mask filters the dimension rows that enter the table
    dkeep = RR.bernoulli_mask(np.arange(50), RR.key_of(2), 1, 50)
    got = _path(c, "SELECT t.id, d.pk FROM t JOIN d TABLESAMPLE BERNOULLI (50) REPEATABLE (2) ON t.k = d.pk",
                ("dense_join",)).sort_values("id")
    np.testing.assert_array_equal(got["id"].to_numpy(), df.id.to_numpy()[dkeep[df.k.to_numpy()]])

    got = _path(c, f"SELECT SUM(t.x * d.gf) AS s, COUNT(*) AS n FROM {samp} JOIN d ON t.k = d.pk WHERE t.x > 0.1",
                ("join_agg",), ("star_fused",))
    ref = sub[sub.x > 0.1]
    assert got["n"][0] == len(ref)
    np.testing.assert_allclose(got["s"][0], (ref.x * (ref.k % 7 * 0.5 - 1.0)).sum(), rtol=1e-12)

    # the Q3 shape over a sampled fact table: the star path declines a sampled side, so the query runs as the
    # direct-address join followed by the dense group-by
    got = _path(c, f"SELECT d.g, SUM(t.h) AS s FROM {samp} JOIN d ON t.k = d.pk WHERE t.x < 0.9 AND d.g < 5 "
                   "GROUP BY d.g", ("dense_join", "dense_groupby"), ("star_fused", "join_agg")).sort_values("g")
    ref = sub[(sub.x < 0.9) & (sub.k % 7 < 5)].assign(g=lambda f: f.k % 7).groupby("g").h.sum()
    np.testing.assert_array_equal(got["s"].to_numpy(), ref.to_numpy())


def test_system_keeps_the_partitions_the_reference_chooses(c, tmp_path):
    df = _frame()
    c.create_table("t", df, npartitions=40)
    key = RR.key_of(9)
    step = len(df) // 40 // 32 * 32 + 32
    part_of = df["id"].to_numpy() // step
    kept = RR.system_keep(40, key, 1, 30)
    got = c.sql("SELECT id FROM t TABLESAMPLE SYSTEM (30) REPEATABLE (9)").compute()
    np.testing.assert_array_equal(np.sort(got["id"].to_numpy()), df.id.to_numpy()[kept[part_of]])

    path = _parquet(tmp_path, df, 1000)
    c.create_table("tp", path)
    table = c.schema[c.schema_name].tables["tp"].df.source.table
    ngroups = table.num_row_groups
    kept = RR.system_keep(ngroups, key, 2, 30)          # RAND is call site 1, TABLESAMPLE call site 2
    got = c.sql("SELECT id, RAND(2) AS r FROM tp TABLESAMPLE SYSTEM (30) REPEATABLE (9)").compute()
    ids = np.sort(got["id"].to_numpy())
    np.testing.assert_array_equal(ids, df.id.to_numpy()[kept[df.id.to_numpy() // 1000]])
    np.testing.assert_array_equal(got.sort_values("id")["r"].to_numpy(), RR.rand(ids, RR.key_of(2), 1))
    assert table.stats["row_groups_sampled_out"] == ngroups - kept.sum()
    assert {g for g, _ in table._cache} == set(np.flatnonzero(kept).tolist()), "a dropped row group was read"


def test_rand_in_where_group_by_and_order_by(c):
    df = _frame()
    c.create_table("t", df, npartitions=3)
    rows = df.id.to_numpy()
    got = c.sql("SELECT id FROM t WHERE RAND(4) < 0.2").compute()
    np.testing.assert_array_equal(np.sort(got["id"].to_numpy()), rows[RR.rand(rows, 4, 1) < 0.2])

    got = c.sql("SELECT id, RAND(4) AS r FROM t WHERE k < 10").compute().sort_values("id")
    sel = rows[df.k.to_numpy() < 10]
    np.testing.assert_array_equal(got["r"].to_numpy(), RR.rand(sel, 4, 1))

    # a group key that is an expression reaches the aggregate as a column of the block below it
    got = c.sql("SELECT g, COUNT(*) AS n FROM (SELECT RAND_INTEGER(5, 10) AS g FROM t) s GROUP BY g").compute()
    got = got.sort_values("g")
    ref = np.bincount(RR.rand_integer(rows, 5, 1, 10), minlength=10)
    np.testing.assert_array_equal(got["n"].to_numpy(), ref)

    got = c.sql("SELECT id FROM t ORDER BY RAND(6) LIMIT 25").compute()
    np.testing.assert_array_equal(got["id"].to_numpy(), rows[np.argsort(RR.rand(rows, 6, 1), kind="stable")[:25]])

    got = c.sql("SELECT SUM(RAND(1)) AS s FROM t").compute()
    np.testing.assert_allclose(got["s"][0], RR.rand(rows, 1, 1).sum(), rtol=1e-12)


def test_alias_used_twice_is_one_call_site(c):
    df = _frame(1000)
    c.create_table("t", df, npartitions=2)
    got = c.sql("SELECT r, r * 2 AS r2 FROM (SELECT RAND() AS r FROM t) s").compute()
    np.testing.assert_array_equal(got["r"].to_numpy() * 2, got["r2"].to_numpy())
    two = c.sql("SELECT RAND() AS a, RAND() AS b FROM t").compute()
    assert (two["a"] != two["b"]).mean() > 0.99
    again = c.sql("SELECT RAND() AS a, RAND() AS b FROM t").compute()
    assert (two["a"] != again["a"]).mean() > 0.99, "an unseeded statement drew the same key twice"


def test_rand_over_a_join_is_refused(c):
    c.create_table("t", _frame(100))
    c.create_table("u", _frame(100))
    with pytest.raises(NotImplementedError, match="one base table"):
        c.sql("SELECT RAND(1) AS r FROM t JOIN u ON t.id = u.id").compute()
    with pytest.raises(NotImplementedError, match="one base table"):
        c.sql("SELECT RAND(1) AS r FROM (SELECT k, COUNT(*) AS n FROM t GROUP BY k) a").compute()
