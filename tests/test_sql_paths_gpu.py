"""One query per execution path of the executor, through Context.sql(), against the exact reference of
tests/query_ref.py.  Every case records the executor's path counters before it runs and asserts that the
intended path's counter moved, so a threshold change that reroutes a case fails it instead of quietly testing
another path.  Paths are forced with the switches of DESIGN.md section 9, so small data reaches them.  Results
are read from the device columns (values + validity), not through pandas, so int64 results are compared as
integers and a NULL stays distinct from every value."""
import numpy as np
import pandas as pd
import pytest
import torch

from tests import query_ref as Q

pytestmark = pytest.mark.gpu

I64_MAX, I64_MIN = 2 ** 63 - 1, -(2 ** 63)
COUNTERS = ("dense_groupby", "grouped_groupby", "partitioned_groupby", "hash_groupby", "star_fused", "join_agg",
            "dense_join", "chain_join", "keyed_join")


@pytest.fixture()
def c():
    from dask_sql_b200 import Context
    return Context()


def _cells(col):
    """DeviceColumn -> query_ref cells"""
    from dask_sql_b200 import device as D
    from dask_sql_b200 import strings as S
    from dask_sql_b200.device import F64, U8
    n = col.n
    null = np.zeros(n, bool)
    if col.valid is not None:
        bits = col.valid.cpu().numpy().view(np.uint8)
        null = ~np.unpackbits(bits, bitorder="little")[:n].astype(bool)
    if S.is_varchar(col.logical):
        host = D.column_to_host(col)
        return [None if pd.isna(x) else str(x) for x in host]
    vals = col.data[:n].cpu().numpy()
    if col.dtype == F64:
        return [float("nan") if nl else float(v) for v, nl in zip(vals, null)]
    if col.dtype == U8:
        return [None if nl else bool(v) for v, nl in zip(vals, null)]
    return [None if nl else int(v) for v, nl in zip(vals.astype(np.int64), null)]


def _host_matches(col, cells, what):
    """the pandas column a Context.sql() user gets for the same device column: of the result's type (integers
    stay integers unless a NULL forces pandas' float64 promotion, booleans stay booleans, strings are a
    category) and holding the same values"""
    from dask_sql_b200 import device as D
    from dask_sql_b200 import strings as S
    from dask_sql_b200.device import F64, U8
    s = pd.Series(D.column_to_host(col))
    if S.is_varchar(col.logical):
        assert isinstance(s.dtype, pd.CategoricalDtype), f"{what}: VARCHAR comes back as {s.dtype}"
        return
    if col.dtype == U8:
        assert pd.api.types.is_bool_dtype(s.dtype), f"{what}: BOOLEAN comes back as {s.dtype}"
        assert [None if pd.isna(v) else bool(v) for v in s] == cells, what
    elif col.dtype == F64:
        assert pd.api.types.is_float_dtype(s.dtype), f"{what}: DOUBLE comes back as {s.dtype}"
        v = s.to_numpy(dtype=np.float64, na_value=np.nan)
        assert v.view(np.int64).tolist() == np.array(cells, np.float64).view(np.int64).tolist() or \
            np.array_equal(v, np.array(cells, np.float64), equal_nan=True), what
    elif col.logical.startswith(("int", "Int")):
        if pd.api.types.is_integer_dtype(s.dtype):
            assert [None if pd.isna(v) else int(v) for v in s] == cells, what
        else:          # numpy int64 cannot hold NULL: pandas promotes to float64, as the reference does
            assert s.dtype == np.float64 and None in cells, f"{what}: BIGINT comes back as {s.dtype}"


def run(c, sql, moved, config=None, unmoved=(), ran=(), not_ran=()):
    """execute `sql`; assert that counter `moved` (a name, or a tuple of names that must all move) moved,
    every counter in `unmoved` did not, every kernel in `ran` was launched and none in `not_ran` was;
    -> {column: cells} read from the device columns (each also checked through the host conversion)"""
    from dask_sql_b200 import executor
    before = {k: executor.stats.get(k, 0) for k in COUNTERS}
    lazy = c.sql(sql, config_options=config)
    executor.kernel_events = []
    try:
        parts = [executor.gather_keyrange(p).resolve() for p in executor.execute(lazy, top=True)]
        torch.cuda.synchronize()
        kernels = {rec[0] for rec in executor.kernel_events}
    finally:
        executor.kernel_events = None
    got = {name: [] for name in lazy.columns}
    for p in parts:
        if p.n == 0:
            continue
        for name in lazy.columns:
            cells = _cells(p[name])
            _host_matches(p[name], cells, f"{name} of {sql}")
            got[name] += cells
    after = {k: executor.stats.get(k, 0) for k in COUNTERS}
    if moved is not None:
        names = (moved,) if isinstance(moved, str) else moved
        assert all(after[m] > before[m] for m in names), f"path {moved} did not run: {before} -> {after}\n{sql}"
    for m in unmoved:
        assert after[m] == before[m], f"path {m} ran: {before} -> {after}\n{sql}"
    for k in ran:
        assert k in kernels, f"{k} was not launched ({sorted(kernels)})\n{sql}"
    for k in not_ran:
        assert k not in kernels, f"{k} was launched\n{sql}"
    return got


def _aggs_sql(aggs):
    out = []
    for a in aggs:
        name, fn, arg = a[0], a[1], a[2] if len(a) > 2 else None
        f = {"count_star": "COUNT(*)", "count_distinct": f"COUNT(DISTINCT {arg})"}.get(fn)
        if f is None:
            f = f"{fn.upper()}({arg}{', ' + a[3] if len(a) > 3 else ''})"
        out.append(f"{f} AS {name}")
    return ", ".join(out)


def _keys(rng, n, lo, hi, null_frac=0.0):
    k = rng.integers(0, hi - lo + 1, n, dtype=np.uint64)
    k = (k + np.uint64(lo & (2 ** 64 - 1))).view(np.int64)      # lo + offset, wrapping like the kernels
    if null_frac:
        return pd.array(np.where(rng.random(n) < null_frac, None, k), dtype="Int64")
    return k


def _fact(n, kmin, kmax, seed, null_key=0.05):
    """key k in [kmin, kmax]; x: int64 near 2^62 (sums wrap), f: dyadic floats with +-0.0, b: boolean with NULLs,
    y: Int64 with NULLs"""
    rng = np.random.default_rng(seed)
    return pd.DataFrame({
        "k": _keys(rng, n, kmin, kmax, null_key),
        "x": (2 ** 62 + rng.integers(-2 ** 40, 2 ** 40, n)).astype(np.int64),
        "f": rng.choice(np.array([0.0, -0.0, 0.5, -0.5, 3.25, -1e3, 1e3]), n),
        "b": pd.array(np.where(rng.random(n) < 0.1, None, rng.random(n) < 0.9), dtype="boolean"),
        "y": pd.array(np.where(rng.random(n) < 0.2, None, rng.integers(-2 ** 62, 2 ** 62, n)), dtype="Int64"),
        "i": np.arange(n, dtype=np.int64)})


# two queries: one GROUP BY holds at most 8 accumulators
DENSE_AGGS = ([("n", "count_star"), ("ny", "count", "y"), ("sx", "sum", "x"), ("sy", "sum", "y"), ("lo", "min", "f"),
               ("hi", "max", "f"), ("sf", "sum", "f"), ("ax", "avg", "x")],
              [("n", "count_star"), ("ba", "bit_and", "y"), ("bo", "bit_or", "y"), ("bx", "bit_xor", "y"),
               ("ev", "every", "b")])
# key ranges: ordinary, and the int64 edges (a dense table whose range starts at INT64_MIN or ends at INT64_MAX)
RANGES = {"mid": (-20, 40), "min": (I64_MIN, I64_MIN + 60), "max-1": (I64_MAX - 61, I64_MAX - 1),
          "max": (I64_MAX - 60, I64_MAX)}


def _group_case(c, df, npart, aggsets, moved, where=None, mask=None, config=None, unmoved=()):
    """aggsets: a list of aggregates, or a tuple of such lists (one query each)"""
    c.create_table("t", df, npartitions=npart)
    w = f" WHERE {where}" if where else ""
    rel = Q.table(df)
    for aggs in aggsets if isinstance(aggsets, tuple) else (aggsets,):
        got = run(c, f"SELECT k, {_aggs_sql(aggs)} FROM t{w} GROUP BY k", moved, config, unmoved)
        Q.assert_result(got, Q.aggregate(rel, ["k"], aggs, mask=None if mask is None else mask(rel)))


# ---- global aggregate: no group counter moves ------------------------------------------------------------------
@pytest.mark.parametrize("n,npart", [(0, 1), (1, 1), (33, 3), (4097, 3)])
@pytest.mark.parametrize("where", [None, "i >= 0", "i < 0"])
def test_global_aggregate(c, n, npart, where):
    df = _fact(n, -5, 5, seed=n)
    c.create_table("t", df, npartitions=npart)
    w = f" WHERE {where}" if where else ""
    rel = Q.table(df)
    mask = None if where is None else Q.cmp(rel["i"], where.split()[1], int(where.split()[2]))
    for aggs in DENSE_AGGS:
        got = run(c, f"SELECT {_aggs_sql(aggs)} FROM t{w}", None, unmoved=COUNTERS)
        Q.assert_result(got, Q.aggregate(rel, [], aggs, mask=mask))


# ---- dense group tables -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rng_name", list(RANGES))
@pytest.mark.parametrize("nullable", [True, False])
def test_dense_per_row_atomics(c, monkeypatch, rng_name, nullable):
    monkeypatch.setenv("B200SQL_NO_WARPAGG", "1")
    lo, hi = RANGES[rng_name]
    df = _fact(20_000, lo, hi, seed=1, null_key=0.05 if nullable else 0.0)
    df.loc[0, "k"], df.loc[1, "k"] = lo, hi     # the range ends where it says: both ends present
    _group_case(c, df, 3, DENSE_AGGS, "dense_groupby", unmoved=("hash_groupby", "partitioned_groupby"))


@pytest.mark.parametrize("skew", ["hot", "warp"])
@pytest.mark.parametrize("rng_name", list(RANGES))
def test_dense_skewed_keys(c, monkeypatch, skew, rng_name):
    monkeypatch.setenv("B200SQL_SKEW", skew)
    lo, _ = RANGES[rng_name]
    rng = np.random.default_rng(2)
    n = 200_000
    df = _fact(n, 0, 0, seed=2, null_key=0.0)
    off = np.minimum(rng.zipf(1.2, n), 60).astype(np.int64) - 1
    df["k"] = (off.astype(np.uint64) + np.uint64(lo & (2 ** 64 - 1))).view(np.int64)
    df.loc[0, "k"] = RANGES[rng_name][1]           # the range ends where it says
    aggs = [("n", "count_star"), ("sx", "sum", "x"), ("sf", "sum", "f"), ("hi", "max", "f")]
    _group_case(c, df, 2, aggs, "grouped_groupby", where="f <> 0.5",
                mask=lambda r: Q.cmp(r["f"], "<>", 0.5), unmoved=("hash_groupby",))


@pytest.mark.parametrize("indicator", [True, False])
@pytest.mark.parametrize("rng_name", list(RANGES))
def test_dense_float_sum_existence_mark(c, monkeypatch, indicator, rng_name):
    """a float SUM alone over a NaN-free column: the -0.0 start value marks the groups (indicator) or the
    presence bitmap does.  Groups whose rows sum to zero, or hold only -0.0, are still groups, with SUM +0.0;
    groups whose rows are all filtered are not."""
    if not indicator:
        monkeypatch.setenv("B200SQL_NO_INDICATOR", "1")
    lo, hi = RANGES[rng_name]
    rng = np.random.default_rng(3)
    n = 30_000
    k = _keys(rng, n, lo, hi)
    k[:2] = lo, hi
    f = rng.choice(np.array([-0.0, 0.25, -0.25, 2.0, -2.0]), n)
    off = (k.view(np.uint64) - np.uint64(lo & (2 ** 64 - 1))).astype(np.int64)
    f[off % 7 == 0] = -0.0                  # groups of -0.0 only
    f[off % 7 == 1] = np.where(np.arange((off % 7 == 1).sum()) % 2, 0.25, -0.25)    # cancelling
    df = pd.DataFrame({"k": k, "f": f, "i": np.arange(n)})
    _group_case(c, df, 3, [("sf", "sum", "f")], "dense_groupby", where="i % 5 <> 1",
                mask=lambda r: np.arange(n) % 5 != 1)


@pytest.mark.parametrize("rng_name", list(RANGES))
@pytest.mark.parametrize("split_out", [1, 3])
def test_dense_not_deferred(c, monkeypatch, rng_name, split_out):
    monkeypatch.setenv("B200SQL_NO_DEFER", "1")
    lo, hi = RANGES[rng_name]
    df = _fact(10_000, lo, hi, seed=4, null_key=0.0)
    df.loc[0, "k"], df.loc[1, "k"] = lo, hi
    _group_case(c, df, 1, DENSE_AGGS, "dense_groupby", config={"sql.aggregate.split_out": split_out})


@pytest.mark.parametrize("rng_name", list(RANGES))
def test_range_partitioned(c, monkeypatch, rng_name):
    """the range-partitioned, ordered dense path: several buckets, a nullable key, a predicate"""
    monkeypatch.setenv("B200SQL_PARTITION_MIN_BYTES", "0")
    monkeypatch.setenv("B200SQL_PARTITION_BUCKET_BYTES", "512")
    lo = {"mid": -3000, "min": I64_MIN, "max-1": I64_MAX - 3001, "max": I64_MAX - 3000}[rng_name]
    hi = lo + 3000
    df = _fact(40_000, lo, hi, seed=5, null_key=0.05)
    df.loc[0, "k"], df.loc[1, "k"] = lo, hi
    aggs = [("n", "count_star"), ("sx", "sum", "x"), ("sf", "sum", "f"), ("lo", "min", "f")]
    _group_case(c, df, 3, aggs, "partitioned_groupby", where="i % 3 <> 0", mask=lambda r: np.arange(40_000) % 3 != 0)


# ---- hash group tables --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("split_out", [1, 3])
def test_hash1_int64_extremes(c, split_out):
    rng = np.random.default_rng(6)
    n = 50_000
    k = rng.choice(np.array([I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, 0, -1, 2 ** 53 + 1, 2 ** 53], np.int64), n)
    df = _fact(n, 0, 0, seed=6)
    df["k"] = pd.array(np.where(rng.random(n) < 0.05, None, k), dtype="Int64")
    _group_case(c, df, 3, DENSE_AGGS, "hash_groupby", config={"sql.aggregate.split_out": split_out})


def test_hash1_float_key(c):
    rng = np.random.default_rng(7)
    n = 40_000
    nan2 = np.array([0x7FF8000000000001], np.int64).view(np.float64)[0]
    df = _fact(n, 0, 0, seed=7)
    df["k"] = rng.choice(np.array([0.0, -0.0, np.nan, nan2, np.inf, -np.inf, 5e-324, 2.0 ** 53]), n)
    _group_case(c, df, 3, [("n", "count_star"), ("sx", "sum", "x"), ("lo", "min", "f"), ("d", "count_distinct", "f")],
                "hash_groupby")


@pytest.mark.parametrize("keys,path", [(["k"], "dense_groupby"), (["k", "ks"], "hash_groupby"),
                                       (["k", "ks", "b"], "hash_groupby")])
def test_count_distinct_of_the_null_group(c, keys, path):
    """DISTINCT aggregates run as a second pass joined back to the first by group key: the NULL group must meet
    itself there (an equi-join never matches NULL keys)"""
    rng = np.random.default_rng(12)
    n = 20_000
    df = _fact(n, -5, 5, seed=12, null_key=0.1)
    df["ks"] = pd.Series(np.where(rng.random(n) < 0.2, None, rng.choice(["p", "q"], n)), dtype="category")
    c.create_table("t", df, npartitions=3)
    aggs = [("n", "count_star"), ("sx", "sum", "x"), ("d", "count_distinct", "f"), ("dy", "count_distinct", "y")]
    got = run(c, f"SELECT {', '.join(keys)}, {_aggs_sql(aggs)} FROM t GROUP BY {', '.join(keys)}", path)
    Q.assert_result(got, Q.aggregate(Q.table(df), keys, aggs))


@pytest.mark.parametrize("keys", [["ki", "kf"], ["ks", "kf", "ki"], ["kb", "ks", "ki"], ["ks", "kf", "kb", "ki"]])
def test_hashk_mixed_keys(c, keys):
    rng = np.random.default_rng(8)
    n = 30_000
    df = _fact(n, 0, 0, seed=8)
    df["ki"] = pd.array(np.where(rng.random(n) < 0.1, None, rng.choice([I64_MIN, I64_MAX, 0, 7], n)), dtype="Int64")
    df["kf"] = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -np.inf]), n)
    df["kb"] = pd.array(np.where(rng.random(n) < 0.1, None, rng.random(n) < 0.5), dtype="boolean")
    df["ks"] = pd.Series(np.where(rng.random(n) < 0.1, None, rng.choice(["a", "b", "é", ""], n)), dtype="category")
    c.create_table("t", df, npartitions=3)
    aggs = [("n", "count_star"), ("sx", "sum", "x"), ("hi", "max", "f"), ("ev", "every", "b")]
    got = run(c, f"SELECT {', '.join(keys)}, {_aggs_sql(aggs)} FROM t GROUP BY {', '.join(keys)}", "hash_groupby")
    Q.assert_result(got, Q.aggregate(Q.table(df), keys, aggs), what=str(keys))


def test_variance_and_regr(c):
    rng = np.random.default_rng(9)
    n = 20_000
    df = pd.DataFrame({"k": rng.integers(0, 30, n), "x": 1e6 + rng.normal(0, 3, n), "y": rng.normal(0, 1, n)})
    df.loc[rng.random(n) < 0.1, "x"] = np.nan
    df.loc[rng.random(n) < 0.1, "y"] = np.nan
    df.loc[:2, "k"] = [100, 101, 101]
    aggs = [("vs", "var_samp", "x"), ("vp", "var_pop", "x"), ("ss", "stddev_samp", "x"), ("sp", "stddev_pop", "x"),
            ("sxx", "regr_sxx", "y", "x"), ("syy", "regr_syy", "y", "x"), ("rc", "regr_count", "y", "x")]
    _group_case(c, df, 3, aggs, "dense_groupby")


# ---- star join ------------------------------------------------------------------------------------------------------
def _star(nd=2000, nf=100_000, glo=0, ghi=49, seed=10, dup=False):
    rng = np.random.default_rng(seed)
    pk = rng.permutation(nd).astype(np.int64)
    if dup:
        pk[1] = pk[0]
    g = _keys(rng, nd, glo, ghi)
    g[:2] = glo, ghi
    dim = pd.DataFrame({"pk": pk, "flag": rng.integers(0, 10, nd), "g": g})
    if dup:
        dim.loc[:1, "flag"] = 0                      # both copies of the key pass the dim predicate
    fact = pd.DataFrame({"fk": rng.integers(-5, nd + 5, nf), "x": rng.integers(-100, 100, nf),
                         "v": rng.integers(-2 ** 20, 2 ** 20, nf) * 2.0 ** -10,
                         "w": (2 ** 62 + rng.integers(0, 2 ** 40, nf)).astype(np.int64)})
    return dim, fact


STAR_SQL = ("SELECT d.g AS g, SUM(f.v) AS s, SUM(f.w) AS sw, COUNT(*) AS n, MAX(f.v) AS hi FROM fact f "
            "JOIN dim d ON f.fk = d.pk WHERE f.x > {x} AND d.flag < {fl} GROUP BY d.g")


def _star_ref(dim, fact, x, fl):
    j = Q.join(Q.table(fact), Q.table(dim), ["fk"], ["pk"], "inner")
    mask = Q.cmp(j["x"], ">", x) & Q.cmp(j["flag"], "<", fl)
    return Q.aggregate(j, ["g"], [("s", "sum", "v"), ("sw", "sum", "w"), ("n", "count_star"), ("hi", "max", "v")],
                       mask=mask)


@pytest.mark.parametrize("grange", ["mid", "min", "max-1", "max"])
@pytest.mark.parametrize("prepared", [True, False])
def test_star(c, monkeypatch, grange, prepared):
    if not prepared:
        monkeypatch.setenv("B200SQL_NO_PREPARED", "1")
    glo, ghi = {"mid": (0, 49), "min": (I64_MIN, I64_MIN + 49), "max-1": (I64_MAX - 50, I64_MAX - 1),
                "max": (I64_MAX - 49, I64_MAX)}[grange]
    dim, fact = _star(glo=glo, ghi=ghi)
    c.create_table("fact", fact, npartitions=3, persist=True)
    c.create_table("dim", dim, persist=True)
    for x, fl in ((0, 5), (-50, 9)):                  # the second run: other literals (a prepared plan's re-run)
        got = run(c, STAR_SQL.format(x=x, fl=fl), "star_fused")
        Q.assert_result(got, _star_ref(dim, fact, x, fl), what=f"x > {x}, flag < {fl}")


def test_star_duplicate_pk_falls_back(c):
    dim, fact = _star(dup=True)
    c.create_table("fact", fact, npartitions=3, persist=True)
    c.create_table("dim", dim, persist=True)
    from dask_sql_b200 import executor
    before = executor.stats["star_fused"]
    got = run(c, STAR_SQL.format(x=0, fl=5), None)
    assert executor.stats["star_fused"] == before, "a duplicate build key must leave the star path"
    Q.assert_result(got, _star_ref(dim, fact, 0, 5))


# ---- join + global aggregate -----------------------------------------------------------------------------------
@pytest.mark.parametrize("generic", [False, True])
def test_join_aggregate(c, monkeypatch, generic):
    if generic:
        monkeypatch.setenv("B200SQL_JA_GENERIC", "1")
    dim, fact = _star()
    dim["p"] = np.arange(len(dim)) * 0.5 - 300.0
    c.create_table("fact", fact, npartitions=3, persist=True)
    c.create_table("dim", dim, persist=True)
    got = run(c, "SELECT SUM(f.v * d.p) AS s, SUM(d.p) AS sp, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk "
                 "WHERE f.x > 10", "join_agg")
    j = Q.join(Q.table(fact), Q.table(dim), ["fk"], ["pk"], "inner")
    j["vp"] = Q.Column(j["v"].values * j["p"].values, None, Q.F64)
    exp = Q.aggregate(j, [], [("s", "sum", "vp"), ("sp", "sum", "p"), ("n", "count_star")], mask=Q.cmp(j["x"], ">", 10))
    Q.assert_result(got, exp)


# ---- general joins -----------------------------------------------------------------------------------------------
def _join_frames(kind, seed=11):
    rng = np.random.default_rng(seed)
    na, nb = 5000, (3000 if kind in ("int", "dup") else 40)     # few distinct keys: a small build side
    if kind == "int":
        ka = rng.integers(-50, 3000, na).astype(np.int64)
        kb = rng.permutation(3000).astype(np.int64)            # unique, dense: the direct-address table
    elif kind == "dup":
        ka = rng.integers(0, 400, na).astype(np.int64)
        kb = rng.integers(0, 400, nb).astype(np.int64)
    elif kind == "edge":                                         # int against float at 2^53 +- 1
        e = np.array([2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 0, -1], np.int64)
        ka = rng.choice(e, na)
        kb = rng.choice(np.array([2.0 ** 53, 2.0 ** 53 - 1, -0.0, np.nan, 7.0]), nb)
    else:                                                        # VARCHAR keys of two dictionaries
        ka = pd.Series(rng.choice(["x", "y", "zz", "é", None], na), dtype="category")
        kb = pd.Series(rng.choice(["y", "zz", "w", None, "é"], nb), dtype="category")
    a = pd.DataFrame({"ak": ka, "ai": np.arange(na), "av": rng.integers(-9, 9, na)})
    b = pd.DataFrame({"bk": kb, "bi": np.arange(nb), "bv": rng.integers(-9, 9, nb) * 0.5})
    return a, b


def _join_path(kind, how, switch=None):
    """run() arguments for the path a join must take: a unique dense int64 build side is the direct-address
    table (dense_join), probed in one pass and with key-ordered payloads unless a switch or FULL JOIN rules
    them out; RIGHT JOIN builds the left input, whose keys repeat, and every other key kind is a chained table"""
    dense = kind == "int" and how != "right"
    if not dense:
        return dict(moved="chain_join", unmoved=("dense_join", "keyed_join"), not_ran=("b2_join_onepass",))
    keyed = how != "full" and switch != "B200SQL_NO_KEY_LAYOUT"
    onepass = how != "full" and switch != "B200SQL_NO_ONEPASS"
    return dict(moved=("dense_join", "keyed_join") if keyed else "dense_join",
                unmoved=("chain_join",) + (() if keyed else ("keyed_join",)),
                ran=("b2_join_onepass",) if onepass else (), not_ran=() if onepass else ("b2_join_onepass",))


@pytest.mark.parametrize("how", ["inner", "left", "right", "full", "semi", "anti"])
@pytest.mark.parametrize("kind", ["int", "dup", "edge", "str"])
def test_join(c, how, kind):
    a, b = _join_frames(kind)
    c.create_table("a", a, npartitions=3)
    c.create_table("b", b, npartitions=2)
    op = {"semi": "LEFT SEMI", "anti": "LEFT ANTI"}.get(how, how.upper())
    cols = "a.ai AS ai, a.av AS av" + ("" if how in ("semi", "anti") else ", b.bi AS bi, b.bv AS bv")
    path = _join_path(kind, how)
    got = run(c, f"SELECT {cols} FROM a {op} JOIN b ON a.ak = b.bk", **path)
    rel = Q.join(Q.table(a), Q.table(b), ["ak"], ["bk"], how)
    names = ["ai", "av"] + ([] if how in ("semi", "anti") else ["bi", "bv"])
    Q.assert_result(got, Q.select(rel, names))


@pytest.mark.parametrize("switch", [None, "B200SQL_NO_ONEPASS", "B200SQL_NO_KEY_LAYOUT"])
@pytest.mark.parametrize("how", ["inner", "left"])
def test_join_then_group_and_order(c, monkeypatch, switch, how):
    if switch:
        monkeypatch.setenv(switch, "1")
    a, b = _join_frames("int")
    c.create_table("a", a, npartitions=3)
    c.create_table("b", b, npartitions=1)
    rel = Q.join(Q.table(a), Q.table(b), ["ak"], ["bk"], how)
    path = _join_path("int", how, switch)
    got = run(c, f"SELECT a.av AS av, COUNT(*) AS n, SUM(b.bv) AS s, MIN(b.bi) AS m FROM a {how.upper()} JOIN b "
                 f"ON a.ak = b.bk GROUP BY a.av", **path)
    Q.assert_result(got, Q.aggregate(rel, ["av"], [("n", "count_star"), ("s", "sum", "bv"), ("m", "min", "bi")]))
    got = run(c, f"SELECT a.ai AS ai, b.bv AS bv, b.bi AS bi FROM a {how.upper()} JOIN b ON a.ak = b.bk "
                 f"ORDER BY bv DESC NULLS LAST, ai LIMIT 700 OFFSET 11", **path)
    exp = Q.order_by(Q.select(rel, ["ai", "bv", "bi"]), [("bv", True, False), ("ai", False)], 11, 700)
    Q.assert_result(got, exp)


# ---- ORDER BY / LIMIT over VARCHAR, nullable int, float and grouped results ---------------------------------------
@pytest.mark.parametrize("order,sql,window", [
    ([("ks", False, True), ("k", True, False), ("i", False)], "ks NULLS FIRST, k DESC NULLS LAST, i", (7, 100)),
    ([("ks", True), ("f", False), ("i", True)], "ks DESC, f, i DESC", (0, None)),
    ([("k", False, True), ("ks", False), ("f", True)], "k NULLS FIRST, ks, f DESC", (4000, 500)),   # cuts ties
])
def test_order_by(c, order, sql, window):
    rng = np.random.default_rng(13)
    n = 6000
    df = _fact(n, -3, 3, seed=13, null_key=0.1)
    df["ks"] = pd.Series(np.where(rng.random(n) < 0.1, None, rng.choice(["b", "a", "é", "B", ""], n)), dtype="category")
    c.create_table("t", df, npartitions=3)
    off, lim = window
    tail = (f" LIMIT {lim}" if lim is not None else "") + (f" OFFSET {off}" if off else "")
    got = run(c, f"SELECT ks, k, f, i FROM t ORDER BY {sql}{tail}", None)
    Q.assert_result(got, Q.order_by(Q.select(Q.table(df), ["ks", "k", "f", "i"]), order, off, lim))


def test_order_by_grouped_result_cut_inside_a_tie(c):
    """ORDER BY over a GROUP BY result whose float SUMs are not dyadic; the LIMIT cuts a run of tied counts"""
    rng = np.random.default_rng(14)
    n = 30_000
    df = pd.DataFrame({"k": rng.integers(0, 300, n), "v": rng.random(n) * 1e3 - 500, "c": rng.integers(0, 4, n)})
    c.create_table("t", df, npartitions=2)
    got = run(c, "SELECT k, COUNT(*) AS n, SUM(v) AS s FROM t GROUP BY k ORDER BY n DESC LIMIT 37", "dense_groupby")
    exp = Q.order_by(Q.aggregate(Q.table(df), ["k"], [("n", "count_star"), ("s", "sum", "v")]), [("n", True)], 0, 37)
    Q.assert_result(got, exp)


# ---- partitions of 0, 1, 33 and 4097 rows side by side ---------------------------------------------------------
@pytest.mark.parametrize("sizes", [(0, 1, 33, 4097), (4097, 0, 33, 1)])
@pytest.mark.parametrize("path", ["global", "dense", "hash"])
def test_uneven_partitions(c, sizes, path):
    """a table whose partitions hold 0, 1, 33 and 4097 rows, through the global, dense (key range ending at
    INT64_MAX) and hash paths"""
    from dask_sql_b200.table import DeviceTable
    lo, hi = RANGES["max"]
    df = _fact(sum(sizes), lo, hi, seed=15, null_key=0.05)
    if path == "hash":
        df["k"] = pd.array(np.where(df["k"].isna(), None, df["i"] * (2 ** 50) - 2 ** 62), dtype="Int64")
    bounds = np.cumsum((0,) + sizes)
    parts = [p for lo_, hi_ in zip(bounds[:-1], bounds[1:])
             for p in DeviceTable.from_pandas(df.iloc[lo_:hi_].reset_index(drop=True), persist=False).partitions]
    assert [next(iter(p.values())).n for p in parts] == list(sizes)
    c.create_table("t", DeviceTable(parts))
    rel = Q.table(df)
    for aggs in DENSE_AGGS:
        if path == "global":
            got = run(c, f"SELECT {_aggs_sql(aggs)} FROM t WHERE i % 2 = 0", None, unmoved=COUNTERS)
            Q.assert_result(got, Q.aggregate(rel, [], aggs, mask=np.arange(len(df)) % 2 == 0))
        else:
            got = run(c, f"SELECT k, {_aggs_sql(aggs)} FROM t GROUP BY k", f"{path}_groupby")
            Q.assert_result(got, Q.aggregate(rel, ["k"], aggs))
