"""VARCHAR end to end through Context.sql() on the GPU: the reference's known answers
(tests/golden/reference_strings.py), seeded comparisons with pandas for every predicate form, GROUP BY /
MIN / MAX / COUNT(DISTINCT) / DISTINCT / ORDER BY / LIMIT, every join type on string keys of two
dictionaries, round trips of every accepted input, the Q3 shape on string columns (fused star join, no
interpreter pass for its string predicates) and Parquet row-group pruning on a string-sorted file."""
import re

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from tests import strings_ref as R
from tests.golden import reference_strings as G

pytestmark = pytest.mark.gpu


def _ctx():
    import torch
    torch.cuda.set_device(0)
    from dask_sql_b200 import Context
    return Context()


def _strs(series):
    """a result column as Python values (None for NULL)"""
    return [None if (v is None or (isinstance(v, float) and v != v)) else v for v in series.astype(object)]


# ---- the reference's known answers -----------------------------------------------------------
@pytest.mark.parametrize("pred,rows", G.LIKE_CASES + G.FILTER_CASES)
def test_reference_golden_predicates(pred, rows):
    c = _ctx()
    c.create_table("string_table", pd.DataFrame({"a": G.STRING_TABLE}), dictionary=["a"])
    got = c.sql(f"SELECT * FROM string_table WHERE {pred}").compute()
    assert isinstance(got["a"].dtype, pd.CategoricalDtype)
    assert sorted(_strs(got["a"])) == sorted(G.STRING_TABLE[i] for i in rows)


@pytest.mark.parametrize("pred,rows", G.SIMILAR_CASES)
def test_reference_similar_to_raises(pred, rows):
    c = _ctx()
    c.create_table("string_table", pd.DataFrame({"a": pd.Series(G.STRING_TABLE, dtype="category")}))
    with pytest.raises(NotImplementedError):
        c.sql(f"SELECT * FROM string_table WHERE {pred}").compute()


def test_reference_sort():
    c = _ctx()
    c.create_table("string_table", pd.DataFrame({"a": pd.Series(G.SORT_TABLE, dtype="category")}))
    got = c.sql("SELECT * FROM string_table ORDER BY a").compute()
    assert _strs(got["a"]) == G.SORT_ASC


# ---- seeded comparisons with pandas ----------------------------------------------------------
WORDS = ["", "apple", "apricot", "banana", "BANANA", "band", "bandana", "cherry", "öl", "ölkanne", "zebra",
         "a%b", "a_b", "x\ny", "😀", "😀x", "中文", "date", "dates"]


def _frame(seed, n=3000, null_rate=0.1, words=WORDS):
    rng = np.random.default_rng(seed)
    s = np.array(words, dtype=object)[rng.integers(0, len(words), n)]
    s[rng.random(n) < null_rate] = None
    return pd.DataFrame({"s": s, "x": rng.integers(-1000, 1000, n), "v": rng.random(n)})


PREDICATES = [
    ("s = 'banana'", lambda s: s == "banana"),
    ("s = 'absent'", lambda s: s == "absent"),
    ("s <> 'banana'", lambda s: s != "banana"),
    ("s <> 'absent'", lambda s: True),
    ("s < 'band'", lambda s: s < "band"),
    ("s <= 'bane'", lambda s: s <= "bane"),
    ("s > 'öl'", lambda s: s > "öl"),
    ("s >= ''", lambda s: s >= ""),
    ("'cherry' > s", lambda s: "cherry" > s),
    ("s BETWEEN 'apple' AND 'bandz'", lambda s: "apple" <= s <= "bandz"),
    ("s NOT BETWEEN 'b' AND 'd'", lambda s: not ("b" <= s <= "d")),
    ("s IN ('apple', 'zebra', 'absent', '')", lambda s: s in ("apple", "zebra", "absent", "")),
    ("s NOT IN ('apple', 'absent')", lambda s: s not in ("apple", "absent")),    # NULL passes, as in pandas
    ("s LIKE 'ban%'", lambda s: R.like(s, "ban%")),
    ("s LIKE 'ö%'", lambda s: R.like(s, "ö%")),
    ("s LIKE '😀%'", lambda s: R.like(s, "😀%")),
    ("s LIKE 'band'", lambda s: s == "band"),
    ("s LIKE '%'", lambda s: True),
    ("s LIKE 'a\\%%'", lambda s: R.like(s, "a\\%%")),
    ("s LIKE '%an%'", lambda s: R.like(s, "%an%")),
    ("s LIKE '_'", lambda s: R.like(s, "_")),
    ("s LIKE 'x_y'", lambda s: R.like(s, "x_y")),
    ("s NOT LIKE '%an%'", lambda s: not R.like(s, "%an%")),
    ("s NOT LIKE 'ban%'", lambda s: not R.like(s, "ban%")),
    ("s ILIKE 'BAN%'", lambda s: R.like(s, "BAN%", ilike=True)),
    ("s NOT ILIKE '%A%'", lambda s: not R.like(s, "%A%", ilike=True)),
    ("s LIKE 'a!_b' ESCAPE '!'", lambda s: s == "a_b"),
    ("s IS NULL", None),
    ("s NOT LIKE '%'", lambda s: False),                # NULL LIKE '%' is NULL, and so is its NOT
    ("NOT (s LIKE '%%')", lambda s: False),
    ("NOT (s <> 'absent')", lambda s: False),
    ("NOT (s = 'absent')", lambda s: True),
    ("s LIKE 'ban%' AND x > 0", lambda s: R.like(s, "ban%")),
]


@pytest.mark.parametrize("sql,fn", PREDICATES, ids=[p for p, _ in PREDICATES])
def test_predicates_match_pandas(sql, fn):
    df = _frame(1)
    c = _ctx()
    c.create_table("t", df.assign(s=df["s"].astype("category")), npartitions=3)
    got = c.sql(f"SELECT x, s FROM t WHERE {sql}").compute()
    if fn is None:
        mask = df["s"].isna()
    else:
        mask = np.array([s is not None and bool(fn(s)) for s in _strs(df["s"])])
    if "x > 0" in sql:
        mask &= df["x"].to_numpy() > 0
    if "NOT IN" in sql:        # ~isin, as the reference evaluates it: a NULL operand is not in the list
        mask |= df["s"].isna().to_numpy()
    want = df[mask]
    assert sorted(zip(got["x"], _strs(got["s"])), key=repr) == sorted(zip(want["x"], _strs(want["s"])), key=repr)


def test_select_list_comparisons_keep_null():
    df = _frame(4, n=500)
    c = _ctx()
    c.create_table("t", df.assign(s=df["s"].astype("category"), id=np.arange(len(df))))
    got = c.sql("SELECT id, s <> 'absent' AS ne_absent, s LIKE '%' AS any_, s = 'absent' AS eq_absent, "
                "s = 'banana' AS eq_banana FROM t").compute()
    assert len(got) == len(df)
    want = dict(enumerate(_strs(df["s"])))
    for x, a, b, e, f in zip(got["id"], got["ne_absent"], got["any_"], got["eq_absent"], got["eq_banana"]):
        s = want[x]
        if s is None:
            assert all(pd.isna(v) for v in (a, b, e, f)), (x, a, b, e, f)
        else:
            assert (bool(a), bool(b), bool(e), bool(f)) == (True, True, False, s == "banana"), (x, s)


def test_group_by_min_max_count_distinct_and_distinct():
    df = _frame(2, n=5000)
    c = _ctx()
    c.create_table("t", df.assign(s=df["s"].astype("category"), k=df["x"] % 3), npartitions=2)
    got = c.sql("SELECT s, SUM(v) AS sv, COUNT(*) AS n FROM t GROUP BY s").compute()
    g = {k: (a, b) for k, a, b in zip(_strs(got["s"]), got["sv"], got["n"])}
    w = {}
    for k, v in zip(_strs(df["s"]), df["v"]):
        a, b = w.get(k, (0.0, 0))
        w[k] = (a + v, b + 1)
    assert g.keys() == w.keys()
    for k in w:
        assert g[k][1] == w[k][1] and abs(g[k][0] - w[k][0]) < 1e-9 * max(1, abs(w[k][0]))
    agg = c.sql("SELECT MIN(s) AS lo, MAX(s) AS hi, COUNT(s) AS n, COUNT(DISTINCT s) AS d FROM t").compute()
    nn = [s for s in _strs(df["s"]) if s is not None]
    assert _strs(agg["lo"]) == [min(nn)] and _strs(agg["hi"]) == [max(nn)]
    assert agg["n"].tolist() == [len(nn)] and agg["d"].tolist() == [len(set(nn))]
    per = c.sql("SELECT k, MIN(s) AS lo, MAX(s) AS hi FROM t GROUP BY k").compute()
    for k, lo, hi in zip(per["k"], _strs(per["lo"]), _strs(per["hi"])):
        vals = [s for s, x in zip(_strs(df["s"]), df["x"]) if s is not None and x % 3 == k]
        assert (lo, hi) == (min(vals), max(vals))
    dist = c.sql("SELECT DISTINCT s FROM t").compute()
    assert sorted(_strs(dist["s"]), key=repr) == sorted(set(_strs(df["s"])), key=repr)


@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("nulls_first", [True, False])
def test_order_by_with_nulls_limit_offset(asc, nulls_first):
    df = _frame(3, n=400)
    c = _ctx()
    c.create_table("t", df.assign(s=df["s"].astype("category")))
    order = f"{'ASC' if asc else 'DESC'} NULLS {'FIRST' if nulls_first else 'LAST'}"
    got = c.sql(f"SELECT s FROM t ORDER BY s {order} LIMIT 50 OFFSET 7").compute()
    nn = sorted((s for s in _strs(df["s"]) if s is not None), reverse=not asc)
    nulls = [None] * int(df["s"].isna().sum())
    full = nulls + nn if nulls_first else nn + nulls
    assert _strs(got["s"]) == full[7:57]


def _join_frames():
    rng = np.random.default_rng(9)
    left_words = WORDS[:14] + ["only-left"]
    right_words = WORDS[5:] + ["only-right", "zz"]
    ls = np.array(left_words, dtype=object)[rng.integers(0, len(left_words), 800)]
    rs = np.array(right_words, dtype=object)[rng.integers(0, len(right_words), 60)]
    ls[rng.random(800) < 0.05] = None
    rs[rng.random(60) < 0.1] = None
    return (pd.DataFrame({"ls": ls, "lx": np.arange(800)}), pd.DataFrame({"rs": rs, "rx": np.arange(60)}))


@pytest.mark.parametrize("how", ["INNER", "LEFT", "RIGHT", "FULL"])
def test_joins_on_keys_of_two_dictionaries(how):
    l, r = _join_frames()
    c = _ctx()
    c.create_table("l", l.assign(ls=l["ls"].astype("category")))
    c.create_table("r", r.assign(rs=r["rs"].astype("category")))
    got = c.sql(f"SELECT l.lx, l.ls, r.rx, r.rs FROM l {how} JOIN r ON l.ls = r.rs").compute()
    lrows = list(zip(l["lx"], _strs(l["ls"])))
    rrows = list(zip(r["rx"], _strs(r["rs"])))
    want = [(a, s, b, t) for a, s in lrows for b, t in rrows if s is not None and s == t]   # NULL keys never match
    if how in ("LEFT", "FULL"):
        want += [(a, s, None, None) for a, s in lrows if s is None or all(s != t for _, t in rrows)]
    if how in ("RIGHT", "FULL"):
        want += [(None, None, b, t) for b, t in rrows if t is None or all(s != t for _, s in lrows)]
    norm = lambda v: None if (v is None or (isinstance(v, float) and v != v)) else int(v) if isinstance(v, float) else v  # noqa: E731
    g = sorted(repr((norm(a), b, norm(cc), d)) for a, b, cc, d in
               zip(got["lx"].astype(object), _strs(got["ls"]), got["rx"].astype(object), _strs(got["rs"])))
    assert g == sorted(repr((a if a is None else int(a), s, b if b is None else int(b), t)) for a, s, b, t in want)
    # both key columns decode through their own dictionaries
    both = got.dropna(subset=["ls", "rs"])
    assert all(a == b for a, b in zip(_strs(both["ls"]), _strs(both["rs"])))


def test_semi_anti_and_multi_key_joins():
    l, r = _join_frames()
    c = _ctx()
    c.create_table("l", l.assign(ls=l["ls"].astype("category"), m=l["lx"] % 2))
    c.create_table("r", r.assign(rs=r["rs"].astype("category"), m=r["rx"] % 2))
    rset = set(s for s in _strs(r["rs"]) if s is not None)
    semi = c.sql("SELECT l.lx FROM l LEFT SEMI JOIN r ON l.ls = r.rs").compute()
    assert sorted(semi["lx"]) == sorted(x for x, s in zip(l["lx"], _strs(l["ls"])) if s in rset)
    anti = c.sql("SELECT l.lx FROM l LEFT ANTI JOIN r ON l.ls = r.rs").compute()
    assert sorted(anti["lx"]) == sorted(x for x, s in zip(l["lx"], _strs(l["ls"])) if s not in rset)
    mk = c.sql("SELECT l.lx, r.rx FROM l JOIN r ON l.ls = r.rs AND l.m = r.m").compute()
    want = [(x, y) for x, s, m in zip(l["lx"], _strs(l["ls"]), l["lx"] % 2)
            for y, t, n in zip(r["rx"], _strs(r["rs"]), r["rx"] % 2)
            if s is not None and s == t and m == n]
    assert sorted(zip(mk["lx"], mk["rx"])) == sorted(want)


def test_cross_dictionary_comparison_after_a_join():
    l, r = _join_frames()
    c = _ctx()
    c.create_table("l", l.assign(ls=l["ls"].astype("category"), k=l["lx"] % 7))
    c.create_table("r", r.assign(rs=r["rs"].astype("category"), k=r["rx"] % 7))
    for op, fn in [("<", lambda a, b: a < b), ("=", lambda a, b: a == b), (">=", lambda a, b: a >= b)]:
        got = c.sql(f"SELECT l.lx, r.rx FROM l JOIN r ON l.k = r.k WHERE l.ls {op} r.rs").compute()
        want = [(x, y) for x, s, k in zip(l["lx"], _strs(l["ls"]), l["lx"] % 7)
                for y, t, kk in zip(r["rx"], _strs(r["rs"]), r["rx"] % 7)
                if k == kk and s is not None and t is not None and fn(s, t)]
        assert sorted(zip(got["lx"], got["rx"])) == sorted(want), op


# ---- round trips ---------------------------------------------------------------------------
def test_round_trips_of_every_input(tmp_path):
    vals = ["b", None, "a", "", "ö", "b", "😀", None]
    c = _ctx()
    cat = pd.Series(vals, dtype="category")
    chunked = pa.chunked_array([pa.array(vals[:3]).dictionary_encode(), pa.array(vals[3:]).dictionary_encode()])
    pq.write_table(pa.table({"s": pa.array(vals).dictionary_encode()}), str(tmp_path / "d.parquet"))
    pq.write_table(pa.table({"s": vals}), str(tmp_path / "p.parquet"))
    pd.DataFrame({"s": vals}).to_csv(str(tmp_path / "c.csv"), index=False)
    c.create_table("pandas", pd.DataFrame({"s": cat}))
    c.create_table("persisted", pd.DataFrame({"s": cat}), persist=True)
    c.create_table("arrow", pa.table({"s": chunked}))
    c.create_table("pq_eager", str(tmp_path / "d.parquet"), persist=True)
    c.create_table("pq_lazy", str(tmp_path / "d.parquet"))
    c.create_table("pq_plain", str(tmp_path / "p.parquet"), dictionary=["s"])
    c.create_table("csv", str(tmp_path / "c.csv"), dictionary=["s"])
    c.sql("CREATE TABLE ctas AS SELECT s FROM pandas")
    for name in ("pandas", "persisted", "arrow", "pq_eager", "pq_lazy", "pq_plain", "csv", "ctas"):
        got = c.sql(f"SELECT s FROM {name}").compute()
        assert isinstance(got["s"].dtype, pd.CategoricalDtype), name
        # CSV writes NULL as an empty cell, which reads back as the empty string
        want = ["" if (name == "csv" and v is None) else v for v in vals]
        assert _strs(got["s"]) == want, name
        assert c.sql(f"SELECT COUNT(*) AS n FROM {name} WHERE s = 'b'").compute()["n"].tolist() == [2], name


def test_lazy_parquet_prunes_row_groups_by_string_statistics(tmp_path):
    from dask_sql_b200 import executor
    words = sorted("w%05d" % i for i in range(4000))
    path = str(tmp_path / "sorted.parquet")
    pq.write_table(pa.table({"s": pa.array(words).dictionary_encode(), "x": np.arange(4000)}), path,
                   row_group_size=500)
    c = _ctx()
    c.create_table("t", path)
    before = executor.stats.get("rowgroups_skipped", 0)
    got = c.sql("SELECT x FROM t WHERE s >= 'w03000' AND s LIKE 'w03%'").compute()
    assert sorted(got["x"]) == list(range(3000, 4000))
    assert executor.stats.get("rowgroups_skipped", 0) - before > 0
    got = c.sql("SELECT x FROM t WHERE s = 'w00042'").compute()
    assert got["x"].tolist() == [42]


# ---- fusion ------------------------------------------------------------------------------------
def _q3(seed=0, nd=4000, nf=200_000):
    rng = np.random.default_rng(seed)
    segs = np.array(["AUTOMOBILE", "BUILDING", "FURNITURE", "HOUSEHOLD", "MACHINERY"], dtype=object)
    seg_i = rng.integers(0, 5, nd)
    grp_i = rng.integers(0, 60, nd)
    grp_words = np.array(["g%02d-%s" % (i, "x" * (i % 5)) for i in range(60)], dtype=object)
    dim = pd.DataFrame({"pk": rng.permutation(nd), "seg_i": seg_i, "grp_i": grp_i,
                        "segment": pd.Series(segs[seg_i]).astype("category"),
                        "grp": pd.Series(grp_words[grp_i]).astype("category")})
    fact = pd.DataFrame({"fk": rng.integers(0, nd, nf), "x": rng.integers(-100, 100, nf), "val": rng.random(nf)})
    return dim, fact


def test_q3_with_string_predicate_and_group_key_runs_the_fused_star(monkeypatch):
    from dask_sql_b200 import _lib, executor
    dim, fact = _q3()
    c = _ctx()
    c.create_table("fact", fact, npartitions=4)
    c.create_table("dim", dim)
    programs = []
    real = _lib.expr_eval

    def spy(prog_ref, *rest):
        prog = prog_ref._obj
        programs.append(tuple((prog.code[i].op, prog.code[i].a, prog.code[i].imm_i) for i in range(prog.n)))
        return real(prog_ref, *rest)

    monkeypatch.setattr(_lib, "expr_eval", spy)

    def run(q):
        programs.clear()
        before = executor.stats["star_fused"]
        out = c.sql(q).compute()
        assert executor.stats["star_fused"] > before, q
        return out, list(programs)

    base = "SELECT d.{g} AS g, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fk = d.pk WHERE f.x > 0 AND {w} GROUP BY d.{g}"
    want, p_int = run(base.format(g="grp_i", w="d.seg_i = 1"))
    want = dict(zip(["g%02d-%s" % (i, "x" * (i % 5)) for i in want["g"]], want["rev"]))
    for w in ["d.segment = 'BUILDING'", "d.segment LIKE 'BUI%'"]:
        got, p_str = run(base.format(g="grp", w=w))
        # no interpreter pass beyond those of the integer twin, and none holds a string predicate
        assert len(p_str) <= len(p_int) and all(p in p_int for p in p_str), (w, p_str, p_int)
        assert not any(op == _lib.OP_MAP for prog in p_str for op, _, _ in prog)
        assert isinstance(got["g"].dtype, pd.CategoricalDtype)
        g = dict(zip(_strs(got["g"]), got["rev"]))
        assert g.keys() == want.keys()
        np.testing.assert_allclose([g[k] for k in sorted(g)], [want[k] for k in sorted(want)], rtol=1e-12)
    # a general LIKE evaluates its per-entry table once per dimension pass and still fuses
    got, progs = run(base.format(g="grp", w="d.segment LIKE '%ILD%'"))
    g = dict(zip(_strs(got["g"]), got["rev"]))
    assert g.keys() == want.keys()
    np.testing.assert_allclose([g[k] for k in sorted(g)], [want[k] for k in sorted(want)], rtol=1e-12)
    assert any(op == _lib.OP_MAP for prog in progs for op, _, _ in prog)


def test_q3_joined_on_string_keys_takes_the_general_join():
    dim, fact = _q3(1, nd=500, nf=20_000)
    dim = dim.assign(pks=pd.Series(["k%04d" % i for i in dim["pk"]]).astype("category"))
    fact = fact.assign(fks=pd.Series(["k%04d" % i for i in fact["fk"]]).astype("category"))
    c = _ctx()
    c.create_table("fact", fact)
    c.create_table("dim", dim)
    got = c.sql("SELECT d.grp AS g, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fks = d.pks "
                "WHERE d.segment = 'BUILDING' GROUP BY d.grp").compute()
    m = fact.merge(dim, left_on="fk", right_on="pk")
    want = m[m["segment"] == "BUILDING"].groupby("grp", observed=True)["val"].sum()
    g = dict(zip(_strs(got["g"]), got["rev"]))
    assert sorted(g) == sorted(want.index)
    np.testing.assert_allclose([g[k] for k in sorted(g)], [want[k] for k in sorted(g)], rtol=1e-12)


def test_results_are_categories_with_the_column_dictionary():
    c = _ctx()
    c.create_table("t", pd.DataFrame({"s": pd.Series(["b", "a", None, "b"], dtype="category")}))
    got = c.sql("SELECT s FROM t WHERE s <> 'zz'").compute()
    assert list(got["s"].cat.categories) == ["a", "b"]
    assert _strs(got["s"]) == ["b", "a", "b"]
    assert re.match("category", str(c.sql("SELECT s FROM t").dtypes["s"]))
