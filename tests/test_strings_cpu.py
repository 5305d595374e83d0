"""VARCHAR columns on the host: dictionary build from every accepted input, literal -> code-term rules,
LIKE shapes, parser cases and the plan-time refusals.  No GPU needed."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from dask_sql_b200 import Context
from dask_sql_b200 import _lib as L
from dask_sql_b200 import expr as E
from dask_sql_b200 import strings as S
from dask_sql_b200.expr import ColRef
from dask_sql_b200.planner.sqlparse import parse_sql
from dask_sql_b200.table import DeviceTable, _host_column, arrow_columns, ParquetTable
from tests import strings_ref as R

WORDS = ["pear", "apple", "", "Zebra", "öl", "apple", None, "😀", "app", "ápple"]


def _col(values):
    codes, null, lg = S.encode_arrow(pa.array(values, type=pa.string()))
    return codes, null, lg


def _decode(codes, null, lg):
    d = lg.dictionary.to_list()
    return [None if (null is not None and null[i]) else d[c] for i, c in enumerate(codes)]


# ---- dictionary build -------------------------------------------------------------------------
def test_dictionary_is_sorted_unique_and_round_trips():
    codes, null, lg = _col(WORDS)
    assert lg == "category" and S.is_varchar(lg)
    assert lg.dictionary.to_list() == R.dictionary(WORDS)
    assert _decode(codes, null, lg) == WORDS
    assert codes.dtype == np.int64


def test_every_input_type_builds_the_same_dictionary():
    ref = R.dictionary(WORDS)
    cat = pd.Series(WORDS, dtype="category")
    arrow_dict = pa.array(WORDS).dictionary_encode()
    chunked = pa.chunked_array([pa.array(WORDS[:4]).dictionary_encode(), pa.array(WORDS[4:]).dictionary_encode()])
    assert chunked.chunk(0).dictionary != chunked.chunk(1).dictionary
    outs = [S.encode_pandas(cat), S.encode_arrow(arrow_dict), S.encode_arrow(chunked),
            S.encode_arrow(pa.array(WORDS, type=pa.large_string()))]
    for codes, null, lg in outs:
        assert lg.dictionary.to_list() == ref
        assert _decode(codes, null, lg) == WORDS
    # equal dictionaries are recognised as one
    assert len({id(lg.dictionary) for _, _, lg in outs}) == 1


def test_arrow_dictionary_edge_cases():
    # duplicate entries, a NULL entry, an unused entry
    words = pa.array(["b", "a", "b", None, "unused"])
    idx = pa.array([0, 1, 2, 3, None, 2], type=pa.int8())
    codes, null, lg = S.encode_arrow(pa.DictionaryArray.from_arrays(idx, words))
    assert lg.dictionary.to_list() == ["a", "b"]
    assert _decode(codes, null, lg) == ["b", "a", "b", None, None, "b"]


def test_ordered_categorical_with_unused_and_non_lexical_order():
    s = pd.Series(pd.Categorical(["m", "z", None, "a"], categories=["z", "m", "a", "q"], ordered=True))
    codes, null, lg = S.encode_pandas(s)
    assert lg.dictionary.to_list() == ["a", "m", "z"]
    assert _decode(codes, null, lg) == ["m", "z", None, "a"]


def test_empty_and_all_null_columns():
    codes, null, lg = _col([])
    assert len(lg.dictionary) == 0 and len(codes) == 0
    codes, null, lg = _col([None, None])
    assert len(lg.dictionary) == 0 and null.tolist() == [True, True]
    codes, null, lg = S.encode_pandas(pd.Series(pd.Categorical([None, None], categories=["x"])))
    assert len(lg.dictionary) == 0 and null.all()


def test_non_string_categories_raise():
    with pytest.raises(NotImplementedError):
        S.encode_pandas(pd.Series([1, 2, 1], dtype="category"))
    with pytest.raises(NotImplementedError):
        arrow_columns(pa.table({"d": pa.array([1, 2, 1]).dictionary_encode()}))


def test_plain_strings_still_raise_and_point_to_the_opt_in():
    with pytest.raises(NotImplementedError, match="category"):
        _host_column(pd.Series(["a", "b"]), pin=False)
    with pytest.raises(NotImplementedError, match="dictionary="):
        arrow_columns(pa.table({"s": ["a", "b"]}))
    got = arrow_columns(pa.table({"s": ["b", "a", None]}), dictionary=["s"])["s"]
    assert got.logical.dictionary.to_list() == ["a", "b"] and got.values.tolist()[:2] == [1, 0]


def test_partitions_share_one_dictionary():
    s = pd.Series(["x%03d" % (i % 97) for i in range(1000)], dtype="category")
    t = DeviceTable.from_columns({"s": s}, npartitions=4, persist=False)
    assert t.npartitions == 4
    assert len({id(p["s"].logical.dictionary) for p in t.partitions}) == 1
    assert t.schema()[0][2] == "category"


@pytest.mark.parametrize("dist", ["sharded", "root"])
def test_sharded_and_root_tables_refuse_varchar(dist):
    with pytest.raises(NotImplementedError, match="replicated"):
        DeviceTable.from_columns({"s": pd.Series(["a", "b"], dtype="category")}, persist=False, distribution=dist)
    DeviceTable.from_columns({"s": pd.Series(["a", "b"], dtype="category")}, persist=False, distribution="replicated")


def test_lazy_parquet_fixes_one_dictionary_and_code_statistics(tmp_path):
    path = str(tmp_path / "s.parquet")
    vals = sorted("k%04d" % i for i in range(400))
    pq.write_table(pa.table({"s": pa.array(vals).dictionary_encode(), "x": np.arange(400)}), path, row_group_size=100)
    t = ParquetTable(path)
    lg = t.schema()[0][2]
    assert S.is_varchar(lg) and lg.dictionary.to_list() == vals
    cols = [t._column(g, "s") for g in range(4)]
    assert all(c.logical is lg for c in cols)
    assert [int(c.data[0]) for c in cols] == [0, 100, 200, 300]
    assert [(g["cols"]["s"]["min"], g["cols"]["s"]["max"]) for g in t._groups] == \
        [(0, 99), (100, 199), (200, 299), (300, 399)]
    e = S.compare_literal("ge", ColRef("s", L.I64, lg), "k0250")
    assert t.surviving_groups([E.as_term(e)]) == [2, 3]
    with pytest.raises(NotImplementedError):
        ParquetTable(path, distribution="sharded")
    plain = str(tmp_path / "p.parquet")
    pq.write_table(pa.table({"s": ["b", "a"]}), plain)
    with pytest.raises(NotImplementedError):
        ParquetTable(plain).schema()
    assert S.is_varchar(ParquetTable(plain, dictionary=["s"]).schema()[0][2])


def test_sql_type_is_varchar():
    from dask_sql_b200.mappings import python_to_sql_type
    assert python_to_sql_type(pd.CategoricalDtype(["a"])).name == "VARCHAR"
    assert python_to_sql_type("category").name == "VARCHAR"


# ---- literal -> term rules --------------------------------------------------------------------
D_WORDS = ["", "b", "bb", "c", "ö", "😀"]


def _s():
    codes, null, lg = _col(D_WORDS)
    assert lg.dictionary.to_list() == D_WORDS
    return ColRef("s", L.I64, lg)


def _eval_codes(e, codes):
    """evaluate a term expression on the host over codes (the kernels' int64 semantics)"""
    if isinstance(e, E.Call):
        if e.op == "and":
            return _eval_codes(e.args[0], codes) & _eval_codes(e.args[1], codes)
        if e.op == "not":
            return ~_eval_codes(e.args[0], codes)
        if e.op == "isnull":
            return np.zeros(len(codes), bool)
        v = e.args[1].value
        return {"eq": codes == v, "ne": codes != v, "lt": codes < v, "le": codes <= v, "gt": codes > v,
                "ge": codes >= v}[e.op]
    raise AssertionError(e)


LITERALS = ["", "a", "b", "ba", "bb", "bbb", "c", "d", "ö", "öa", "😀", "😀😀", "\x00", "zzz"]


@pytest.mark.parametrize("op", ["eq", "ne", "lt", "le", "gt", "ge"])
def test_comparison_terms_are_exact_for_present_and_absent_literals(op):
    s = _s()
    codes = np.arange(len(D_WORDS))
    pyop = {"eq": "__eq__", "ne": "__ne__", "lt": "__lt__", "le": "__le__", "gt": "__gt__", "ge": "__ge__"}[op]
    for lit in LITERALS:
        e = E.binop(op, s, lit)
        exp = np.array([getattr(w, pyop)(lit) for w in D_WORDS])
        np.testing.assert_array_equal(_eval_codes(e, codes), exp, err_msg=f"{op} {lit!r}")
        for c in E.conjuncts(e):
            if not (isinstance(c, E.Call) and c.op == "not"):
                assert E.as_term(c) is not None, f"{op} {lit!r} is not a scan term"
        # the literal on the left flips the operator
        flip = {"lt": "gt", "le": "ge", "gt": "lt", "ge": "le"}.get(op, op)
        np.testing.assert_array_equal(_eval_codes(E.binop(flip, lit, s), codes), exp)


def test_absent_literal_rules():
    s = _s()
    e = E.binop("eq", s, "zz")
    assert E.as_term(e) == ("s", L.EQ, -1)                     # no code: no row passes
    assert E.as_term(E.binop("ne", s, "zz")) == ("s", L.GE, 0)   # every code; NULL stays NULL
    assert E.as_term(E.binop("lt", s, "\x00")) == ("s", L.LT, 1)   # after '' and before 'b'
    assert E.as_term(E.binop("gt", s, "😀😀")) == ("s", L.GE, 6)   # after the last entry


PATTERNS = ["b%", "b", "bb%", "%", "%%", "", "b%%", "ö%", "😀%", "x%", "b\\%", "b\\%%", "b\\_%", "\\%", "c_",
            "%b", "_", "b_%", "B%"]


@pytest.mark.parametrize("pattern", PATTERNS)
def test_like_shapes_and_ranges(pattern):
    s = _s()
    e = S.like(s, pattern)
    exp = np.array([R.like(w, pattern) for w in D_WORDS])
    kind, _ = S.like_shape(pattern, "\\")
    if kind == "general":
        assert isinstance(e, E.Call) and e.op == "map" and isinstance(e.param, S.LikeTable)
        return
    got = _eval_codes(e, np.arange(len(D_WORDS)))
    np.testing.assert_array_equal(got, exp)
    assert all(E.as_term(c) is not None for c in E.conjuncts(e)) and len(E.conjuncts(e)) <= 2


def test_like_prefix_with_multibyte_last_character():
    codes, null, lg = _col(["é", "éa", "éz", "ê", "e", "f", "é😀"])
    s = ColRef("s", L.I64, lg)
    e = S.like(s, "é%")
    got = _eval_codes(e, np.arange(len(lg.dictionary)))
    np.testing.assert_array_equal(got, [R.like(w, "é%") for w in lg.dictionary.to_list()])
    assert S.successor("é".encode()) == b"\xc3\xaa"


@pytest.mark.parametrize("build", [lambda s: E.binop("ne", s, "absent"), lambda s: S.like(s, "%"),
                                   lambda s: S.like(s, "%%")])
def test_always_true_rewrites_keep_null_rows_null(build):
    """`s <> 'absent'` and `s LIKE '%'` are one GE 0 term: true for every code and NULL for a NULL row, so
    NOT of them (and a SELECT list) keeps NULL NULL instead of turning into IS NULL"""
    e = build(_s())
    assert E.as_term(e) == ("s", L.GE, 0)
    neg = E.unop("not", e)
    assert E.as_term(neg) is None and neg.op == "not" and neg.args[0] is e


def test_like_host_fold_matches_reference():
    for w in ["xr%", "XR%", "x%", "X%a", "xRa", "r", "R"]:         # a letter escape is recognised as written
        for p in ["xR%", "xr%", "Xr%", "r%", "R%", "rr"]:
            for ilike in (False, True):
                assert S.like_host(w, p, "r", ilike) == R.like(w, p, "r", ilike), (w, p, ilike)
    assert R.like("x%", "xr%", "r", True) and not R.like("xyz", "xr%", "r", True)
    assert R.like("XrZ", "xR%", "r", True)
    for w in ["abc", "ABC", "a\nc", "Ä", "ä", "", "%_%", "a_c"]:
        for p in ["a%", "A_C", "%\\%%", "a_c", "ä", "_", "%", ""]:
            for ilike in (False, True):
                assert S.like_host(w, p, "\\", ilike) == R.like(w, p, "\\", ilike), (w, p, ilike)


def test_different_dictionaries_compare_through_the_order_table():
    _, _, la = _col(["a", "c", "e"])
    _, _, lb = _col(["b", "c", "f"])
    a, b = ColRef("a", L.I64, la), ColRef("b", L.I64, lb)
    e = E.binop("lt", a, b)
    assert e.args[0].op == "mul" and e.args[1].op == "map" and isinstance(e.args[1].param, S.OrderTable)
    _, _, la2 = _col(["e", "c", "a"])
    same = E.binop("eq", a, ColRef("a2", L.I64, la2))
    assert [x.op if isinstance(x, E.Call) else type(x).__name__ for x in same.args] == ["ColRef", "ColRef"]
    ka, kb = S.join_keys(a, b, translate_a=True)
    assert ka.op == "map" and isinstance(ka.param, S.MatchTable) and kb is b


def test_map_program_reads_tables_after_the_columns():
    _, _, lg = _col(["a", "b"])
    s = ColRef("s", L.I64, lg)
    e = E.unop("not", S.like(s, "%a%"))
    tables = E.map_tables(e)
    prog = E.compile_expr(e, ["s"], tables)
    ops = [(prog.code[i].op, prog.code[i].a, prog.code[i].imm_i) for i in range(prog.n)]
    assert ops[:2] == [(L.OP_LOAD, 0, 0), (L.OP_MAP, 1, 2)]
    with pytest.raises(NotImplementedError):
        E.compile_expr(e, ["s"])


# ---- parser and planner -----------------------------------------------------------------------
def test_parser_like_forms():
    w = parse_sql("SELECT a FROM t WHERE s NOT ILIKE 'x%' ESCAPE '!'")["where"]
    assert (w.kind, w.negated, w.ilike, w.escape, w.pattern.value) == ("like", True, True, "!", "x%")
    w = parse_sql("SELECT a FROM t WHERE s LIKE 'x'")["where"]
    assert (w.kind, w.negated, w.ilike, w.escape) == ("like", False, False, None)
    w = parse_sql("SELECT a FROM t WHERE NOT s LIKE 'x' AND b = 1")["where"]
    assert w.l.kind == "not" and w.l.e.kind == "like"


@pytest.mark.parametrize("sql", [
    "SELECT a FROM t WHERE s SIMILAR TO 'x'",
    "SELECT a FROM t WHERE s NOT SIMILAR TO 'x'",
    "SELECT s || 'x' FROM t",
    "SELECT UPPER(s) FROM t", "SELECT LOWER(s) FROM t", "SELECT CONCAT(s, s) FROM t",
    "SELECT SUBSTRING(s FROM 1 FOR 2) FROM t", "SELECT TRIM(s) FROM t", "SELECT POSITION('a' IN s) FROM t",
    "SELECT CHAR_LENGTH(s) FROM t", "SELECT REPLACE(s, 'a', 'b') FROM t",
])
def test_out_of_scope_string_syntax_raises(sql):
    with pytest.raises(NotImplementedError):
        parse_sql(sql)


def _ctx():
    c = Context()
    c.create_table("t", pd.DataFrame({"s": pd.Series(["b", "a", None], dtype="category"), "x": [1, 2, 3]}))
    return c


@pytest.mark.filterwarnings("ignore:The optimizer failed")
@pytest.mark.parametrize("sql", [
    "SELECT SUM(s) FROM t", "SELECT AVG(s) FROM t", "SELECT VAR_POP(s) FROM t",
    "SELECT CAST(s AS VARCHAR) FROM t", "SELECT CAST(x AS VARCHAR) FROM t", "SELECT CAST(s AS BIGINT) FROM t",
    "SELECT CASE WHEN x > 1 THEN s ELSE 'z' END FROM t",
    "SELECT 'lit' AS l FROM t", "SELECT s + 1 FROM t",
])
def test_plan_time_refusals(sql):
    with pytest.raises(NotImplementedError):
        _ctx().sql(sql)


def test_string_value_from_two_sources_and_like_on_numbers_raise():
    from dask_sql_b200.utils import ParsingException
    s = _s()
    with pytest.raises(NotImplementedError):
        E.fillna(s, "z")
    with pytest.raises(NotImplementedError):
        E.case(E.Lit(True), s, s)
    with pytest.raises(ParsingException):
        _ctx().sql("SELECT x FROM t WHERE x LIKE 'a%'")


def test_catalog_reports_varchar_and_plain_strings_still_raise():
    c = _ctx()
    assert dict(c._catalog(None, "t")[1])["s"] == "VARCHAR"
    with pytest.raises(NotImplementedError):
        c.create_table("u", pd.DataFrame({"s": ["x", "y"]}))
    c.create_table("u", pd.DataFrame({"s": ["x", "y"]}), dictionary=["s"])
    assert dict(c._catalog(None, "u")[1])["s"] == "VARCHAR"
    with pytest.raises(NotImplementedError):
        c.create_table("v", pd.DataFrame({"s": pd.Series(["x"], dtype="category")}), distribution="sharded")


def test_encode_into_remaps_a_chunk_through_its_own_distinct_values():
    _, _, lg = _col(WORDS)
    for chunk in [pa.array(["öl", None, "apple", "😀", "apple"]),
                  pa.array(["öl", None, "apple", "😀", "apple"]).dictionary_encode(),
                  pa.chunked_array([pa.array(["öl", None]).dictionary_encode(),
                                    pa.array(["apple", "😀", "apple"]).dictionary_encode()]),
                  pa.array([], type=pa.string()), pa.array([None, None], type=pa.string())]:
        codes, null, out = S.encode_into(chunk, lg)
        assert out is lg
        vals = chunk.to_pylist()
        assert _decode(codes, null, lg) == vals
