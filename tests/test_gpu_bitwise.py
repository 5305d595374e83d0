"""The AND / OR / XOR accumulators of every aggregation kernel word for word against tests/groupagg_bits_ref.py,
through the C-ABI with the helpers of tests/test_gpu_groupagg.py: b2_groupby_dense with its grouped (table on
and off) and heavy-hitter paths (hot lists: b2_hot_slots', all -1, hostile), b2_groupby_dense_ordered after a
range partition, b2_groupby_hash1 (with overflow and rerun), b2_groupby_hashk, b2_star_agg over its three
lookup kinds, the generic b2_join_agg kernel and b2_scan_agg; plus b2_bitwise_combine and the argument checks.
Inputs hold INT64_MIN, -1, 0 and INT64_MAX, U8 (0/1) values, NULL masks, and 1 to 3 partitions per state."""
import ctypes as C

import numpy as np
import pytest

from tests import groupagg_bits_ref as B
from tests import groupagg_ref as G
from tests import rowwise_ref as R
from tests.test_gpu_groupagg import (
    KEY, KMIN, PRED, State, _aggs, _concat_inputs, _dtypes, _eq, _full, _np, _t, check_dense_family, check_out_slots,
    dense_expected, dense_part, dim_part, fact_part, hash_part, hashk_part, run_star_agg, scan_of, _dim_selection,
    _grp_slot, DIM_PRED, GRP_MIN, NGRP, build_side, probe_part, run_join_agg, join_agg_expected, check_global, BUILD,
    run_dense_kernel)
from tests.test_gpu_rowwise import _dev, _L, _ptr, _stream

pytestmark = pytest.mark.gpu

MIN, MAX = R.INT64_MIN, R.INT64_MAX
AND, OR, XOR, COUNT, SUM = B.AGG_AND, B.AGG_OR, B.AGG_XOR, G.AGG_COUNT, G.AGG_SUM
BIT_POOL = np.array([MIN, -1, 0, MAX, 1, 2, 5, -6, 0x5555555555555555, -0x5555555555555556, 1 << 40, -(1 << 40)],
                    np.int64)
VB, VBN, VU = 7, 8, 9      # appended to the dense columns: edge ints with NULLs, edge ints without, U8 with NULLs


@pytest.fixture(autouse=True)
def bitwise_reference(monkeypatch):
    """the helpers of tests/test_gpu_groupagg.py (State, dense_expected, check_dense_family, ...) read the
    reference through groupagg_ref: let them see the bitwise ops"""
    B.install(monkeypatch)


def with_bits(cols, rng, mostly=None):
    """the dense columns plus VB / VBN / VU.  mostly: a value most rows carry (AND stays informative under skew)"""
    n = cols[0].n
    vb = rng.choice(BIT_POOL, n) if n else np.zeros(0, np.int64)
    vbn = rng.choice(BIT_POOL, n) if n else np.zeros(0, np.int64)
    if mostly is not None and n:
        keep = rng.random(n) < 0.97
        vbn = np.where(keep, mostly, vbn)
    return cols + [R.Column(vb, rng.random(n) < 0.1, R.I64), R.Column(vbn, None, R.I64),
                   R.Column(rng.integers(0, 2, n).astype(np.uint8), rng.random(n) < 0.1, R.U8)]


BIT_SPECS = {
    # every op on both input types with a cnt array each (nullable inputs): too many arrays for the CTA tables
    "all": ([(-1, COUNT), (VB, AND), (VB, OR), (VB, XOR), (VU, AND), (VU, OR), (VU, XOR), (VBN, SUM)], True),
    # three never-NULL bitwise accumulators + rows: all four carried by the heavy-hitter partials
    "hh": ([(VBN, AND), (VBN, OR), (VBN, XOR)], False),
    # NULL-able inputs in the heavy-hitter partials (no cnt arrays): an all-NULL hitter must not touch them
    "hh_null": ([(VB, AND), (VU, OR), (VBN, XOR)], False),
}


@pytest.mark.parametrize("pred", [False, True], ids=["all_rows", "predicate"])
@pytest.mark.parametrize("n", [0, 1, 33, 2049, 8229, 100_003])
def test_bitwise_dense_family(n, pred):
    rng = np.random.default_rng(4000 + n + pred)
    nparts = 1 + n % 3
    parts = [with_bits(dense_part("uniform" if i % 2 == 0 else "zipf", n, rng), rng) for i in range(nparts)]
    terms = PRED if pred else []
    for spec in BIT_SPECS.values():
        ordered = all(parts[0][c].null is None and parts[0][c].dtype != R.U8 for c, _ in spec[0] if c >= 0)
        check_dense_family(parts, terms, KMIN, 502, spec, f"bits n={n} x{nparts} {spec[0][:2]}", ordered=ordered)


@pytest.mark.parametrize("spec", list(BIT_SPECS))
@pytest.mark.parametrize("shape", ["one", "two", "hitters33", "many_repeats", "zipf"])
def test_bitwise_dense_skew(shape, spec):
    """skewed keys through the grouped reduction (one REDG per match group) and the heavy-hitter partials
    (one bitwise atomic per CTA and hitter); most rows carry -2 so that an AND flushed as an OR shows"""
    rng = np.random.default_rng(50 * len(shape) + len(spec))
    span = 1500 if shape == "many_repeats" else 500
    parts = [with_bits(dense_part(shape, 100_003, rng, span), rng, mostly=-2),
             with_bits(dense_part(shape, 4097, rng, span), rng, mostly=-2)]
    check_dense_family(parts, PRED, KMIN, span + 2, BIT_SPECS[spec], f"{shape} {spec}", ordered=False)


def test_bitwise_dense_u8_keys_and_all_null_groups():
    """U8 keys; a group whose inputs are all NULL keeps -1 / 0 / 0 while its cnt stays 0"""
    rng = np.random.default_rng(17)
    n = 8229
    parts = []
    for _ in range(2):
        cols = with_bits(dense_part("uniform", n, rng), rng)
        cols[KEY] = R.Column(rng.integers(0, 2, n).astype(np.uint8), rng.random(n) < 0.2, R.U8)
        k1 = cols[KEY].values == 1
        cols[VB].null = cols[VB].null | k1
        cols[VU].null = cols[VU].null | k1
        parts.append(cols)
    specs, cnt = BIT_SPECS["all"]
    ex, _ = dense_expected(parts, PRED, KEY, 0, 3, specs)
    assert ex.cnt[1][1] == 0 and ex.acc[1][1] == -1 and ex.acc[2][1] == 0 and ex.rows[1] > 0
    check_dense_family(parts, PRED, 0, 3, (specs, cnt), "u8 keys", ordered=False, hot=False)
    for hl in ([0, 1, 2, 2] + [-1] * 28, [2, 1, 0] * 10 + [1, 1]):
        for name in ("hh", "hh_null"):
            sp = BIT_SPECS[name][0]
            ex, gids = dense_expected(parts, PRED, KEY, 0, 3, sp)
            st = State(sp, _dtypes(parts[0], sp), 3, cnt=False)
            outs = run_dense_kernel("hot", parts, PRED, KEY, 0, 3, sp, st, _t(np.array(hl, np.int32)))
            st.check(ex, True, f"u8 hot {name} {hl[:4]}")
            check_out_slots(outs, gids, "u8 hot")


# ---- hash1 / hashk ----------------------------------------------------------------------------------------
def _bits_cols(cols, rng):
    n = cols[0].n
    return cols + [R.Column(rng.choice(BIT_POOL, n) if n else np.zeros(0, np.int64), rng.random(n) < 0.1, R.I64),
                   R.Column(rng.integers(0, 2, n).astype(np.uint8), rng.random(n) < 0.1, R.U8)]


def _hash_bit_specs(b):
    return [(-1, COUNT), (b, AND), (b, OR), (b, XOR), (b + 1, AND), (b + 1, OR), (b + 1, XOR), (b, COUNT)]


def check_hash1_bits(parts, terms, cap, what):
    import torch
    L = _L()
    specs = _hash_bit_specs(len(parts[0]) - 2)
    st = State(specs, _dtypes(parts[0], specs), cap + 2)
    tk = _full(cap + 2, G.EMPTY_KEY)
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    outs = []
    for cols in parts:
        scan = scan_of(cols, terms)
        buf = _full(cols[0].n, 0x5A5A5A5A, dtype=torch.int32)
        L.groupby_hash1(C.byref(scan), 1, _ptr(tk), cap, _aggs(specs), len(specs), st.with_out_slot(buf), _ptr(flags),
                        _stream())
        outs.append((buf, cols[0].n))
    if _np(flags)[0]:
        return False
    tk = _np(tk)
    ident = []
    for cols in parts:
        ok = R.eval_terms(cols, terms, cols[0].n)
        ident += [x if ok[i] else None for i, x in enumerate(G.hash1_identity(cols[1]))]
    gid, groups = G.codes(ident, np.array([x is not None for x in ident], bool))
    ins = _concat_inputs(parts, specs)
    ex = B.aggregate(ins, [op for _, op in specs], gid, len(groups))
    slot_of = {int(tk[h]): h for h in range(cap) if tk[h] != G.EMPTY_KEY}
    slot_of[G.NULL_GROUP], slot_of[G.EMPTY_GROUP] = cap, cap + 1
    st.check(B.permute(ex, [slot_of[g] for g in groups], cap + 2, inputs=ins, ops=[op for _, op in specs]), True, what)
    got = np.concatenate([_np(b, n).astype(np.int64) for b, n in outs])
    _eq(got, np.array([slot_of[x] if x is not None else -1 for x in ident], np.int64), f"{what}: out_slot")
    return True


@pytest.mark.parametrize("kind", ["i64", "wide"])
@pytest.mark.parametrize("n", [1, 33, 8229, 100_003])
def test_bitwise_hash1(n, kind):
    rng = np.random.default_rng(5000 + n + len(kind))
    parts = [_bits_cols(hash_part(kind, n, rng), rng) for _ in range(1 + n % 3)]
    if kind == "wide" and n >= 2049:
        assert not check_hash1_bits(parts, PRED, 8, "cap=8"), "an overfull table must set d_flags[0]"
    cap = 1 << max(4, int(np.ceil(np.log2(max(1, 2 * n * len(parts))))))
    assert check_hash1_bits(parts, PRED, cap, f"{kind} n={n}")
    assert check_hash1_bits(parts, [], cap, f"{kind} n={n} no predicate")


@pytest.mark.parametrize("kinds", [("i64",), ("u8", "f64"), ("i64", "f64", "u8")], ids="-".join)
@pytest.mark.parametrize("n", [33, 100_003])
def test_bitwise_hashk(n, kinds):
    import torch
    L = _L()
    rng = np.random.default_rng(6000 + n + len(kinds))
    nk = len(kinds)
    parts = [_bits_cols(hashk_part(kinds, n, rng), rng) for _ in range(1 + n % 3)]
    specs = _hash_bit_specs(len(parts[0]) - 2)
    cap = 4096
    st = State(specs, _dtypes(parts[0], specs), cap)
    tk, tn = _full(nk * cap, 0x5A5A), torch.full((cap,), 0x5A, dtype=torch.uint8, device=_dev())
    ts, flags = torch.zeros(cap, dtype=torch.int32, device=_dev()), torch.zeros(4, dtype=torch.int32, device=_dev())
    kc = (C.c_int32 * nk)(*range(1, 1 + nk))
    for cols in parts:
        scan = scan_of(cols, PRED)
        L.groupby_hashk(C.byref(scan), kc, nk, _ptr(tk), _ptr(tn), _ptr(ts), cap, _aggs(specs), len(specs),
                        st.with_out_slot(None), _ptr(flags), _stream())
    assert not _np(flags)[0]
    ident = []
    for cols in parts:
        ok = R.eval_terms(cols, PRED, cols[0].n)
        ident += [x if ok[i] else None for i, x in enumerate(G.hashk_identity(cols[1:1 + nk]))]
    gid, groups = G.codes(ident, np.array([x is not None for x in ident], bool))
    ins = _concat_inputs(parts, specs)
    ex = B.aggregate(ins, [op for _, op in specs], gid, len(groups))
    tkh, tnh, tsh = _np(tk).reshape(nk, cap), _np(tn), _np(ts)
    slot_of = {tuple(int(tkh[k, h]) for k in range(nk)) + (int(tnh[h]),): int(h) for h in np.flatnonzero(tsh == 2)}
    assert set(slot_of) == set(groups)
    st.check(B.permute(ex, [slot_of[g] for g in groups], cap, inputs=ins, ops=[op for _, op in specs]), True,
             f"hashk {kinds} n={n}")


# ---- star ------------------------------------------------------------------------------------------------
STAR_BIT_SPECS = [(-1, COUNT), (6, AND), (6, OR), (6, XOR), (7, AND), (7, XOR), (6, COUNT), (2, SUM)]


def _star_lookups(rng):
    """the three lookup kinds over the same dim: ranked bitmap, int32 per key, hash; -> [(name, lk, map, keep)]"""
    import torch
    L = _L()
    pk_min, nd = 1000, 3000
    dims = [dim_part(nd, rng, pk_min), dim_part(nd, rng, pk_min + 2 * nd)]
    rng_ = 4 * nd
    out = []
    # bitmap from the unfiltered partitions
    dirw = torch.zeros((rng_ + 31) // 32, dtype=torch.int64, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    slots = _full(rng_, 0x5A5A5A5A, dtype=torch.int32)
    scans = [scan_of(cols, DIM_PRED) for cols in dims]
    for s in scans:
        L.star_build_mark(C.byref(s), 1, pk_min, rng_, _ptr(dirw), _ptr(flags), _stream())
    L.star_build_rank(_ptr(dirw), rng_, _stream())
    for s in scans:
        L.star_build_fill(C.byref(s), 1, 2, pk_min, rng_, GRP_MIN, NGRP - 1, _ptr(dirw), _ptr(slots), _stream())
    m = {}
    for cols in dims:
        r = np.flatnonzero(R.eval_terms(cols, DIM_PRED, nd))
        m.update(G.star_map(cols[1], r, _grp_slot(cols[2], r))[0])
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir = 2, slots.data_ptr(), pk_min, rng_, dirw.data_ptr()
    out.append(("bitmap", lk, m, (dirw, slots, scans)))
    # dense and hash over one (selected) partition
    dim = dims[0]
    sel, sor = _dim_selection(dim, rng)
    from tests.test_gpu_rowwise import Dev
    d, sel_t, sor_t = Dev(dim[1]), _t(sel), _t(sor)
    lookup = torch.full((rng_,), -1, dtype=torch.int32, device=_dev())
    L.star_build_dense(C.byref(d.struct()), _ptr(sel_t), len(sel), _ptr(sor_t), pk_min, rng_, _ptr(lookup), _ptr(flags),
                       _stream())
    m1 = G.star_map(dim[1], sel, sor)[0]
    lk1 = L.StarLookup()
    lk1.dense, lk1.lookup, lk1.kmin, lk1.range = 1, lookup.data_ptr(), pk_min, rng_
    out.append(("dense", lk1, m1, (lookup, d, sel_t, sor_t)))
    cap = 8192
    tk, ts = _full(cap, G.EMPTY_KEY), _full(cap, 0x5A5A5A5A, dtype=torch.int32)
    L.star_build_hash(C.byref(d.struct()), _ptr(sel_t), len(sel), _ptr(sor_t), _ptr(tk), _ptr(ts), cap, _ptr(flags),
                      _stream())
    lk2 = L.StarLookup()
    lk2.dense, lk2.table_keys, lk2.table_slots, lk2.cap = 0, tk.data_ptr(), ts.data_ptr(), cap
    out.append(("hash", lk2, m1, (tk, ts)))
    assert not _np(flags)[:2].any()
    return pk_min, rng_, out


@pytest.mark.parametrize("n", [1, 4097, 100_003])
def test_bitwise_star_agg(n):
    rng = np.random.default_rng(7000 + n)
    pk_min, rng_, lookups = _star_lookups(rng)
    facts = [_bits_cols(fact_part(n, rng, pk_min, rng_), rng) for _ in range(1 + n % 3)]
    for name, lk, m, _keep in lookups:
        for terms in (PRED, []):
            st, outs = run_star_agg(lk, facts, terms, STAR_BIT_SPECS, NGRP)
            gids = [G.star_slots(cols[1], R.eval_terms(cols, terms, cols[0].n), m) for cols in facts]
            ex = B.aggregate(_concat_inputs(facts, STAR_BIT_SPECS), [op for _, op in STAR_BIT_SPECS],
                             np.concatenate(gids), NGRP)
            st.check(ex, True, f"star {name} n={n} terms={terms}")
            check_out_slots(outs, gids, f"star {name}")


# ---- global: b2_join_agg (generic kernel) and b2_scan_agg ----------------------------------------------------
@pytest.mark.parametrize("n", [0, 33, 4097, 100_003])
def test_bitwise_join_agg(n):
    """AND / OR / XOR of P, B and the int combinations P*B, P+B, P-B, B-P (I64, U32 + base, sentinel U32
    payloads), two partitions combined with accumulate = 1; the fast kernel is SUM-only, so every case runs the
    generic kernel"""
    rng = np.random.default_rng(8000 + n)
    bs = build_side(rng)
    facts = [probe_part(n, rng), probe_part(n // 2 + 1, rng)]
    for comb in [G.JA_P, G.JA_B, G.JA_MUL, G.JA_ADD, G.JA_SUB, G.JA_RSUB]:
        for pc, bc in [(2, 0), (4, 2), (2, 3)]:
            aggs = [(pc, bc, comb, op) for op in (AND, OR, XOR)] + [(pc, bc, comb, COUNT), (-1, -1, G.JA_ROWS, COUNT)]
            for terms in ([], PRED):
                exp = join_agg_expected(facts, terms, 1, bs, BUILD, aggs)
                got = run_join_agg(facts, terms, 1, bs, BUILD, aggs)
                check_global(*got, exp, True, f"join_agg c{comb} p{pc} b{bc} terms={terms}")


@pytest.mark.parametrize("n", [0, 1, 33, 4097, 8229, 100_003])
def test_bitwise_scan_agg(n):
    """AND / OR / XOR over int64 edges (with and without NULLs) and U8, three partitions with accumulate; an
    empty input yields the identities -1 / 0 / 0"""
    import torch
    L = _L()
    rng = np.random.default_rng(9000 + n)
    parts = []
    for i in range(3):
        m = n + i
        parts.append([R.Column(rng.integers(-3, 10, m).astype(np.int64), None, R.I64),
                      R.Column(rng.choice(BIT_POOL, m) if m else np.zeros(0, np.int64), rng.random(m) < 0.1, R.I64),
                      R.Column(rng.choice(BIT_POOL[:4], m) if m else np.zeros(0, np.int64), None, R.I64),
                      R.Column(rng.integers(0, 2, m).astype(np.uint8), rng.random(m) < 0.1, R.U8)])
    specs = [(1, AND), (1, OR), (1, XOR), (2, AND), (3, AND), (3, OR), (3, XOR), (-1, COUNT)]
    for terms in ([], PRED):
        acc, cnt = _full(len(specs), 0x5A5A), _full(len(specs), 0x5A5A)
        ws = torch.empty(L.scan_agg_ws_bytes(), dtype=torch.uint8, device=_dev())
        gids = []
        for i, cols in enumerate(parts):
            L.scan_agg(C.byref(scan_of(cols, terms)), _aggs(specs), len(specs), _ptr(acc), _ptr(cnt), 1 if i else 0,
                       _ptr(ws), _stream())
            gids.append(np.where(R.eval_terms(cols, terms, cols[0].n), 0, -1))
        ins = _concat_inputs(parts, specs)
        ops = [op for _, op in specs]
        ex = B.aggregate(ins, ops, np.concatenate(gids), 1)
        check_global(_np(acc), _np(cnt), B.global_words(ex, ops, ins), True, f"scan_agg n={n} terms={terms}")


# ---- the 32-bit word combine and argument checks --------------------------------------------------------------
def test_bitwise_combine_and_argument_checks():
    import torch
    L = _L()
    rng = np.random.default_rng(3)
    a = rng.integers(-2 ** 63, 2 ** 63 - 1, 1001, dtype=np.int64)
    b = rng.integers(-2 ** 63, 2 ** 63 - 1, 1001, dtype=np.int64)
    for op, f in ((AND, np.bitwise_and), (OR, np.bitwise_or), (XOR, np.bitwise_xor)):
        d, s = _t(a.copy()), _t(b)
        L.bitwise_combine(_ptr(d), _ptr(s), 2 * 1001, op, _stream())
        _eq(_np(d), f(a, b), f"combine op {op}")
    with pytest.raises(L.B200SqlError, match="bad bitwise op"):
        L.bitwise_combine(_ptr(d), _ptr(s), 2, SUM, _stream())
    cols = [R.Column(np.zeros(4, np.int64), None, R.I64), R.Column(np.ones(4), None, R.F64)]
    acc, cnt = _full(1, 0), _full(1, 0)
    ws = torch.empty(L.scan_agg_ws_bytes(), dtype=torch.uint8, device=_dev())
    for op in (AND, OR, XOR):
        with pytest.raises(L.B200SqlError, match="bitwise"):
            L.scan_agg(C.byref(scan_of(cols, [])), _aggs([(1, op)]), 1, _ptr(acc), _ptr(cnt), 0, _ptr(ws), _stream())
    with pytest.raises(L.B200SqlError, match="bad agg op"):
        L.scan_agg(C.byref(scan_of(cols, [])), _aggs([(0, XOR + 1)]), 1, _ptr(acc), _ptr(cnt), 0, _ptr(ws), _stream())
