"""The group-by and fused-aggregate kernels word for word against the NumPy reference of
tests/groupagg_ref.py, through the C-ABI: b2_groupby_dense and its _grouped / _hot / _ordered variants (with
b2_hot_slots and b2_range_partition_*), b2_groupby_hash1, b2_groupby_hashk, b2_star_agg over its three lookup
kinds with their builds, b2_join_agg (fast and generic kernels) and the aggregates of b2_scan_agg.

Every word of the state is compared: int SUM, MIN, MAX, counts, rows, the presence bitmap and out_slot
bit-exact (out_slot starts as garbage); float SUMs bit-exact on dyadic data, the sign of zero included, and
within the exact-sum bound elsewhere.  Slots no row reaches must keep the caller's initial words.  Several
partitions accumulate into one state, so the combination across calls is covered too."""
import ctypes as C
import math
import os
from contextlib import contextmanager

import numpy as np
import pytest

from tests import groupagg_ref as G
from tests import rowwise_ref as R
from tests.test_gpu_rowwise import Dev, _dev, _L, _ptr, _stream, make_scan

pytestmark = pytest.mark.gpu

MIN, MAX = R.INT64_MIN, R.INT64_MAX
SUM, SUMF, AMIN, AMAX, COUNT = G.AGG_SUM, G.AGG_SUMF, G.AGG_MIN, G.AGG_MAX, G.AGG_COUNT
SIZES = [0, 1, 31, 32, 33, 2047, 2048, 2049, 4095, 4096, 4097, 8229, 100_003]   # 8229 > 4 x 2048: staged path
BIG_INTS = np.array([MAX, MIN, MAX - 1, MIN + 1, 2 ** 62, -2 ** 62, 2 ** 53 + 1, -7, 0, 3], np.int64)
EDGE_FLOATS = np.array([0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, math.nan,
                        1.5, -1.5, 1.7976931348623157e308, -1.7976931348623157e308])
PRED = [(0, R.GE, 0, 0, 0.0)]       # the predicate term: column 0 (p) >= 0


@contextmanager
def env(**kw):
    """environment switches the library reads on every call (B200SQL_NO_HOT_TABLE, B200SQL_JA_*)"""
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _t(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).to(_dev())


def _full(n, value, dtype=None):
    import torch
    return torch.full((max(n, 1),), value, dtype=dtype or torch.int64, device=_dev())


def _np(t, n=None):
    import torch
    torch.cuda.synchronize()
    a = t.cpu().numpy()
    return a if n is None else a[:n]


def scan_of(cols, terms):
    """a b2_scan_t over device copies of `cols`.  The struct holds raw pointers only, so the copies ride on
    it: freed any earlier, their memory could be handed to the next allocation before the kernel runs."""
    devs = [Dev(c) for c in cols]
    s = make_scan(devs, terms, cols[0].n)
    s.devs = devs
    return s


def _aggs(specs):
    L = _L()
    arr = (L.Agg * max(1, len(specs)))()
    for i, (c, op) in enumerate(specs):
        arr[i].col, arr[i].op = c, op
    return arr


# ---- the aggregation state --------------------------------------------------------------------------------
class State:
    """a b2_aggstate_t initialised as the header prescribes: SUM / COUNT 0 (-0.0 for the indicator SUM), MIN
    INT64_MAX, MAX INT64_MIN.  cnt arrays: every aggregate when `cnt`, else only COUNT's."""

    def __init__(self, specs, dtypes, nslots, indicator=None, cnt=True, rows=True, present=True):
        import torch
        L = _L()
        self.specs, self.dtypes, self.nslots, self.indicator = specs, dtypes, nslots, indicator
        self.st = L.AggState()
        self.acc, self.cnt = [], []
        for a, ((c, op), dt) in enumerate(zip(specs, dtypes)):
            acc = _full(nslots, G.initial_word(op, dt, indicator == a)) if c >= 0 and op != COUNT else None
            cn = _full(nslots, 0) if c >= 0 and (cnt or op == COUNT) else None
            self.acc.append(acc), self.cnt.append(cn)
            self.st.acc[a] = acc.data_ptr() if acc is not None else 0
            self.st.cnt[a] = cn.data_ptr() if cn is not None else 0
        self.rows = _full(nslots, 0) if rows or any(c < 0 for c, _ in specs) else None
        self.present = _full((nslots + 31) // 32, 0, dtype=torch.int32) if present else None
        self.st.rows = self.rows.data_ptr() if self.rows is not None else 0
        self.st.present = self.present.data_ptr() if self.present is not None else 0

    def with_out_slot(self, buf):
        self.st.out_slot = buf.data_ptr() if buf is not None else 0
        return C.byref(self.st)

    def check(self, ex: G.Expected, dyadic, what, slots=None):
        """every word of slots [0, nslots) (or the listed ones) against the reference"""
        n = self.nslots
        sel = np.arange(n) if slots is None else np.asarray(slots)
        if self.rows is not None:
            _eq(_np(self.rows, n)[sel], ex.rows[sel], f"{what}: rows")
        if self.present is not None:
            words = G.pack_bits(ex.present)
            got = _np(self.present).view(np.uint32)[: len(words)]
            if slots is None:
                _eq(got, words, f"{what}: presence bitmap")
            else:
                bits = np.unpackbits(got.view(np.uint8), bitorder="little")[sel].astype(bool)
                _eq(bits, ex.present[sel], f"{what}: presence bits")
        for a, ((c, op), dt) in enumerate(zip(self.specs, self.dtypes)):
            if self.cnt[a] is not None:
                _eq(_np(self.cnt[a], n)[sel], ex.cnt[a][sel], f"{what}: cnt[{a}]")
            if self.acc[a] is None:
                continue
            got = _np(self.acc[a], n)[sel]
            if G.is_float_sum(op, dt):
                G.check_float_sum(got, ex.exact[a][sel], ex.bound[a][sel], ex.touched[a][sel],
                                  G.initial_word(op, dt, self.indicator == a), dyadic, f"{what}: float sum acc[{a}]")
            else:
                _eq(got, ex.acc[a][sel], f"{what}: acc[{a}] (op {op})")


def _eq(got, exp, what):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, f"{what}: shape {got.shape} vs {exp.shape}"
    bad = np.flatnonzero(got != exp)
    if len(bad):
        i = bad[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} words differ; first at {i}: got {got[i]!r}, "
                             f"expected {exp[i]!r}")


# ---- data of the dense family -----------------------------------------------------------------------------
# columns: 0 p (predicate), 1 key, 2 vi (int64, huge, NULLs), 3 vf (dyadic float, -0.0, NaN), 4 vm (IEEE edges
# for MIN / MAX), 5 vs (small int64, no bitmap: SUMF), 6 vz (never-NULL dyadic float: the -0.0 indicator)
P, KEY, VI, VF, VM, VS, VZ = range(7)
KMIN = -1000
K_FAIL = KMIN + 7      # a key whose rows all fail the predicate: hottest key of the skewed shapes


def _keys(shape, n, rng, span=500):
    r = np.arange(n)
    if shape == "uniform":
        k = rng.integers(0, span, n)
    elif shape == "one":
        k = np.full(n, 3)
    elif shape == "two":
        k = np.where(r % 2 == 0, 3, 11)
    elif shape == "hitters33":       # 40 keys of ~2 % each, the K_FAIL key at 20 %, a uniform tail
        u = rng.random(n)
        k = np.where(u < 0.2, K_FAIL - KMIN, np.where(u < 0.2 + 40 * 0.02, 20 + rng.integers(0, 40, n),
                                                      rng.integers(0, span, n)))
    elif shape == "many_repeats":    # pairs of rows share a key, > 256 distinct per CTA: overflows the table
        k = (r // 2) % 1500
    elif shape == "zipf":
        k = np.minimum(rng.zipf(1.3, n) - 1, span - 1)
        k = np.where(k == 0, K_FAIL - KMIN, k)
    else:
        raise ValueError(shape)
    return k.astype(np.int64) + KMIN


def dense_part(shape, n, rng, span=500, zero_indicator=None):
    keys = _keys(shape, n, rng, span)
    p = rng.integers(-3, 10, n).astype(np.int64)
    p[keys == K_FAIL] = -1
    knull = rng.random(n) < (0.0 if shape == "one" else 0.03)
    vi = rng.choice(BIG_INTS, n) if n else np.zeros(0, np.int64)
    vf = rng.integers(-2 ** 20, 2 ** 20, n) * 2.0 ** -10
    vf[rng.random(n) < 0.05] = -0.0
    vf[rng.random(n) < 0.05] = math.nan
    vm = rng.choice(EDGE_FLOATS, n) if n else np.zeros(0)
    vs = rng.integers(-2 ** 20, 2 ** 20, n).astype(np.int64)
    vz = rng.integers(-64, 64, n) * 0.25
    if zero_indicator == "neg_zero":
        vz = np.full(n, -0.0)
    elif zero_indicator == "cancel":      # rows come in pairs (same key, same predicate) of +1.0 and -1.0
        keys[1::2], p[1::2] = keys[0::2][: n // 2], p[0::2][: n // 2]
        vz = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
        if n % 2:
            vz[-1] = -0.0
        knull[:] = False
    return [R.Column(p, None, R.I64), R.Column(keys, knull, R.I64),
            R.Column(vi, rng.random(n) < 0.1, R.I64), R.Column(vf, rng.random(n) < 0.05, R.F64),
            R.Column(vm, rng.random(n) < 0.05, R.F64), R.Column(vs, None, R.I64), R.Column(vz, None, R.F64)]


SPECS = {
    # 3 carried arrays (rows, two SUM accumulators): the per-CTA table of the grouped kernel is on
    "three": ([(-1, COUNT), (VF, SUM), (VI, SUM)], False),
    # eight aggregates with a cnt array each: more than 4 carried arrays switch the table off
    "eight": ([(-1, COUNT), (VI, SUM), (VI, AMIN), (VM, AMAX), (VM, AMIN), (VF, SUM), (VF, COUNT), (VS, SUMF)], True),
    # a never-NULL float SUM that starts at -0.0 and is the only existence mark
    "indicator": ([(VZ, SUM), (VS, SUM)], False),
}


def _dtypes(cols, specs):
    return [cols[c].dtype if c >= 0 else R.I64 for c, _ in specs]


def dense_expected(parts, terms, key_col, kmin, nslots, specs, indicator=None):
    gids = []
    for cols in parts:
        n = cols[0].n
        ok = R.eval_terms(cols, terms, n)
        gids.append(G.dense_slots(cols[key_col], ok, kmin, nslots))
    gid = np.concatenate(gids) if gids else np.zeros(0, np.int64)
    inputs = []
    for a, (c, _) in enumerate(specs):
        if c < 0:
            inputs.append(None)
            continue
        cs = [cols[c] for cols in parts]
        inputs.append(R.Column(np.concatenate([x.values for x in cs]),
                               np.concatenate([x.null_mask() for x in cs]), cs[0].dtype))
    return G.aggregate(inputs, [op for _, op in specs], gid, nslots, indicator), gids


def run_dense_kernel(variant, parts, terms, key_col, kmin, nslots, specs, state, hot=None):
    """run one of the dense kernels over every partition into `state`; returns the out_slot buffers"""
    import torch
    L = _L()
    outs = []
    for cols in parts:
        n = cols[0].n
        devs = [Dev(c) for c in cols]
        scan = make_scan(devs, terms, n)
        buf = _full(n, 0x5A5A5A5A, dtype=torch.int32)
        st = state.with_out_slot(buf)
        args = (C.byref(scan), key_col, kmin, nslots, _aggs(specs), len(specs), st)
        if variant == "dense":
            L.groupby_dense(*args, _stream())
        elif variant == "grouped":
            L.groupby_dense_grouped(*args, _stream())
        elif variant == "grouped_no_table":
            with env(B200SQL_NO_HOT_TABLE=1):
                L.groupby_dense_grouped(*args, _stream())
        elif variant == "hot":
            L.groupby_dense_hot(*args, _ptr(hot), _stream())
        else:
            raise ValueError(variant)
        outs.append((buf, n))
    return outs


def check_out_slots(outs, gids, what):
    for (buf, n), g in zip(outs, gids):
        _eq(_np(buf, n).astype(np.int64), g, f"{what}: out_slot")


def hot_lists(parts, kmin, nslots, terms):
    """the three hot lists of b2_groupby_dense_hot: b2_hot_slots' own, all -1, and a hostile one (duplicates,
    the NULL slot, slots no row hits, slots whose rows all fail the predicate), all inside [0, nslots)"""
    import torch
    L = _L()
    key = Dev(parts[0][KEY])
    sampled = torch.full((32,), 77, dtype=torch.int32, device=_dev())
    L.hot_slots(C.byref(key.struct()), parts[0][KEY].n, kmin, nslots, _ptr(sampled), _stream())
    hit = set()
    for cols in parts:
        hit |= set(G.dense_slots(cols[KEY], R.eval_terms(cols, terms, cols[0].n), kmin, nslots).tolist())
    unused = [s for s in range(nslots - 1) if s not in hit][:4]
    hostile = [K_FAIL - kmin, K_FAIL - kmin, nslots - 1, 3, 3] + unused + [8, 11, 0, 1, nslots - 2, 3, 11]
    hostile = [s for s in hostile if 0 <= s < nslots]
    hostile = np.resize(np.array(hostile, np.int32), 32)
    return {"sampled": sampled, "none": _t(np.full(32, -1, np.int32)), "hostile": _t(hostile)}


def check_dense_family(parts, terms, kmin, nslots, spec, what, dyadic=True, ordered=True, hot=True):
    """the same partitions through dense, grouped (table on and off), hot (three lists) and, when `ordered`,
    range partition + ordered; spec: a name of SPECS or (specs, keep a cnt array per aggregate)"""
    specs, cnt = SPECS[spec] if isinstance(spec, str) else spec
    dtypes = _dtypes(parts[0], specs)
    indicator = 0 if spec == "indicator" else None
    ex, gids = dense_expected(parts, terms, KEY, kmin, nslots, specs, indicator)
    variants = ["dense", "grouped", "grouped_no_table"]
    lists = hot_lists(parts, kmin, nslots, terms) if hot and parts[0][KEY].dtype == R.I64 else {}
    for v in variants + [("hot", k) for k in lists]:
        name, hl = (v, None) if isinstance(v, str) else (v[0], lists[v[1]])
        st = State(specs, dtypes, nslots, indicator, cnt=cnt, present=indicator is None)
        outs = run_dense_kernel(name, parts, terms, KEY, kmin, nslots, specs, st, hl)
        label = f"{what} {v}"
        st.check(ex, dyadic, label)
        check_out_slots(outs, gids, label)
    if ordered and parts[0][KEY].dtype == R.I64:
        check_ordered(parts, terms, kmin, nslots, specs, dtypes, ex, indicator, dyadic, what)


# ---- b2_range_partition_* + b2_groupby_dense_ordered ---------------------------------------------------
def check_ordered(parts, terms, kmin, nslots, specs, dtypes, ex, indicator, dyadic, what, nbuckets=None):
    """reorder every partition by key range into ONE output (hist per input, scan once, scatter per input),
    check the buckets against the reference, then aggregate the output with b2_groupby_dense_ordered
    (nslots + 1 slots: the reordered NULL key is the value kmin + nslots - 1)"""
    import torch
    L = _L()
    carry = sorted({c for c, _ in specs if c >= 0})
    for c in carry:
        assert parts[0][c].null is None, "carried columns have no bitmap"
    shift = max(0, int(math.ceil(math.log2(max(nslots, 2)))) - 4)
    nbuckets = nbuckets or (((nslots - 1) >> shift) + 1)
    total_n = sum(cols[0].n for cols in parts)
    ws = torch.zeros(L.range_partition_ws_bytes(nbuckets) // 8, dtype=torch.int64, device=_dev())
    fill = kmin + nslots + 1
    out_key = _full(total_n, fill)
    out_cols = [_full(total_n, 0x5A5A) for _ in carry]
    scans = []
    for cols in parts:
        devs = [Dev(c) for c in cols]
        scans.append((make_scan(devs, terms, cols[0].n), devs))
        L.range_partition_hist(C.byref(scans[-1][0]), KEY, kmin, nslots, shift, nbuckets, _ptr(ws), _stream())
    L.range_partition_scan(nbuckets, _ptr(ws), _stream())
    cc = (C.c_int32 * max(1, len(carry)))(*carry)
    oc = (C.c_void_p * max(1, len(carry)))(*[o.data_ptr() for o in out_cols])
    for scan, _ in scans:
        L.range_partition_scatter(C.byref(scan), KEY, kmin, nslots, shift, nbuckets, len(carry), cc, _ptr(out_key), oc,
                                  _ptr(ws), _stream())
    passing = [R.eval_terms(cols, terms, cols[0].n) for cols in parts]
    starts, buckets = G.range_partition(parts, passing, KEY, kmin, nslots, shift, nbuckets, carry)
    _eq(_np(ws)[: nbuckets + 1], starts, f"{what}: bucket starts")
    got_key = _np(out_key, total_n)
    got_cols = [_np(o, total_n) for o in out_cols]
    for b in range(nbuckets):
        rows = np.stack([got_key[starts[b]:starts[b + 1]]] + [g[starts[b]:starts[b + 1]] for g in got_cols], axis=1)
        rows = rows[np.lexsort(rows.T[::-1])] if len(rows) else rows
        _eq(rows.reshape(-1), buckets[b].reshape(-1), f"{what}: rows of bucket {b}")
    _eq(got_key[starts[-1]:], np.full(total_n - starts[-1], fill), f"{what}: rows past the total")
    # aggregate the reordered rows
    cols2 = [R.Column(got_key, None, R.I64)] + [R.Column(g.view(np.float64) if parts[0][c].dtype == R.F64 else g,
                                                         None, parts[0][c].dtype) for g, c in zip(got_cols, carry)]
    devs2 = [Dev(R.Column(np.ascontiguousarray(c.values[:total_n]), None, c.dtype)) for c in cols2]
    devs2[0].data = out_key[:max(total_n, 1)]
    for d, o in zip(devs2[1:], out_cols):
        d.data = o[:max(total_n, 1)]
    scan2 = make_scan(devs2, [], total_n)
    specs2 = [(1 + carry.index(c) if c >= 0 else -1, op) for c, op in specs]
    st = State(specs2, dtypes, nslots + 1, indicator, cnt=True, present=indicator is None)
    buf = _full(total_n, 0x5A5A5A5A, dtype=torch.int32)
    ticket = torch.zeros(1, dtype=torch.int64, device=_dev())
    L.groupby_dense_ordered(C.byref(scan2), 0, kmin, nslots + 1, _aggs(specs2), len(specs2), st.with_out_slot(buf),
                            _ptr(ticket), _stream())
    ex2 = G.Expected(nslots + 1)
    ex2.rows, ex2.present = np.r_[ex.rows, 0], np.r_[ex.present, False]
    for a in range(len(specs)):
        ex2.acc.append(None if ex.acc[a] is None else np.r_[ex.acc[a], G.initial_word(specs[a][1], dtypes[a])])
        ex2.exact.append(None if ex.exact[a] is None else np.r_[ex.exact[a], 0.0])
        ex2.bound.append(None if ex.bound[a] is None else np.r_[ex.bound[a], 0.0])
        ex2.touched.append(None if ex.touched[a] is None else np.r_[ex.touched[a], False])
        ex2.cnt.append(np.r_[ex.cnt[a], 0])
    st.check(ex2, dyadic, f"{what} ordered")
    exp_slot = np.where(np.arange(total_n) < starts[-1], got_key - kmin, -1)
    _eq(_np(buf, total_n).astype(np.int64), exp_slot, f"{what} ordered: out_slot")


# ---- the dense family: sizes, predicate, skew shapes, key edges --------------------------------------------
@pytest.mark.parametrize("pred", [False, True], ids=["all_rows", "predicate"])
@pytest.mark.parametrize("n", SIZES)
def test_groupby_dense_family_sizes(n, pred):
    rng = np.random.default_rng(n * 2 + pred)
    nparts = 1 + n % 3
    parts = [dense_part("uniform" if i % 2 == 0 else "zipf", n, rng) for i in range(nparts)]
    terms = PRED if pred else []
    for spec in ("three", "eight"):
        specs = SPECS[spec][0]
        ordered = all(parts[0][c].null is None for c, _ in specs if c >= 0)
        check_dense_family(parts, terms, KMIN, 502, spec, f"n={n} x{nparts} {spec}", ordered=ordered)
    check_dense_family(parts, terms, KMIN, 502, "indicator", f"n={n} x{nparts} indicator")


ORDERED_SPEC = [(-1, COUNT), (VF, SUM), (VM, AMIN), (VM, AMAX), (VS, SUMF), (VS, SUM), (VZ, COUNT)]


@pytest.mark.parametrize("pred", [False, True], ids=["all_rows", "predicate"])
@pytest.mark.parametrize("n", [0, 33, 4097, 8229, 100_003])
def test_groupby_dense_ordered_after_range_partition(n, pred):
    """3 inputs reordered into one output, then aggregated in key-range order"""
    rng = np.random.default_rng(100 + n + pred)
    parts = [dense_part("uniform", n + i, rng, span=1500) for i in range(3)]
    for cols in parts:      # carried columns have no bitmap (NaN still makes NULLs)
        cols[VF].null = cols[VM].null = None
    terms = PRED if pred else []
    nslots = 1502
    dtypes = _dtypes(parts[0], ORDERED_SPEC)
    ex, _ = dense_expected(parts, terms, KEY, KMIN, nslots, ORDERED_SPEC)
    check_ordered(parts, terms, KMIN, nslots, ORDERED_SPEC, dtypes, ex, None, True, f"n={n}")


@pytest.mark.parametrize("spec", ["three", "eight", "indicator"])
@pytest.mark.parametrize("shape", ["one", "two", "hitters33", "many_repeats", "zipf"])
def test_groupby_dense_family_skew(shape, spec):
    """one key for all rows, two alternating, 33+ hitters, > 256 repeating slots per CTA, Zipf; the hottest
    key of the hitter shapes has all its rows filtered out (b2_hot_slots lists it, no group may appear)"""
    rng = np.random.default_rng(10 * len(shape) + len(spec))
    n = 100_003
    span = 1500 if shape == "many_repeats" else 500
    parts = [dense_part(shape, n, rng, span), dense_part(shape, 4097, rng, span)]
    check_dense_family(parts, PRED, KMIN, span + 2, spec, f"{shape} {spec}", ordered=False)


@pytest.mark.parametrize("zero", ["neg_zero", "cancel"])
@pytest.mark.parametrize("shape", ["one", "two", "zipf", "uniform"])
def test_groupby_dense_indicator_zero_sums(shape, zero):
    """a never-NULL float SUM whose values are all -0.0, or cancel to 0: every touched group reads +0.0,
    every untouched slot keeps -0.0"""
    rng = np.random.default_rng(7)
    parts = [dense_part(shape, 100_003, rng, zero_indicator=zero), dense_part(shape, 2049, rng, zero_indicator=zero)]
    check_dense_family(parts, PRED, KMIN, 502, "indicator", f"{shape} {zero}", ordered=False)


@pytest.mark.parametrize("edge", ["int64_max", "int64_min", "u8"])
def test_groupby_dense_key_edges(edge):
    """key ranges that touch INT64_MAX / INT64_MIN (slots in uint64 arithmetic; keys outside the range are
    dropped), and U8 (boolean) keys with NULLs"""
    rng = np.random.default_rng(11)
    n = 8229
    parts = [dense_part("uniform", n, rng) for _ in range(2)]
    if edge == "u8":
        for cols in parts:
            cols[KEY] = R.Column(rng.integers(0, 2, n).astype(np.uint8), rng.random(n) < 0.2, R.U8)
        kmin, nslots = 0, 3
    else:
        kmin = MAX - 100 if edge == "int64_max" else MIN
        nslots = 102
        for cols in parts:
            off = rng.integers(0, 101, n)
            k = (np.uint64(kmin & 0xFFFFFFFFFFFFFFFF) + off.astype(np.uint64)).view(np.int64)
            outside = rng.random(n) < 0.02
            k[outside] = (kmin - 1) if edge == "int64_max" else MAX   # below kmin / far above the range
            cols[KEY] = R.Column(k, cols[KEY].null, R.I64)
    for spec in ("three", "eight"):
        check_dense_family(parts, PRED, kmin, nslots, spec, f"{edge} {spec}", ordered=False, hot=edge != "u8")
    if edge == "u8":   # dense_hot with a given list still works on U8 keys
        specs = SPECS["three"][0]
        ex, gids = dense_expected(parts, PRED, KEY, kmin, nslots, specs)
        for hl in ([0, 1, 2, 2] + [-1] * 28, [2, 1, 0] * 10 + [1, 1]):
            st = State(specs, _dtypes(parts[0], specs), nslots, cnt=False)
            outs = run_dense_kernel("hot", parts, PRED, KEY, kmin, nslots, specs, st, _t(np.array(hl, np.int32)))
            st.check(ex, True, f"u8 hot {hl[:4]}")
            check_out_slots(outs, gids, "u8 hot")


def test_groupby_dense_float_sums_within_the_bound():
    """general (non-dyadic) float values and SUMF over int64 beyond 2^53: within gamma_{m-1} sum |x| of fsum"""
    rng = np.random.default_rng(12)
    parts = []
    for n in (100_003, 8229):
        cols = dense_part("zipf", n, rng)
        cols[VF] = R.Column(rng.normal(0, 1, n) * 10.0 ** rng.integers(-8, 9, n), cols[VF].null, R.F64)
        cols[VS] = R.Column(rng.integers(-2 ** 62, 2 ** 62, n), None, R.I64)
        parts.append(cols)
    specs = [(-1, COUNT), (VF, SUM), (VS, SUMF), (VF, SUMF)]
    check_dense_family(parts, PRED, KMIN, 502, (specs, True), "general floats", dyadic=False, ordered=False)


def test_groupby_dense_float_sum_overflows_to_inf():
    """all values large and positive: the exact sum is beyond float64 and every order gives +inf"""
    n = 4097
    rng = np.random.default_rng(13)
    cols = dense_part("two", n, rng)
    cols[VF] = R.Column(np.full(n, 1.0e308), None, R.F64)
    check_dense_family([cols], [], KMIN, 502, ([(VF, SUM)], False), "overflow", dyadic=False, ordered=False)


# ---- b2_hot_slots --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2049, 100_003, 1_000_003])
def test_hot_slots_properties(n):
    """sampling is not exact, so only properties: distinct entries in [0, nslots - 1), -1 padding from the first
    -1 on, a key holding >= 20 % of the rows (no other above 5 %) listed first, never a slot no row holds"""
    import torch
    L = _L()
    rng = np.random.default_rng(n)
    kmin, nslots = -50, 3002
    k = rng.integers(0, 3000, n)
    k[rng.random(n) < 0.25] = 1234
    k[k == 999] = 998                  # 999 is held by no row
    col = R.Column(k.astype(np.int64) + kmin, rng.random(n) < 0.05, R.I64)
    d = Dev(col)
    out = torch.full((32,), 77, dtype=torch.int32, device=_dev())
    L.hot_slots(C.byref(d.struct()), n, kmin, nslots, _ptr(out), _stream())
    got = _np(out)
    live = got[got >= 0]
    first_pad = np.flatnonzero(got < 0)
    if len(first_pad):
        assert (got[first_pad[0]:] == -1).all(), got
    assert len(set(live.tolist())) == len(live), got
    assert ((live >= 0) & (live < nslots - 1)).all(), got
    assert 999 not in live.tolist()
    held = set((k[~col.null]).tolist())
    assert set(live.tolist()) <= held, got
    if n >= 2049:
        assert got[0] == 1234, got


# ---- b2_groupby_hash1 ------------------------------------------------------------------------------------------
def _hash_inputs(n, rng):
    """value columns shared by the hash tests (after the key columns): vi, vf, vm, vs"""
    vi = rng.choice(BIG_INTS, n) if n else np.zeros(0, np.int64)
    vf = rng.integers(-2 ** 20, 2 ** 20, n) * 2.0 ** -10
    vf[rng.random(n) < 0.05] = -0.0
    vf[rng.random(n) < 0.05] = math.nan
    vm = rng.choice(EDGE_FLOATS, n) if n else np.zeros(0)
    return [R.Column(vi, rng.random(n) < 0.1, R.I64), R.Column(vf, rng.random(n) < 0.05, R.F64),
            R.Column(vm, rng.random(n) < 0.05, R.F64), R.Column(rng.integers(-2 ** 20, 2 ** 20, n), None, R.I64)]


def _hash_specs(base):
    vi, vf, vm, vs = base, base + 1, base + 2, base + 3
    return [(-1, COUNT), (vi, SUM), (vi, AMIN), (vm, AMAX), (vm, AMIN), (vf, SUM), (vf, COUNT), (vs, SUMF)]


def _concat_inputs(parts, specs):
    out = []
    for c, _ in specs:
        if c < 0:
            out.append(None)
            continue
        cs = [cols[c] for cols in parts]
        out.append(R.Column(np.concatenate([x.values for x in cs]), np.concatenate([x.null_mask() for x in cs]),
                            cs[0].dtype))
    return out


I64_KEY_POOL = np.array([MIN, MIN + 1, MAX, -1, 0, 1, 2 ** 53 + 1, 42, -42, 7, 8, 9], np.int64)
NAN_PAYLOADS = np.array([0x7FF8000000000000, 0x7FF8000000000001, -0x0007FFFFFFFFFFFF, 0x7FF0000000000001,
                         -0x0008000000000000], np.int64).view(np.float64)   # quiet / signalling, both signs
F64_KEY_POOL = np.r_[[0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 1.5, -1.5, 2.0 ** 63], NAN_PAYLOADS]


def hash_part(kind, n, rng):
    if kind == "i64":
        key = R.Column(rng.choice(I64_KEY_POOL, n), rng.random(n) < 0.05, R.I64)
    elif kind == "f64":
        key = R.Column(rng.choice(F64_KEY_POOL, n), rng.random(n) < 0.05, R.F64)
    else:   # many distinct int keys
        key = R.Column(rng.integers(-2 ** 40, 2 ** 40, n) * 3, rng.random(n) < 0.01, R.I64)
    p = R.Column(rng.integers(-3, 10, n).astype(np.int64), None, R.I64)
    return [p, key] + _hash_inputs(n, rng)


def run_hash1(parts, terms, cap, specs):
    import torch
    L = _L()
    dtypes = _dtypes(parts[0], specs)
    st = State(specs, dtypes, cap + 2)
    tk = _full(cap + 2, G.EMPTY_KEY)
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    outs = []
    for cols in parts:
        n = cols[0].n
        scan = scan_of(cols, terms)
        buf = _full(n, 0x5A5A5A5A, dtype=torch.int32)
        L.groupby_hash1(C.byref(scan), 1, _ptr(tk), cap, _aggs(specs), len(specs), st.with_out_slot(buf), _ptr(flags),
                        _stream())
        outs.append((buf, n))
    return st, _np(tk), _np(flags), outs


def check_hash1(parts, terms, cap, what):
    specs = _hash_specs(2)
    st, tk, flags, outs = run_hash1(parts, terms, cap, specs)
    if flags[0]:
        return False
    ident, gids = [], []
    for cols in parts:
        ok = R.eval_terms(cols, terms, cols[0].n)
        ident += [x if ok[i] else None for i, x in enumerate(G.hash1_identity(cols[1]))]
    passing = np.array([x is not None for x in ident], bool)
    gid, groups = G.codes(ident, passing)
    ex = G.aggregate(_concat_inputs(parts, specs), [op for _, op in specs], gid, len(groups))
    # where the kernel put each group
    slot_of = {}
    for h in range(cap):
        if tk[h] != G.EMPTY_KEY:
            slot_of[int(tk[h])] = h
    slot_of[G.NULL_GROUP], slot_of[G.EMPTY_GROUP] = cap, cap + 1
    assert set(k for k in slot_of if k not in (G.NULL_GROUP, G.EMPTY_GROUP)) == \
        set(g for g in groups if g not in (G.NULL_GROUP, G.EMPTY_GROUP)), f"{what}: table keys"
    assert flags[1] == (G.NULL_GROUP in groups) and flags[2] == (G.EMPTY_GROUP in groups), f"{what}: flags {flags}"
    ex2 = G.permute(ex, [slot_of[g] for g in groups], cap + 2, inputs=_concat_inputs(parts, specs),
                    ops=[op for _, op in specs])
    st.check(ex2, True, what)
    got_slot = np.concatenate([_np(b, n).astype(np.int64) for b, n in outs]) if outs else np.zeros(0, np.int64)
    exp_slot = np.array([slot_of[x] if x is not None else -1 for x in ident], np.int64)
    _eq(got_slot, exp_slot, f"{what}: out_slot")
    return True


@pytest.mark.parametrize("pred", [False, True], ids=["all_rows", "predicate"])
@pytest.mark.parametrize("kind", ["i64", "f64", "wide"])
@pytest.mark.parametrize("n", [0, 1, 33, 2049, 8229, 100_003])
def test_groupby_hash1(n, kind, pred):
    """INT64_MIN keys in slot cap + 1, NULL and every NaN payload in slot cap, -0.0 with +0.0; a table too small
    must raise d_flags[0], and a rerun with room must match the reference"""
    rng = np.random.default_rng(n + len(kind) + pred)
    parts = [hash_part(kind, n, rng) for _ in range(1 + n % 3)]
    terms = PRED if pred else []
    if kind == "wide" and n >= 2049:
        assert not check_hash1(parts, terms, 8, f"{kind} n={n} cap=8"), "an overfull table must set d_flags[0]"
    cap = 1 << max(4, int(math.ceil(math.log2(max(1, 2 * n * len(parts))))))
    assert check_hash1(parts, terms, cap, f"{kind} n={n} cap={cap}"), "overflow with room to spare"


# ---- b2_groupby_hashk ------------------------------------------------------------------------------------------
def hashk_part(kinds, n, rng):
    keys = []
    for k in kinds:
        if k == "i64":
            keys.append(R.Column(rng.choice(np.array([0, 1, MIN, MAX, -1], np.int64), n), rng.random(n) < 0.3, R.I64))
        elif k == "f64":
            keys.append(R.Column(rng.choice(np.r_[[0.0, -0.0, 1.0, -math.inf], NAN_PAYLOADS[:2]], n),
                                 rng.random(n) < 0.3, R.F64))
        else:
            keys.append(R.Column(rng.integers(0, 2, n).astype(np.uint8), rng.random(n) < 0.3, R.U8))
    p = R.Column(rng.integers(-3, 10, n).astype(np.int64), None, R.I64)
    return [p] + keys + _hash_inputs(n, rng)


def check_hashk(parts, terms, nkeys, cap, what):
    import torch
    L = _L()
    specs = _hash_specs(1 + nkeys)
    dtypes = _dtypes(parts[0], specs)
    st = State(specs, dtypes, cap)
    tk = _full(nkeys * cap, 0x5A5A)
    tn = torch.full((cap,), 0x5A, dtype=torch.uint8, device=_dev())
    ts = torch.zeros(cap, dtype=torch.int32, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    kc = (C.c_int32 * nkeys)(*range(1, 1 + nkeys))
    outs = []
    for cols in parts:
        n = cols[0].n
        scan = scan_of(cols, terms)
        buf = _full(n, 0x5A5A5A5A, dtype=torch.int32)
        L.groupby_hashk(C.byref(scan), kc, nkeys, _ptr(tk), _ptr(tn), _ptr(ts), cap, _aggs(specs), len(specs),
                        st.with_out_slot(buf), _ptr(flags), _stream())
        outs.append((buf, n))
    if _np(flags)[0]:
        return False
    ident = []
    for cols in parts:
        ok = R.eval_terms(cols, terms, cols[0].n)
        ident += [x if ok[i] else None for i, x in enumerate(G.hashk_identity(cols[1:1 + nkeys]))]
    passing = np.array([x is not None for x in ident], bool)
    gid, groups = G.codes(ident, passing)
    ex = G.aggregate(_concat_inputs(parts, specs), [op for _, op in specs], gid, len(groups))
    tkh, tnh, tsh = _np(tk).reshape(nkeys, cap), _np(tn), _np(ts)
    slot_of = {}
    for h in np.flatnonzero(tsh == 2):
        slot_of[tuple(int(tkh[k, h]) for k in range(nkeys)) + (int(tnh[h]),)] = int(h)
    assert ((tsh == 0) | (tsh == 2)).all(), f"{what}: table state words {set(tsh.tolist())}"
    assert set(slot_of) == set(groups), f"{what}: table groups {sorted(slot_of)} vs {sorted(groups)}"
    ex2 = G.permute(ex, [slot_of[g] for g in groups], cap, inputs=_concat_inputs(parts, specs),
                    ops=[op for _, op in specs])
    st.check(ex2, True, what)
    got_slot = np.concatenate([_np(b, n).astype(np.int64) for b, n in outs])
    _eq(got_slot, np.array([slot_of[x] if x is not None else -1 for x in ident], np.int64), f"{what}: out_slot")
    return True


@pytest.mark.parametrize("kinds", [("i64",), ("f64",), ("u8",), ("i64", "i64"), ("i64", "f64", "u8"),
                                   ("u8", "f64", "i64", "f64")], ids="-".join)
@pytest.mark.parametrize("n", [1, 33, 4097, 100_003])
def test_groupby_hashk(n, kinds):
    """1 to 4 keys of mixed types with NULLs in every combination: (NULL, 0), (0, NULL) and (0, 0) are three
    groups; -0.0 is 0.0 and every NaN is NULL"""
    rng = np.random.default_rng(n + 31 * len(kinds))
    parts = [hashk_part(kinds, n, rng) for _ in range(1 + n % 3)]
    nk = len(kinds)
    if n >= 4097:
        assert not check_hashk(parts, PRED, nk, 2, f"{kinds} cap=2"), "an overfull table must set d_flags[0]"
    assert check_hashk(parts, PRED, nk, 4096, f"{kinds} n={n}")
    assert check_hashk(parts, [], nk, 4096, f"{kinds} n={n} no predicate")


def test_groupby_hashk_null_masks_are_distinct_groups():
    n = 6
    k0 = R.Column(np.zeros(n, np.int64), np.array([1, 0, 0, 1, 0, 0], bool), R.I64)
    k1 = R.Column(np.zeros(n, np.int64), np.array([0, 1, 0, 0, 1, 0], bool), R.I64)
    p = R.Column(np.zeros(n, np.int64), None, R.I64)
    cols = [p, k0, k1] + _hash_inputs(n, np.random.default_rng(0))
    assert check_hashk([cols], [], 2, 16, "null masks")
    assert len(set(G.hashk_identity([k0, k1]))) == 3


# ---- star: builds and b2_star_agg -------------------------------------------------------------------------------
STAR_SPECS = [(-1, COUNT), (2, SUM), (2, AMIN), (3, SUM), (4, AMAX), (4, AMIN), (3, COUNT), (5, SUMF)]


def fact_part(n, rng, pk_min, pk_range):
    """0 p, 1 fk (NULLs, outside the range, INT64_MIN), 2 vi, 3 vf, 4 vm, 5 vs"""
    fk = rng.integers(pk_min - 5, pk_min + pk_range + 5, n).astype(np.int64)
    fk[rng.random(n) < 0.01] = MIN
    p = R.Column(rng.integers(-3, 10, n).astype(np.int64), None, R.I64)
    return [p, R.Column(fk, rng.random(n) < 0.03, R.I64)] + _hash_inputs(n, rng)


def dim_part(n, rng, pk_min, holes=True, dup=None):
    """0 flag, 1 pk (a permutation with holes), 2 grp (NULLs)"""
    pk = rng.permutation(np.arange(pk_min, pk_min + 2 * n, 2 if holes else 1)[:n]).astype(np.int64)
    flag = rng.integers(0, 10, n).astype(np.int64)
    pk_null = rng.random(n) < 0.02
    if dup == "passing":
        pk[1], flag[0], flag[1], pk_null[:2] = pk[0], 0, 0, False
    elif dup == "filtered":
        pk[1], flag[0], flag[1], pk_null[:2] = pk[0], 0, 9, False
    return [R.Column(flag, None, R.I64), R.Column(pk, pk_null, R.I64),
            R.Column(rng.integers(100, 140, n).astype(np.int64), rng.random(n) < 0.05, R.I64)]


DIM_PRED = [(0, R.LT, 0, 5, 0.0)]
GRP_MIN, NGRP = 100, 41     # groups 0..39 plus the NULL slot 40


def run_star_agg(lk, facts, terms, specs, nslots):
    L = _L()
    st = State(specs, _dtypes(facts[0], specs), nslots)
    outs = []
    for cols in facts:
        n = cols[0].n
        scan = scan_of(cols, terms)
        buf = _full(n, 0x5A5A5A5A, dtype=__import__("torch").int32)
        L.star_agg(C.byref(scan), 1, C.byref(lk), _aggs(specs), len(specs), st.with_out_slot(buf), _stream())
        outs.append((buf, n))
    return st, outs


def check_star_agg(lk, facts, terms, pk_to_slot, what):
    specs = STAR_SPECS
    st, outs = run_star_agg(lk, facts, terms, specs, NGRP)
    gids = [G.star_slots(cols[1], R.eval_terms(cols, terms, cols[0].n), pk_to_slot) for cols in facts]
    ex = G.aggregate(_concat_inputs(facts, specs), [op for _, op in specs], np.concatenate(gids), NGRP)
    st.check(ex, True, what)
    check_out_slots(outs, gids, what)


def _grp_slot(g: R.Column, rows):
    return np.where(g.null_mask()[rows], NGRP - 1, g.values[rows] - GRP_MIN).astype(np.int32)


@pytest.mark.parametrize("dup", [None, "passing", "filtered"])
@pytest.mark.parametrize("n", [1, 33, 4097, 100_003])
def test_star_bitmap(n, dup):
    """b2_star_build_mark / rank / fill over two dim partitions, dir and slots word for word, then b2_star_agg"""
    import torch
    L = _L()
    rng = np.random.default_rng(n + 3 * (dup is not None))
    pk_min, nd = -77, 3000
    dims = [dim_part(nd, rng, pk_min, dup=dup), dim_part(nd, rng, pk_min + 2 * nd)]
    pk_range = 4 * nd
    nw = (pk_range + 31) // 32
    dirw = torch.zeros(nw, dtype=torch.int64, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    slots = _full(pk_range, 0x5A5A5A5A, dtype=torch.int32)
    scans = [scan_of(cols, DIM_PRED) for cols in dims]
    for s in scans:
        L.star_build_mark(C.byref(s), 1, pk_min, pk_range, _ptr(dirw), _ptr(flags), _stream())
    L.star_build_rank(_ptr(dirw), pk_range, _stream())
    for s in scans:
        L.star_build_fill(C.byref(s), 1, 2, pk_min, pk_range, GRP_MIN, NGRP - 1, _ptr(dirw), _ptr(slots), _stream())
    passing = [R.eval_terms(cols, DIM_PRED, nd) for cols in dims]
    exp_dir, exp_slots, exp_dup = G.star_build_bitmap(dims, passing, 1, 2, pk_min, pk_range, GRP_MIN, NGRP - 1)
    assert bool(_np(flags)[0]) == exp_dup == (dup == "passing"), _np(flags)
    if exp_dup:
        return                      # the caller falls back to the general join: only the flag is defined
    _eq(_np(dirw), exp_dir, "dir words")
    _eq(_np(slots, len(exp_slots)), exp_slots, "slots")
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range, lk.dir = 2, slots.data_ptr(), pk_min, pk_range, dirw.data_ptr()
    rows = [np.flatnonzero(ok) for ok in passing]
    m = {}
    for cols, r in zip(dims, rows):
        m.update(G.star_map(cols[1], r, _grp_slot(cols[2], r))[0])
    facts = [fact_part(n, rng, pk_min, pk_range) for _ in range(1 + n % 3)]
    check_star_agg(lk, facts, PRED, m, f"bitmap n={n}")
    check_star_agg(lk, facts, [], m, f"bitmap n={n} no predicate")


def _dim_selection(cols, rng):
    ok = R.eval_terms(cols, DIM_PRED, cols[0].n)
    sel = rng.permutation(np.flatnonzero(ok)).astype(np.int32)        # not the identity
    return sel, _grp_slot(cols[2], sel)


@pytest.mark.parametrize("dup", [None, "passing", "filtered"])
@pytest.mark.parametrize("n", [1, 4097, 100_003])
def test_star_dense_lookup(n, dup):
    """b2_star_build_dense over a shuffled selection (lookup word for word), then b2_star_agg"""
    import torch
    L = _L()
    rng = np.random.default_rng(50 + n)
    pk_min, nd = 1000, 5000
    dim = dim_part(nd, rng, pk_min, dup=dup)
    sel, sor = _dim_selection(dim, rng)
    rng_ = 2 * nd
    lookup = torch.full((rng_,), -1, dtype=torch.int32, device=_dev())
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    d, sel_t, sor_t = Dev(dim[1]), _t(sel), _t(sor)
    L.star_build_dense(C.byref(d.struct()), _ptr(sel_t), len(sel), _ptr(sor_t), pk_min, rng_, _ptr(lookup),
                       _ptr(flags), _stream())
    exp, exp_dup = G.star_build_dense(dim[1], sel, sor, pk_min, rng_)
    assert bool(_np(flags)[0]) == exp_dup == (dup == "passing")
    if exp_dup:
        return
    _eq(_np(lookup), exp, "lookup")
    lk = L.StarLookup()
    lk.dense, lk.lookup, lk.kmin, lk.range = 1, lookup.data_ptr(), pk_min, rng_
    facts = [fact_part(n, rng, pk_min, rng_) for _ in range(1 + n % 3)]
    check_star_agg(lk, facts, PRED, G.star_map(dim[1], sel, sor)[0], f"dense n={n}")


@pytest.mark.parametrize("case", [None, "passing", "filtered", "int64_min"])
@pytest.mark.parametrize("n", [1, 4097, 100_003])
def test_star_hash_lookup(n, case):
    """b2_star_build_hash: the table as a key -> slot map, d_flags[0] on a duplicate pk, d_flags[1] on an
    INT64_MIN pk (the empty-slot sentinel); then b2_star_agg, whose INT64_MIN fk never matches"""
    import torch
    L = _L()
    rng = np.random.default_rng(70 + n)
    pk_min, nd, cap = -2 ** 40, 3000, 8192
    dim = dim_part(nd, rng, pk_min, dup=None if case == "int64_min" else case)
    dim[1].values[7::7] += 2 ** 50         # sparse keys (rows 0 and 1 keep the duplicate cases' keys)
    if case == "int64_min":
        dim[1].values[5], dim[0].values[5], dim[1].null[5] = MIN, 0, False
    sel, sor = _dim_selection(dim, rng)
    tk = _full(cap, G.EMPTY_KEY)
    ts = _full(cap, 0x5A5A5A5A, dtype=torch.int32)
    flags = torch.zeros(4, dtype=torch.int32, device=_dev())
    d, sel_t, sor_t = Dev(dim[1]), _t(sel), _t(sor)
    L.star_build_hash(C.byref(d.struct()), _ptr(sel_t), len(sel), _ptr(sor_t), _ptr(tk), _ptr(ts), cap,
                      _ptr(flags), _stream())
    m, dup = G.star_map(dim[1], sel, sor)
    f = _np(flags)
    assert bool(f[0]) == dup == (case == "passing"), f
    assert bool(f[1]) == (case == "int64_min"), f
    if f[0] or f[1]:
        return
    tkh, tsh = _np(tk), _np(ts)
    got = {int(tkh[h]): int(tsh[h]) for h in range(cap) if tkh[h] != G.EMPTY_KEY}
    assert got == m, "hash table contents"
    lk = L.StarLookup()
    lk.dense, lk.table_keys, lk.table_slots, lk.cap = 0, tk.data_ptr(), ts.data_ptr(), cap
    facts = [fact_part(n, rng, pk_min, 2 * nd) for _ in range(1 + n % 3)]
    for cols in facts:                      # probe with keys that exist
        cols[1].values[::3] = rng.choice(dim[1].values, len(cols[1].values[::3]))
    check_star_agg(lk, facts, PRED, m, f"hash n={n}")


# ---- b2_join_agg ---------------------------------------------------------------------------------------------
JKMIN, JRANGE = 5000, 6000
U32_BASE = -2 ** 40


def build_side(rng):
    """key-ordered payloads over [JKMIN, JKMIN + JRANGE) with holes: I64 (huge), F64 (dyadic, NaN, NULL),
    U32 offsets from a base with values up to base + 2^32 - 1, U32 with the 0xFFFFFFFF sentinel, small I64"""
    present = rng.random(JRANGE) < 0.7
    bi = rng.choice(BIG_INTS, JRANGE)
    bf = rng.integers(-2 ** 12, 2 ** 12, JRANGE) * 2.0 ** -6
    bf[rng.random(JRANGE) < 0.03] = math.nan
    bf_null = rng.random(JRANGE) < 0.05
    off = rng.integers(0, 2 ** 32, JRANGE, dtype=np.uint64)
    off[:50] = 2 ** 32 - 1
    bs = rng.integers(0, 2 ** 32 - 1, JRANGE, dtype=np.uint64)
    bs[:50] = 2 ** 32 - 2
    bs[~present] = 2 ** 32 - 1
    bsmall = rng.integers(-2 ** 12, 2 ** 12, JRANGE).astype(np.int64)
    return {"present": present, "bi": R.Column(bi, None, R.I64), "bf": R.Column(bf, bf_null, R.F64),
            "bu": R.Column((U32_BASE + off.astype(np.int64)), None, R.I64), "bu_raw": off.astype(np.uint32),
            "bs": R.Column((U32_BASE + bs.astype(np.int64)), None, R.I64), "bs_raw": bs.astype(np.uint32),
            "bsmall": R.Column(bsmall, None, R.I64)}


def probe_part(n, rng):
    """0 p, 1 fk, 2 pi (huge, NULLs), 3 pf (dyadic, NaN), 4 psmall (no bitmap), 5 fk_nonnull"""
    fk = rng.integers(JKMIN - 10, JKMIN + JRANGE + 10, n).astype(np.int64)
    pf = rng.integers(-2 ** 12, 2 ** 12, n) * 2.0 ** -6
    pf[rng.random(n) < 0.03] = math.nan
    return [R.Column(rng.integers(-3, 10, n).astype(np.int64), None, R.I64),
            R.Column(fk, rng.random(n) < 0.03, R.I64),
            R.Column(rng.choice(BIG_INTS, n) if n else np.zeros(0, np.int64), rng.random(n) < 0.1, R.I64),
            R.Column(pf, None, R.F64), R.Column(rng.integers(-2 ** 12, 2 ** 12, n).astype(np.int64), None, R.I64),
            R.Column(fk.copy(), None, R.I64)]


# build columns as passed to the kernel: index -> (name, storage)
BUILD = [("bi", "i64"), ("bf", "f64"), ("bu", "u32"), ("bs", "sentinel")]


def run_join_agg(facts, terms, key_col, bs, build, aggs):
    import torch
    L = _L()
    present_words = torch.from_numpy(G.pack_bits(bs["present"]).view(np.int32)).to(_dev())
    keep, cols_arr = [], (L.Col * len(build))()
    base = (C.c_int64 * len(build))()
    for b, (name, kind) in enumerate(build):
        c = L.Col()
        if kind in ("u32", "sentinel"):
            t = _t(bs[name + "_raw"])
            c.dtype, base[b] = L.U32, U32_BASE
            c.flags = L.COL_SENTINEL if kind == "sentinel" else 0
        else:
            col = bs[name]
            t = _t(col.values)
            c.dtype = col.dtype
            if col.null is not None:
                v = _t(R.pack_valid(~col.null).view(np.int32))
                keep.append(v)
                c.valid = v.data_ptr()
        keep.append(t)
        c.data = t.data_ptr()
        cols_arr[b] = c
    jt = L.JoinTable()
    jt.nkeys, jt.dense, jt.lookup, jt.kmin, jt.range = 1, 2, present_words.data_ptr(), JKMIN, JRANGE
    ja = (L.JoinAgg * len(aggs))()
    for i, (pc, bc, comb, op) in enumerate(aggs):
        ja[i].pcol, ja[i].bcol, ja[i].combine, ja[i].op = pc, bc, comb, op
    acc = _full(len(aggs), 0x5A5A)
    cnt = _full(len(aggs), 0x5A5A)
    ws = torch.empty(L.scan_agg_ws_bytes(), dtype=torch.uint8, device=_dev())
    for i, cols in enumerate(facts):
        scan = scan_of(cols, terms)
        L.join_agg(C.byref(scan), key_col, C.byref(jt), len(build), cols_arr, base, ja, len(aggs), _ptr(acc), _ptr(cnt),
                   1 if i else 0, _ptr(ws), _stream())
    return _np(acc), _np(cnt)


def join_agg_expected(facts, terms, key_col, bs, build, aggs):
    inputs, gid_parts = [[] for _ in aggs], []
    for cols in facts:
        n = cols[0].n
        ok = R.eval_terms(cols, terms, n) & ~cols[key_col].null_mask()
        d = cols[key_col].values - JKMIN
        inr = ok & (d >= 0) & (d < JRANGE)
        dd = np.where(inr, d, 0)
        matched = inr & bs["present"][dd]
        gid_parts.append(np.where(matched, 0, -1))
        for a, (pc, bc, comb, op) in enumerate(aggs):
            if comb == G.JA_ROWS:
                inputs[a].append(None)
                continue
            pay = None
            if bc >= 0:
                src = bs[build[bc][0]]
                pay = R.Column(src.values[dd], src.null_mask()[dd] if src.null is not None else None, src.dtype)
            probe = cols[pc] if pc >= 0 else None
            inputs[a].append(G.join_agg_values(probe if comb != G.JA_B else None, pay if comb != G.JA_P else None,
                                               comb, matched))
    gid = np.concatenate(gid_parts)
    cat = []
    for a in range(len(aggs)):
        if inputs[a][0] is None:
            cat.append(None)
            continue
        cs = inputs[a]
        cat.append(R.Column(np.concatenate([c.values for c in cs]), np.concatenate([c.null_mask() for c in cs]),
                            cs[0].dtype))
    ops = [COUNT if comb == G.JA_ROWS else op for _, _, comb, op in aggs]
    ex = G.aggregate(cat, ops, gid, 1)
    return G.global_words(ex, ops, cat)


def check_global(got_acc, got_cnt, exp, dyadic, what):
    acc, cnt = exp
    _eq(got_cnt, np.array(cnt, np.int64), f"{what}: counts")
    for a, e in enumerate(acc):
        if isinstance(e, tuple):
            exact, bound, touched = e
            G.check_float_sum(got_acc[a:a + 1], np.array([exact]), np.array([bound]), np.array([touched]), 0,
                              dyadic, f"{what}: acc[{a}]")
        else:
            assert got_acc[a] == e, f"{what}: acc[{a}] = {got_acc[a]}, expected {e}"


def _ja_cases():
    """(name, probe key column, aggregates, float sums dyadic).  Only dyadic float x dyadic float (pf, bf) sums
    are exact whatever the order; sums over the huge ints and the U32 payloads (~2^40) are held to the bound."""
    C_ = [G.JA_MUL, G.JA_ADD, G.JA_SUB, G.JA_RSUB]
    cases = []
    # the fast kernel's shape: SUM / SUMF of P o B plus COUNT(*), nothing nullable by bitmap (so neither the
    # probe key 1 nor the payload bf, which have bitmaps)
    for comb in C_:
        for pc in (3, 4):
            for bc in (0, 2, 3):
                for op in (SUM, SUMF):
                    cases.append((f"fast p{pc} b{bc} c{comb} op{op}", 5,
                                  [(pc, bc, comb, op), (-1, -1, G.JA_ROWS, COUNT)], (pc, bc) == (3, 1)))
    # generic: every combine x every op, NULL and NaN on both sides, wrapping int x int
    ops = [SUM, SUMF, AMIN, AMAX, COUNT]
    for comb in [G.JA_P, G.JA_B] + C_:
        for pc, bc in [(2, 0), (3, 1), (2, 1), (4, 2), (2, 3)]:
            aggs = [(pc, bc, comb, op) for op in ops] + [(-1, -1, G.JA_ROWS, COUNT)]
            cases.append((f"generic p{pc} b{bc} c{comb}", 1, aggs, (pc, bc) == (3, 1)))
    return cases


@pytest.mark.parametrize("n", [0, 33, 4097, 100_003])
def test_join_agg(n):
    """P, B, P*B, P+B, P-B, B-P and COUNT(*) with SUM / SUMF / MIN / MAX / COUNT over I64, F64, U32 + base and
    sentinel U32 payloads, each through the fast kernel (where the shape allows it), the generic kernel and
    its 2-CTA instance; two partitions combined with accumulate = 1"""
    rng = np.random.default_rng(900 + n)
    bs = build_side(rng)
    facts = [probe_part(n, rng), probe_part(n // 2 + 1, rng)]
    modes = {"default": {}, "generic": {"B200SQL_JA_GENERIC": 1},
             "minb2": {"B200SQL_JA_GENERIC": 1, "B200SQL_JA_MINB": 2}}
    for name, key_col, aggs, dyadic in _ja_cases():
        for terms in ([], PRED):
            exp = join_agg_expected(facts, terms, key_col, bs, BUILD, aggs)
            for mode, sw in modes.items():
                with env(**sw):
                    got = run_join_agg(facts, terms, key_col, bs, BUILD, aggs)
                check_global(*got, exp, dyadic, f"{mode} {name} terms={terms}")


# ---- b2_scan_agg aggregates -------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 33, 4097, 8229, 100_003])
def test_scan_agg_sums(n):
    """SUMF over int64 beyond 2^53, float SUM on general data (bound), dyadic float SUM (bit-exact) and int SUM
    wrap, combined over three partitions with accumulate"""
    import torch
    L = _L()
    rng = np.random.default_rng(300 + n)
    parts = []
    for i in range(3):
        m = n + i
        big = rng.integers(-2 ** 62, 2 ** 62, m)
        gen = rng.normal(0, 1, m) * 10.0 ** rng.integers(-8, 9, m)
        dy = rng.integers(-2 ** 20, 2 ** 20, m) * 2.0 ** -10
        dy[rng.random(m) < 0.05] = -0.0
        gen[rng.random(m) < 0.05] = math.nan
        parts.append([R.Column(rng.integers(-3, 10, m).astype(np.int64), None, R.I64),
                      R.Column(big, rng.random(m) < 0.1, R.I64), R.Column(gen, rng.random(m) < 0.05, R.F64),
                      R.Column(dy, None, R.F64), R.Column(rng.choice(BIG_INTS, m) if m else np.zeros(0, np.int64), None, R.I64)])
    exact_specs = [(-1, COUNT), (3, SUM), (3, SUMF), (4, SUM), (3, AMIN), (3, AMAX), (1, COUNT)]
    bound_specs = [(1, SUMF), (2, SUM), (2, SUMF)]
    for specs, dyadic in ((exact_specs, True), (bound_specs, False)):
        for terms in ([], PRED):
            acc = _full(len(specs), 0x5A5A)
            cnt = _full(len(specs), 0x5A5A)
            ws = torch.empty(L.scan_agg_ws_bytes(), dtype=torch.uint8, device=_dev())
            gids = []
            for i, cols in enumerate(parts):
                scan = scan_of(cols, terms)
                L.scan_agg(C.byref(scan), _aggs(specs), len(specs), _ptr(acc), _ptr(cnt), 1 if i else 0, _ptr(ws), _stream())
                gids.append(np.where(R.eval_terms(cols, terms, cols[0].n), 0, -1))
            ins = _concat_inputs(parts, specs)
            ops = [op for _, op in specs]
            ex = G.aggregate(ins, ops, np.concatenate(gids), 1)
            check_global(_np(acc), _np(cnt), G.global_words(ex, ops, ins), dyadic, f"n={n} {specs} terms={terms}")
