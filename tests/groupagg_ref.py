"""Exact NumPy reference of the group-by and fused-aggregate kernels: the accumulator contract of
include/b200sql.h (b2_aggstate_t) for every word of acc[a], cnt[a], rows, present and out_slot, the slot
functions of the dense / hash1 / hashk / star / join_agg kernels, the global outputs of b2_scan_agg and
b2_join_agg, and the build outputs of b2_range_partition_* and b2_star_build_*.

Rules (the header's, restated):
  * SUM on int64 wraps; MIN / MAX compare int64 values, or for F64 the order-preserving image
    (rowwise_ref.ordered), so MIN{-0.0, +0.0} = -0.0 and MAX = +0.0;
  * NaN is NULL in every F64 input; COUNT counts the non-NULL inputs, COUNT(*) (rows) the rows;
  * a slot no row reaches, and an accumulator whose inputs in the slot are all NULL, keeps its initial word;
  * a touched float SUM is never -0.0: the kernels add x + 0.0 (or start from +0.0).
Float SUM / SUMF results depend on the summation order, so they are given as (exact, bound): `exact` is
math.fsum of the float64 summands the kernel adds (SUMF: float64(int) rounded to nearest) and, for any
order, |computed - exact| <= gamma_{m-1} * sum |x_i| with gamma_k = k u / (1 - k u), u = 2^-53 and m the
number of summands (adding +-0 is exact).  On dyadic data (small multiples of one power of two) every
partial sum is exact and the result is bit-identical whatever the order.
No GPU and no package import: only NumPy, and the opcode numbers of the header (repeated below)."""
import math
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from tests.rowwise_ref import F64, I64, INT64_MAX, INT64_MIN, U8, Column, ordered

AGG_SUM, AGG_SUMF, AGG_MIN, AGG_MAX, AGG_COUNT = range(5)
JA_P, JA_B, JA_MUL, JA_ADD, JA_SUB, JA_RSUB, JA_ROWS = range(7)
EMPTY_KEY = INT64_MIN
NEG_ZERO_BITS = INT64_MIN          # bit pattern of -0.0
U = 2.0 ** -53


def null_of(col: Column) -> np.ndarray:
    """NULL in the pandas sense: validity bit clear, or NaN in an F64 column"""
    nul = col.null_mask().copy()
    if col.dtype == F64:
        nul |= np.isnan(col.values)
    return nul


def is_float_sum(op, dtype):
    return op == AGG_SUMF or (op == AGG_SUM and dtype == F64)


# ---- exact float sums ------------------------------------------------------------------------------------
def gamma(m):
    k = max(m - 1, 0)
    return k * U / (1 - k * U)


def exact_sum(x) -> float:
    """the exactly rounded sum of float64 values; +-inf / NaN summands give the IEEE special value"""
    x = np.asarray(x, np.float64)
    if np.isnan(x).any() or (np.isposinf(x).any() and np.isneginf(x).any()):
        return math.nan
    if np.isposinf(x).any():
        return math.inf
    if np.isneginf(x).any():
        return -math.inf
    try:
        return math.fsum(x.tolist()) + 0.0      # + 0.0: an exact zero is +0.0, as the kernels produce
    except OverflowError:                       # the exact sum is beyond the float64 range
        return math.copysign(math.inf, float(np.sum(np.sign(x) * np.minimum(np.abs(x), 1e300))))


def sum_bound(x) -> float:
    """gamma_{m-1} * sum |x_i|, rounded up a little so that the bound itself is safe"""
    x = np.asarray(x, np.float64)
    if not len(x) or not np.isfinite(x).all():
        return 0.0
    try:
        return gamma(len(x)) * math.fsum(np.abs(x).tolist()) * (1 + 2.0 ** -50)
    except OverflowError:
        return math.inf


def check_float_sum(got_bits, exact, bound, touched, init_bits, dyadic, what=""):
    """got_bits: int64 words of a float SUM accumulator.  Touched slots: bit-exact on dyadic data (the sign
    of zero counts), else within `bound` of `exact` (specials must match, NaN any NaN); untouched slots
    keep `init_bits`."""
    got_bits = np.asarray(got_bits, np.int64)
    got = got_bits.view(np.float64)
    for i in np.flatnonzero(~touched):
        assert got_bits[i] == init_bits, f"{what}: untouched slot {i} holds {got[i]!r} ({got_bits[i]:#x})"
    for i in np.flatnonzero(touched):
        e, g = float(exact[i]), float(got[i])
        if math.isnan(e):
            ok = math.isnan(g)
        elif math.isinf(e) or dyadic:
            ok = got_bits[i] == np.float64(e).view(np.int64)
        else:
            ok = math.isfinite(g) and abs(g - e) <= bound[i]
        assert ok, f"{what}: slot {i} = {g!r}, exact {e!r}, bound {bound[i]!r}"


# ---- the accumulator contract ----------------------------------------------------------------------------
@dataclass
class Expected:
    """expected contents of a b2_aggstate_t over `nslots` slots.  acc[a]: int64 words (None for COUNT and
    for float SUMs, which are exact[a] / bound[a] / touched[a] instead)."""
    nslots: int
    acc: List[Optional[np.ndarray]] = field(default_factory=list)
    exact: List[Optional[np.ndarray]] = field(default_factory=list)
    bound: List[Optional[np.ndarray]] = field(default_factory=list)
    touched: List[Optional[np.ndarray]] = field(default_factory=list)
    cnt: List[np.ndarray] = field(default_factory=list)
    rows: Optional[np.ndarray] = None
    present: Optional[np.ndarray] = None      # bool per slot


def initial_word(op, dtype, indicator=False):
    """what the caller stores before the first call: SUM / COUNT 0 (-0.0 for an indicator SUM), MIN
    INT64_MAX, MAX INT64_MIN"""
    if op == AGG_MIN:
        return INT64_MAX
    if op == AGG_MAX:
        return INT64_MIN
    return NEG_ZERO_BITS if indicator else 0


def aggregate(inputs, ops, gid, nslots, indicator=None) -> Expected:
    """inputs[a]: the Column aggregate a reads (None = COUNT(*)), ops[a]: AGG_*, gid: int64 per row, the slot
    the row lands in (-1 = it does not contribute).  indicator: index of a float SUM that starts at -0.0."""
    gid = np.asarray(gid, np.int64)
    live = gid >= 0
    ex = Expected(nslots)
    ex.rows = np.bincount(gid[live], minlength=nslots).astype(np.int64)
    ex.present = ex.rows > 0
    for a, (col, op) in enumerate(zip(inputs, ops)):
        ex.acc.append(None), ex.exact.append(None), ex.bound.append(None), ex.touched.append(None)
        if col is None:
            ex.cnt.append(ex.rows.copy())
            continue
        ok = live & ~null_of(col)
        g = gid[ok]
        ex.cnt.append(np.bincount(g, minlength=nslots).astype(np.int64))
        init = initial_word(op, col.dtype, indicator == a)
        if op == AGG_COUNT:
            continue
        if is_float_sum(op, col.dtype):
            x = col.values[ok].astype(np.float64) if col.dtype != F64 else col.values[ok]
            exact = np.zeros(nslots)
            bound = np.zeros(nslots)
            order = np.argsort(g, kind="stable")
            gs, xs = g[order], x[order]
            starts = np.flatnonzero(np.r_[True, gs[1:] != gs[:-1]]) if len(gs) else np.zeros(0, np.int64)
            ends = np.r_[starts[1:], len(gs)]
            for s, e in zip(starts, ends):
                exact[gs[s]] = exact_sum(xs[s:e])
                bound[gs[s]] = sum_bound(xs[s:e])
            ex.exact[a], ex.bound[a] = exact, bound
            ex.touched[a] = np.bincount(g, minlength=nslots) > 0
            continue
        words = np.full(nslots, init, np.int64)
        v = col.raw()[ok]
        if op == AGG_SUM:
            u = words.view(np.uint64)
            np.add.at(u, g, v.view(np.uint64))
        else:
            img = ordered(v) if col.dtype == F64 else v
            (np.minimum if op == AGG_MIN else np.maximum).at(words, g, img)
        ex.acc[a] = words
    return ex


def pack_bits(flags: np.ndarray) -> np.ndarray:
    """bool per slot -> uint32 words, LSB first"""
    n = len(flags)
    out = np.zeros(((n + 31) // 32) * 4, np.uint8)
    b = np.packbits(flags.astype(bool), bitorder="little")
    out[: len(b)] = b
    return out.view(np.uint32)


def permute(ex: Expected, slot_of_group, nslots, indicator=None, inputs=None, ops=None) -> Expected:
    """the same groups at other slot numbers (hash tables): group k of `ex` goes to slot slot_of_group[k];
    every other slot is untouched"""
    out = Expected(nslots)
    idx = np.asarray(slot_of_group, np.int64)

    def move(arr, fill, dtype):
        if arr is None:
            return None
        r = np.full(nslots, fill, dtype)
        r[idx] = arr
        return r

    out.rows = move(ex.rows, 0, np.int64)
    out.present = move(ex.present, False, bool)
    for a in range(len(ex.cnt)):
        op = ops[a] if ops else AGG_SUM
        dt = inputs[a].dtype if inputs and inputs[a] is not None else I64
        out.acc.append(move(ex.acc[a], initial_word(op, dt, indicator == a), np.int64))
        out.exact.append(move(ex.exact[a], 0.0, np.float64))
        out.bound.append(move(ex.bound[a], 0.0, np.float64))
        out.touched.append(move(ex.touched[a], False, bool))
        out.cnt.append(move(ex.cnt[a], 0, np.int64))
    return out


# ---- slot functions --------------------------------------------------------------------------------------
def dense_slots(key: Column, passing, kmin, nslots):
    """b2_groupby_dense: key - kmin (uint64 arithmetic), NULL key -> nslots - 1, out of range -> -1"""
    d = key.raw().view(np.uint64) - np.uint64(kmin & 0xFFFFFFFFFFFFFFFF)
    inr = d < np.uint64(nslots - 1)
    slot = np.where(inr, d.view(np.int64), -1)
    slot = np.where(key.null_mask(), nslots - 1, slot)
    return np.where(passing, slot, -1).astype(np.int64)


NULL_GROUP, EMPTY_GROUP = ("null",), ("empty",)


def hash1_identity(key: Column):
    """the group each row's key names in b2_groupby_hash1: NULL / NaN -> NULL_GROUP, the INT64_MIN bit
    pattern -> EMPTY_GROUP, otherwise the int64 key (F64: its bits, -0.0 as +0.0)"""
    raw = key.raw().copy()
    if key.dtype == F64:
        raw[raw == NEG_ZERO_BITS] = 0
    nul = null_of(key)
    return [NULL_GROUP if nul[i] else (EMPTY_GROUP if raw[i] == EMPTY_KEY else int(raw[i])) for i in range(key.n)]


def hashk_identity(keys: List[Column]):
    """b2_groupby_hashk: (normalised key bits with NULL -> 0 ..., null mask) per row"""
    n = keys[0].n
    parts, mask = [], np.zeros(n, np.int64)
    for k, c in enumerate(keys):
        raw = c.raw().copy()
        if c.dtype == F64:
            raw[raw == NEG_ZERO_BITS] = 0
        nul = null_of(c)
        raw[nul] = 0
        mask |= nul.astype(np.int64) << k
        parts.append(raw)
    return [tuple(int(p[i]) for p in parts) + (int(mask[i]),) for i in range(n)]


def codes(identity, passing):
    """group codes 0..G-1 of the passing rows (-1 elsewhere) and the group identities in code order"""
    groups, gid = {}, np.full(len(identity), -1, np.int64)
    for i in np.flatnonzero(passing):
        gid[i] = groups.setdefault(identity[i], len(groups))
    return gid, list(groups)


# ---- star join ---------------------------------------------------------------------------------------------
def star_map(pk: Column, rows, slot_of_row):
    """pk -> group slot over build rows `rows` (NULL pk never joins); also whether a pk repeats"""
    m, dup = {}, False
    nul = pk.null_mask()
    for r, s in zip(rows, slot_of_row):
        if nul[r]:
            continue
        k = int(pk.values[r])
        dup |= k in m
        m[k] = int(s)
    return m, dup


def star_build_dense(pk: Column, sel, slot_of_row, kmin, rng):
    """b2_star_build_dense: (lookup int32[range], duplicate flag); valid only without duplicates"""
    lk = np.full(rng, -1, np.int32)
    seen, dup = set(), False
    for r, s in zip(sel, slot_of_row):
        if pk.null_mask()[r]:
            continue
        d = (int(pk.values[r]) - kmin) & 0xFFFFFFFFFFFFFFFF      # uint64 offset: keys below kmin are out too
        if d < rng:
            dup |= d in seen
            seen.add(d)
            lk[d] = s
    return lk, dup


def star_build_bitmap(parts, passing, pk_col, grp_col, pk_min, pk_range, grp_min, null_slot):
    """b2_star_build_mark / rank / fill over all partitions: (dir uint64 words, slots int32, duplicate flag)"""
    keys, grps = [], []
    for cols, ok in zip(parts, passing):
        pk, gc = cols[pk_col], cols[grp_col]
        d = pk.raw().view(np.uint64) - np.uint64(pk_min & 0xFFFFFFFFFFFFFFFF)
        take = ok & ~pk.null_mask() & (d < np.uint64(pk_range))
        keys.append(d[take].astype(np.int64))
        g = np.where(gc.null_mask(), null_slot, gc.raw() - grp_min)
        grps.append(g[take])
    keys, grps = np.concatenate(keys), np.concatenate(grps)
    dup = len(np.unique(keys)) < len(keys)
    nw = (pk_range + 31) // 32
    bits = np.zeros(nw * 32, bool)
    bits[keys] = True
    words = pack_bits(bits[:nw * 32]).astype(np.uint64)[:nw]
    pop = np.array([bin(int(w)).count("1") for w in words], np.uint64)
    rank = np.concatenate([[0], np.cumsum(pop)[:-1]]).astype(np.uint64) if nw else pop
    dirw = (words | (rank << np.uint64(32))).view(np.int64)
    order = np.argsort(keys, kind="stable")
    return dirw, grps[order].astype(np.int32), dup


def star_slots(fk: Column, passing, pk_to_slot):
    """b2_star_agg: slot of each probe row (-1: filtered, NULL fk, or no build partner)"""
    nul = fk.null_mask()
    return np.array([pk_to_slot.get(int(fk.values[i]), -1) if passing[i] and not nul[i] else -1
                     for i in range(fk.n)], np.int64)


# ---- b2_join_agg ----------------------------------------------------------------------------------------------
def join_agg_values(probe: Optional[Column], pay: Optional[Column], combine, matched):
    """the per-row value of one join aggregate as a Column: float64 as soon as one side is F64 (the int side
    converted first, the combination rounded once), else wrapping int64.  Rows that are not matched, or
    where an input is NULL / NaN, are NULL."""
    nul = ~matched
    if probe is not None:
        nul = nul | null_of(probe)
    if pay is not None:
        nul = nul | null_of(pay)
    if combine == JA_P:
        return Column(probe.values.copy(), nul, probe.dtype)
    if combine == JA_B:
        return Column(pay.values.copy(), nul, pay.dtype)
    if F64 in (probe.dtype, pay.dtype):
        u, w = probe.values.astype(np.float64), pay.values.astype(np.float64)
        with np.errstate(all="ignore"):
            r = {JA_MUL: u * w, JA_ADD: u + w, JA_SUB: u - w, JA_RSUB: w - u}[combine]
        return Column(r, nul, F64)
    u, w = probe.raw().view(np.uint64), pay.raw().view(np.uint64)
    r = {JA_MUL: u * w, JA_ADD: u + w, JA_SUB: u - w, JA_RSUB: w - u}[combine]
    return Column(r.view(np.int64), nul, I64)


def global_words(ex: Expected, ops, inputs):
    """b2_scan_agg / b2_join_agg outputs from a one-slot Expected: (acc words with float SUMs as (exact,
    bound), counts).  An output with no row is the identity: 0 (+0.0), INT64_MAX, INT64_MIN; COUNT's acc is 0."""
    acc = []
    for a, op in enumerate(ops):
        if ex.exact[a] is not None:
            acc.append((float(ex.exact[a][0]), float(ex.bound[a][0]), bool(ex.touched[a][0])))
        elif ex.acc[a] is not None:
            acc.append(int(ex.acc[a][0]))
        else:
            acc.append(0)
    return acc, [int(c[0]) for c in ex.cnt]


# ---- b2_range_partition -------------------------------------------------------------------------------------
def range_partition(parts, passing, key_col, kmin, nslots, shift, nbuckets, carry):
    """bucket starts (int64[nbuckets + 1], the last = rows written) and, per bucket, the sorted multiset of
    (kmin + slot, carried values...) rows of every partition that pass (NULL key -> slot nslots - 1)"""
    rows = []
    for cols, ok in zip(parts, passing):
        slot = dense_slots(cols[key_col], ok, kmin, nslots)
        keep = slot >= 0
        vals = [slot[keep]] + [cols[c].raw()[keep] for c in carry]
        rows.append(np.stack(vals, axis=1) if len(vals) else np.zeros((0, 1), np.int64))
    allr = np.concatenate(rows) if rows else np.zeros((0, 1 + len(carry)), np.int64)
    bucket = allr[:, 0] >> shift
    hist = np.bincount(bucket, minlength=nbuckets).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(hist)]).astype(np.int64)
    allr = allr.copy()
    allr[:, 0] = allr[:, 0] + kmin
    per_bucket = []
    for b in range(nbuckets):
        sel = allr[bucket == b]
        per_bucket.append(sel[np.lexsort(sel.T[::-1])] if len(sel) else sel)
    return starts, per_bucket
