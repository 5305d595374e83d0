"""Exact NumPy reference of the join kernels: the chained build (b2_join_build, checked through the invariants
of its chains, not through the hash), the direct-address build (b2_join_build_dense), the key-ordered layout
(b2_join_key_layout) and the rows, tile offsets, gathered columns, validity words and build_matched flags of
the probes (b2_join_count + b2_join_write*, b2_join_onepass).

Rules (the header's, restated):
  * a key is NULL when its validity bit is clear or, in an F64 key, when it is NaN; a row with any NULL key
    never matches;
  * -0.0 and +0.0 are the same key; otherwise two keys are equal when their bit patterns are (NaN payloads do
    not matter: NaN is NULL); multi-key rows match when every key does;
  * every passing probe row emits, in probe-row order: INNER one row per matching build row, as a contiguous
    run whose order is unspecified (chains are built with atomicExch), so runs are compared as sets; LEFT the
    same, or one row with build index -1 when nothing matches; SEMI one row, build index -1, if anything
    matches; ANTI one row, build index -1, if nothing does;
  * a direct-address table holds keys [kmin, kmin + range): offsets are uint64 `key - kmin` (wrapping), keys
    outside are skipped; on a key-ordered table (dense == 2) the build index of a match is the offset;
  * a gathered probe column is a bit copy, valid iff its source is; a gathered build column at build index -1
    holds NaN bits 0x7ff8000000000000 (F64) or 0 (I64 / U8 / U32) and is NULL; a B2_U32 column decodes as
    base + uint32;
  * tile_off is the exclusive scan of the rows each 4096-row probe tile emits, the total last.
No GPU and no package import: only NumPy, and the numbers of include/b200sql.h (repeated below)."""
from dataclasses import dataclass

import numpy as np

from tests.rowwise_ref import F64, I64, INT64_MIN, U8, Column, pack_valid

U32 = 3
COL_SENTINEL = 1
JOIN_INNER, JOIN_LEFT, JOIN_SEMI, JOIN_ANTI = range(4)
MODES = (JOIN_INNER, JOIN_LEFT, JOIN_SEMI, JOIN_ANTI)
TILE = 4096
NAN_FILL = 0x7FF8000000000000
NEG_ZERO_BITS = INT64_MIN


# ---- keys --------------------------------------------------------------------------------------------------
def key_null(col: Column) -> np.ndarray:
    nul = col.null_mask().copy()
    if col.dtype == F64:
        nul |= np.isnan(col.values)
    return nul


def key_image(col: Column) -> np.ndarray:
    """the 64-bit word a key compares by: its bits, -0.0 folded onto +0.0"""
    raw = col.raw().copy()
    if col.dtype == F64:
        raw[raw == NEG_ZERO_BITS] = 0
    return raw


def key_rows(cols):
    """([n, k] key images, [n] any-key-NULL)"""
    img = np.stack([key_image(c) for c in cols], axis=1)
    nul = np.zeros(cols[0].n, bool)
    for c in cols:
        nul |= key_null(c)
    return img, nul


# ---- matches as CSR: probe row i matches build rows rows[ptr[i]:ptr[i + 1]] (ascending) ---------------------
@dataclass
class Matches:
    ptr: np.ndarray    # int64[n + 1]
    rows: np.ndarray   # int64[ptr[-1]]

    @property
    def counts(self):
        return np.diff(self.ptr)


def _csr(counts, start_of_row, sorted_rows):
    ptr = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(counts, out=ptr[1:])
    total = int(ptr[-1])
    flat = np.repeat(start_of_row - ptr[:-1], counts) + np.arange(total, dtype=np.int64)
    return Matches(ptr, sorted_rows[flat] if total else np.zeros(0, np.int64))


def hash_matches(probe_keys, build_keys, passing) -> Matches:
    """matches of a chained table: equal key images, no NULL on either side, passing probe rows only"""
    pimg, pnul = key_rows(probe_keys)
    bimg, bnul = key_rows(build_keys)
    brows = np.flatnonzero(~bnul)
    allimg = np.concatenate([bimg[brows], pimg])
    if allimg.shape[1] == 1:
        allimg = allimg[:, 0]          # one key: the 1-d unique is much faster than the row-wise one
    _, inv = np.unique(allimg, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    bg, pg = inv[: len(brows)], inv[len(brows):]
    ngroups = int(inv.max()) + 1 if len(inv) else 0
    order = np.argsort(bg, kind="stable")
    sorted_rows = brows[order].astype(np.int64)
    gcount = np.bincount(bg, minlength=ngroups).astype(np.int64)
    gstart = np.zeros(ngroups + 1, np.int64)
    np.cumsum(gcount, out=gstart[1:])
    live = passing & ~pnul
    counts = np.where(live, gcount[pg] if len(pg) else 0, 0).astype(np.int64)
    return _csr(counts, gstart[pg] if len(pg) else np.zeros(0, np.int64), sorted_rows)


def offsets(key: Column, kmin, rng):
    """(uint64 key - kmin with wrap, in range and not NULL)"""
    d = key.values.astype(np.int64).view(np.uint64) - np.uint64(kmin & ((1 << 64) - 1))
    return d, (d < np.uint64(rng)) & ~key_null(key)


def dense_matches(probe_key: Column, kmin, rng, table, dense, passing) -> Matches:
    """matches of a direct-address table: `table` is the int32 lookup (dense == 1) or the bool presence of
    every offset (dense == 2, build index = offset)"""
    d, ok = offsets(probe_key, kmin, rng)
    ok &= passing
    dd = np.where(ok, d, 0).astype(np.int64)
    if dense == 1:
        b = np.where(ok, table[dd] if len(table) else -1, -1).astype(np.int64)
    else:
        b = np.where(ok & (table[dd] if len(table) else False), dd, -1)
    hit = b >= 0
    return Matches(np.concatenate([[0], np.cumsum(hit)]).astype(np.int64), b[hit])


# ---- emitted rows ------------------------------------------------------------------------------------------
@dataclass
class Emitted:
    probe: np.ndarray   # int64[total]: probe row of every output row, in order
    build: np.ndarray   # int64[total]: build index (-1 = none), ascending inside each probe row's run
    count: np.ndarray   # int64[n]: rows each probe row emits

    @property
    def total(self):
        return len(self.probe)


def emit(mode, passing, m: Matches) -> Emitted:
    cnt = m.counts
    if mode == JOIN_INNER:
        per = cnt
    elif mode == JOIN_LEFT:
        per = np.where(passing, np.maximum(cnt, 1), 0)
    elif mode == JOIN_SEMI:
        per = (passing & (cnt > 0)).astype(np.int64)
    else:
        per = (passing & (cnt == 0)).astype(np.int64)
    per = per.astype(np.int64)
    probe = np.repeat(np.arange(len(per), dtype=np.int64), per)
    if mode in (JOIN_SEMI, JOIN_ANTI):
        build = np.full(len(probe), -1, np.int64)
    elif mode == JOIN_INNER:
        build = m.rows.copy()
    else:
        # LEFT: the matches, with one -1 slotted in for every passing row that has none
        ptr = np.zeros(len(per) + 1, np.int64)
        np.cumsum(per, out=ptr[1:])
        build = np.full(int(ptr[-1]), -1, np.int64)
        pos = np.repeat(ptr[:-1], cnt) + (np.arange(len(m.rows)) - np.repeat(m.ptr[:-1], cnt))
        build[pos] = m.rows
    return Emitted(probe, build, per)


def sort_runs(probe, build):
    """build indices sorted inside each run of equal probe rows (probe rows must be non-decreasing)"""
    probe, build = np.asarray(probe, np.int64), np.asarray(build, np.int64)
    return build[np.lexsort((build, probe))]


def tile_off(count, n, tile=TILE):
    """int64[ntiles + 1]: exclusive scan of the rows each tile emits, the total last"""
    ntiles = (n + tile - 1) // tile
    per = np.zeros(ntiles * tile, np.int64)
    per[:n] = count
    out = np.zeros(ntiles + 1, np.int64)
    np.cumsum(per.reshape(ntiles, tile).sum(axis=1), out=out[1:])
    return out


def build_matched(mode, e: Emitted, nbuild):
    """uint8[nbuild]: 1 for every build row some output row pairs with (INNER / LEFT)"""
    out = np.zeros(nbuild, np.uint8)
    if mode in (JOIN_INNER, JOIN_LEFT):
        out[e.build[e.build >= 0]] = 1
    return out


# ---- gathered columns --------------------------------------------------------------------------------------
def gather_probe(col: Column, prows):
    """(values as stored: int64 words or uint8, valid bool)"""
    prows = np.asarray(prows, np.int64)
    vals = col.values[prows] if col.dtype == U8 else col.raw()[prows]
    return vals, ~col.null_mask()[prows]


def gather_build(col: Column, brows, base=0):
    """(values as the output holds them: int64 words or uint8, valid bool).  `col` may be a B2_U32 storage
    column (uint32 values), decoded as base + uint32; index -1 gives the NULL fill."""
    brows = np.asarray(brows, np.int64)
    miss = brows < 0
    safe = np.where(miss, 0, brows)
    if col.dtype == U8:
        vals = np.where(miss, 0, col.values[safe] if len(col.values) else 0).astype(np.uint8)
    else:
        if col.dtype == U32:
            src = (np.int64(base) + col.values.astype(np.int64)) if len(col.values) else np.zeros(0, np.int64)
        else:
            src = col.raw()
        fill = NAN_FILL if col.dtype == F64 else 0
        vals = np.where(miss, np.int64(fill), src[safe] if len(src) else 0).astype(np.int64)
    valid = ~miss & (~col.null_mask()[safe] if len(col.values) else False)
    return vals, valid


def valid_words(valid, nwords):
    """validity words of an output holding nwords words: bits of `valid`, everything after it zero"""
    w = np.zeros(nwords, np.uint32)
    p = pack_valid(np.asarray(valid, bool))
    w[: len(p)] = p
    return w


# ---- builds ------------------------------------------------------------------------------------------------
def dense_build(key: Column, kmin, rng):
    """b2_join_build_dense: (int32 lookup with -1 at duplicate offsets too, duplicate flag, {offset: rows} of
    the duplicated offsets).  At a duplicated offset the kernel keeps one of the rows, whichever came last."""
    d, ok = offsets(key, kmin, rng)
    rows = np.flatnonzero(ok)
    dd = d[rows].astype(np.int64)
    lookup = np.full(rng, -1, np.int32)
    cnt = np.bincount(dd, minlength=rng) if len(dd) else np.zeros(rng, np.int64)
    uniq = cnt[dd] == 1 if len(dd) else np.zeros(0, bool)
    lookup[dd[uniq]] = rows[uniq]
    dups = {}
    for r, o in zip(rows[~uniq], dd[~uniq]):
        dups.setdefault(int(o), []).append(int(r))
    return lookup, int(bool(dups)), dups


def key_layout(key: Column, kmin, rng, col, out_dtype, base, out_init, valid_init, present_init):
    """b2_join_key_layout over unique keys: (out, out_valid words, present words) from the initial buffers.
    `col` None: only `present`.  Offsets without a build row keep their initial words."""
    d, ok = offsets(key, kmin, rng)
    rows = np.flatnonzero(ok)
    dd = d[rows].astype(np.int64)
    present = None if present_init is None else present_init.copy()
    if present is not None:
        bits = np.unpackbits(present.view(np.uint8), bitorder="little")
        bits[dd] = 1
        present = np.packbits(bits, bitorder="little").view(np.uint32)
    out = None if out_init is None else out_init.copy()
    valid = None if valid_init is None else valid_init.copy()
    if col is not None:
        if col.dtype == U8:
            out[dd] = col.values[rows]
        elif out_dtype == U32:
            out[dd] = (col.values[rows].view(np.uint64) - np.uint64(base & ((1 << 64) - 1))).astype(np.uint32)
        else:
            out[dd] = col.raw()[rows]
        if valid is not None:
            bits = np.unpackbits(valid.view(np.uint8), bitorder="little")
            bits[dd[~col.null_mask()[rows]]] = 1
            valid = np.packbits(bits, bitorder="little").view(np.uint32)
    return out, valid, present


def check_chains(head, nxt, build_keys):
    """the invariants of a chained table whatever the hash: every non-NULL row is on exactly one chain, NULL
    rows have next = -1 and are on none, chains end, and rows with equal key images share one bucket.
    Returns an error message or None."""
    head, nxt = np.asarray(head, np.int64), np.asarray(nxt, np.int64)
    img, nul = key_rows(build_keys)
    n, cap = len(nul), len(head)
    if len(nxt) < n:
        return f"next has {len(nxt)} entries for {n} rows"
    nxt = nxt[:n]
    if ((head < -1) | (head >= n)).any() or ((nxt < -1) | (nxt >= n)).any():
        return "a link points outside [-1, n)"
    if (nxt[nul] != -1).any():
        return f"NULL row {int(np.flatnonzero(nul & (nxt != -1))[0])} has next != -1"
    indeg = np.bincount(np.concatenate([head[head >= 0], nxt[nxt >= 0]]), minlength=n)[:n]
    if (indeg[nul] != 0).any():
        return f"NULL row {int(np.flatnonzero(nul & (indeg != 0))[0])} is on a chain"
    if (indeg[~nul] != 1).any():
        r = int(np.flatnonzero(~nul & (indeg != 1))[0])
        return f"row {r} is linked {int(indeg[r])} times"
    # walk every chain at once; in-degree 1 everywhere means a cycle would be unreachable from the heads
    bucket = np.full(n, -1, np.int64)
    cur_b = np.flatnonzero(head >= 0)
    cur = head[cur_b]
    steps = 0
    while len(cur):
        bucket[cur] = cur_b
        steps += 1
        if steps > n:
            return "a chain does not end"
        nx = nxt[cur]
        keep = nx >= 0
        cur, cur_b = nx[keep], cur_b[keep]
    if (bucket[~nul] < 0).any():
        return f"row {int(np.flatnonzero(~nul & (bucket < 0))[0])} is on no chain (a cycle)"
    rows = np.flatnonzero(~nul)
    if len(rows):
        _, g = np.unique(img[rows], axis=0, return_inverse=True)
        g = g.reshape(-1)
        lo = np.full(g.max() + 1, cap, np.int64)
        hi = np.full(g.max() + 1, -1, np.int64)
        np.minimum.at(lo, g, bucket[rows])
        np.maximum.at(hi, g, bucket[rows])
        if (lo != hi).any():
            return f"equal keys sit in different buckets (key group {int(np.flatnonzero(lo != hi)[0])})"
    return None
