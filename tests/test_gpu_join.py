"""The join kernels row for row against the NumPy reference of tests/join_ref.py, through the C-ABI:
b2_join_build (chain invariants), b2_join_build_dense, b2_join_key_layout, the two-pass probe b2_join_count +
b2_join_write / _write_gather / _write_gather_keyed over chained, direct-address and key-ordered tables, and
b2_join_onepass in its counted, look-back and streaming forms -- every instance of the specialised streaming
kernel under both B200SQL_JOIN_RESERVE settings, and every shape that falls back to the generic kernel.

Probe indices, tile offsets, gathered words and validity words are compared exactly; the build rows of one
probe row form a run whose order is unspecified (chains are built with atomicExch), so runs are compared as
sets and every gathered build value against the build index emitted beside it.  Outputs start as garbage:
rows past the emitted count must keep it and validity words past it must stay zero.  Row counts straddle the
warp (32), the warp batch (256), the one-pass tile (2048) and the two-pass tile (4096), and one run per probe
kernel is large enough (2112 x 4096 + 1 rows) for every grid-stride tile loop to wrap.

Argument errors are checked through the raw library symbols, with every buffer sized for what an unchecked
launch would touch, so that no version of the library can read or write out of bounds here."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import join_ref as J
from tests import rowwise_ref as R
from tests.test_gpu_groupagg import env, scan_of
from tests.test_gpu_rowwise import Dev, _assert_words, _dev, _L, _ptr, _stream

pytestmark = pytest.mark.gpu

MIN, MAX = R.INT64_MIN, R.INT64_MAX
SIZES = [0, 1, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 100_003]
BIG_N = 2112 * 4096 + 1        # > 2 waves of 132 SMs x 8 blocks even for 4096-row tiles
SLACK = 67                     # garbage rows after the largest possible output
GARBAGE = 0x5A5A5A5A5A5A5A5A
NAN_PAYLOADS = np.array([0x7FF8000000000000, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF, -0x0008000000000000,
                         -0x000FFFFFFFFFFFFF], np.int64).view(np.float64)
FLOAT_KEYS = np.concatenate([[0.0, -0.0, math.inf, -math.inf, 1.5, -2.25, 5e-324], NAN_PAYLOADS])
INT_KEYS = np.array([MIN, MAX, MIN + 1, MAX - 1, 0, -1], np.int64)
MODES = J.MODES
HOT = 5000                     # build rows sharing one key: probe rows with it take the re-walk path


# ---- plumbing ------------------------------------------------------------------------------------------------
def _t(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).to(_dev())


def _np(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _garbage(rows, u8=False):
    import torch
    if u8:
        return torch.full((rows,), 0x5A, dtype=torch.uint8, device=_dev())
    return torch.full((rows,), GARBAGE, dtype=torch.int64, device=_dev())


def _zeros(n, dtype=None):
    import torch
    return torch.zeros(max(n, 1), dtype=dtype or torch.int32, device=_dev())


def _words(rows):
    return (rows + 31) // 32


def col_struct(col: R.Column, keep, flags=0):
    """a b2_col_t over a device copy of `col` (B2_U32 storage columns hold uint32 values); the copy goes to `keep`"""
    d = Dev(R.Column(col.values.view(np.int32), col.null, J.U32) if col.dtype == J.U32 else col)
    keep.append(d)
    c = d.struct()
    c.flags = flags
    return c


def col_array(cols, keep, flags=None):
    L = _L()
    arr = (L.Col * max(1, len(cols)))()
    for i, c in enumerate(cols):
        arr[i] = col_struct(c, keep, flags[i] if flags else 0)
    return arr


def _ptrs(ts):
    return (C.c_void_p * max(1, len(ts)))(*[(t.data_ptr() if t is not None else 0) for t in ts])


class Gathered:
    """output buffers of gathered columns: garbage values over `rows` + SLACK rows, zeroed validity words
    (one more word than needed) or None"""

    def __init__(self, dtypes, rows, with_valid):
        self.dtypes, self.rows = dtypes, rows
        self.data = [_garbage(rows + SLACK, u8=dt == R.U8) for dt in dtypes]
        self.valid = [_zeros(_words(rows) + 1) if with_valid else None for _ in dtypes]
        self.out, self.vout = _ptrs(self.data), _ptrs(self.valid)

    def vptr(self):
        return self.vout if any(v is not None for v in self.valid) else None

    def check(self, k, total, exp_vals, exp_valid, what):
        got = _np(self.data[k])
        u8 = self.dtypes[k] == R.U8
        _assert_words(got[:total], np.asarray(exp_vals, got.dtype), f"{what}: column {k} values")
        tail = np.full(len(got) - total, 0x5A if u8 else GARBAGE, got.dtype)
        _assert_words(got[total:], tail, f"{what}: column {k} rows past the {total} emitted")
        if self.valid[k] is not None:
            w = _np(self.valid[k]).view(np.uint32)
            _assert_words(w, J.valid_words(exp_valid, len(w)), f"{what}: column {k} validity words")


def _out_dtype(col: R.Column):
    return R.U8 if col.dtype == R.U8 else R.I64


# ---- data ----------------------------------------------------------------------------------------------------
# probe columns: 0 pid (row id), 1 p (small int: predicate), 2 k0 (int key, NULLs), 3 k1 (float key: NaN of several
# payloads, ±0.0, ±inf, NULLs), 4 pf (float: NaN, -0.0, NULLs), 5 pu (bool byte, NULLs), 6 kn (int key, no bitmap)
PID, P, K0, K1, PF, PU, KN = range(7)
T_NONE = []
T_OTHER = [(P, R.GE, 0, 0, 0.0)]
T_F64 = [(PF, R.GE, 0, 0, -8.0)]


def t_key(kmid):
    return [(K0, R.LT, 0, kmid, 0.0)]


def probe_cols(n, rng, ikeys, fkeys=None):
    """ikeys: int64 key values (K0 gets a NULL bitmap, KN the same values without one)"""
    pf = rng.integers(-64, 64, n) * 0.25
    pf[rng.random(n) < 0.05] = -0.0
    pf[rng.random(n) < 0.05] = math.nan
    if fkeys is None:
        fkeys = rng.choice(FLOAT_KEYS, n) if n else np.zeros(0)
    return [R.Column(np.arange(n, dtype=np.int64), None, R.I64),
            R.Column(rng.integers(-3, 10, n).astype(np.int64), None, R.I64),
            R.Column(ikeys.copy(), rng.random(n) < 0.05, R.I64),
            R.Column(fkeys, rng.random(n) < 0.04, R.F64),
            R.Column(pf, rng.random(n) < 0.1, R.F64),
            R.Column(rng.integers(0, 256, n).astype(np.uint8), rng.random(n) < 0.1, R.U8),
            R.Column(ikeys.copy(), None, R.I64)]


def build_payload(nb, rng):
    """build columns: 0 bid (row id + 1, no bitmap), 1 bf (float: NaN, -0.0, NULLs), 2 bu (byte, NULLs),
    3 bi (int64 edges, NULLs)"""
    bf = rng.integers(-64, 64, nb) * 0.5
    bf[rng.random(nb) < 0.05] = -0.0
    bf[rng.random(nb) < 0.05] = math.nan
    return [R.Column(np.arange(1, nb + 1, dtype=np.int64), None, R.I64),
            R.Column(bf, rng.random(nb) < 0.1, R.F64),
            R.Column(rng.integers(0, 256, nb).astype(np.uint8), rng.random(nb) < 0.1, R.U8),
            R.Column(rng.choice(INT_KEYS, nb), rng.random(nb) < 0.1, R.I64)]


class Table:
    """a join table on the device plus what the reference needs to know about it"""

    def __init__(self, dense):
        self.dense = dense
        self.keep = []
        self.jt = _L().JoinTable()
        self.jt.dense = dense

    # reference: matches of the probe rows that pass
    def matches(self, pcols, passing, key_cols):
        if self.dense:
            return J.dense_matches(pcols[key_cols[0]], self.kmin, self.range,
                                   self.lookup_h if self.dense == 1 else self.present, self.dense, passing)
        return J.hash_matches([pcols[k] for k in key_cols], self.bkeys, passing)


def chained_table(n, rng, nkeys=2, hot=True):
    """two keys (int with NULLs and edges, float with NaN / ±0.0 / ±inf), duplicates, and HOT rows sharing
    the key (7, -0.0); built by b2_join_build at cap = pow2 >= 2 n_build"""
    import torch
    L = _L()
    nb = min(max(n // 2, 8), 20_000)
    k0 = rng.integers(0, nb // 2 + 2, nb).astype(np.int64)
    edge = rng.random(nb) < 0.03
    k0[edge] = rng.choice(INT_KEYS, int(edge.sum()))
    k1 = rng.choice(FLOAT_KEYS, nb)
    n0, n1 = rng.random(nb) < 0.05, rng.random(nb) < 0.03
    if hot:
        k0 = np.concatenate([k0, np.full(HOT, 7, np.int64)])
        k1 = np.concatenate([k1, np.full(HOT, -0.0)])
        n0, n1 = np.concatenate([n0, np.zeros(HOT, bool)]), np.concatenate([n1, np.zeros(HOT, bool)])
    bkeys = [R.Column(k0, n0, R.I64), R.Column(k1, n1, R.F64)][:nkeys]
    t = Table(0)
    t.nb = len(k0)
    t.bkeys = bkeys
    t.payload = build_payload(t.nb, rng)
    cap = 1 << max(1, (2 * t.nb - 1).bit_length())
    head = torch.full((cap,), -1, dtype=torch.int32, device=_dev())
    nxt = torch.full((t.nb,), 0x5A5A5A5A, dtype=torch.int32, device=_dev())
    arr = col_array(bkeys, t.keep)
    L.join_build(arr, nkeys, t.nb, _ptr(head), _ptr(nxt), cap, _stream())
    t.keep += [head, nxt]
    t.jt.nkeys, t.jt.head, t.jt.next, t.jt.cap = nkeys, head.data_ptr(), nxt.data_ptr(), cap
    for i in range(nkeys):
        t.jt.keys[i] = arr[i]
    return t


def chained_probe_keys(n, t: Table, rng):
    """keys from the build's pool (so most rows match), some misses, the HOT key at two rows of one warp"""
    k0 = rng.integers(-2, t.nb // 2 + 4, n).astype(np.int64) if n else np.zeros(0, np.int64)
    edge = rng.random(n) < 0.03
    k0[edge] = rng.choice(INT_KEYS, int(edge.sum()))
    k1 = rng.choice(FLOAT_KEYS, n) if n else np.zeros(0)
    if t.nb > HOT:
        for r in (3, 40):
            if r < n:
                k0[r], k1[r] = 7, 0.0
    return k0, k1


def direct_table(dense, n, rng, kmin):
    """unique keys over [kmin, kmin + range) with holes.  dense 1: int32 lookup (from the reference) over build
    rows that also hold NULL and out-of-range keys; dense 2: presence bitmap and key-ordered payloads (I64 row id,
    F64, U8, U32 + base, U32 with the 0xFFFFFFFF sentinel)"""
    rng_ = 4099
    t = Table(dense)
    t.kmin, t.range = kmin, rng_
    present = rng.random(rng_) < 0.7
    present[[0, rng_ - 1]] = True
    offs = np.flatnonzero(present)
    keys = (np.uint64(kmin & (2 ** 64 - 1)) + offs.astype(np.uint64)).view(np.int64)
    if dense == 1:
        perm = rng.permutation(len(keys))
        bk = keys[perm]
        extra = np.array([kmin - 1 if kmin != MIN else MAX, kmin + rng_ if kmin <= MAX - rng_ else MIN, keys[0]],
                         np.int64)
        bk = np.concatenate([bk, extra])
        bnull = np.zeros(len(bk), bool)
        bnull[-1] = True                  # a NULL row whose value duplicates a real key
        key = R.Column(bk, bnull, R.I64)
        lookup, dup, _ = J.dense_build(key, kmin, rng_)
        assert dup == 0
        t.nb = len(bk)
        t.payload = build_payload(t.nb, rng)
        t.lookup_h = lookup
        lk = _t(lookup)
        t.keep.append(lk)
        t.jt.lookup = lk.data_ptr()
    else:
        t.present = present
        t.nb = rng_
        pay = build_payload(rng_, rng)
        base = -2 ** 40
        u32 = rng.integers(0, 2 ** 32, rng_, dtype=np.uint64).astype(np.uint32)
        u32[:3] = [0, 2 ** 32 - 1, 2 ** 32 - 2]
        sent = rng.integers(0, 2 ** 32 - 1, rng_, dtype=np.uint64).astype(np.uint32)
        sent[:2] = [2 ** 32 - 2, 0]
        sent[~present] = 2 ** 32 - 1
        t.u32_base = base
        t.payload = pay + [R.Column(u32, None, J.U32), R.Column(sent, None, J.U32)]
        pw = _t(R.pack_valid(present).view(np.int32))
        t.keep.append(pw)
        t.jt.lookup = pw.data_ptr()
    t.keys = keys
    t.jt.nkeys, t.jt.kmin, t.jt.range = 1, kmin, rng_
    t.jt.keys[0] = col_struct(R.Column(keys, None, R.I64), t.keep)
    return t


def direct_probe_keys(n, t: Table, rng):
    """keys in range (hits and holes), just outside it (kmin - 1, kmin + range), and far away"""
    off = rng.integers(-3, t.range + 3, n).astype(np.int64) if n else np.zeros(0, np.int64)
    k = (np.uint64(t.kmin & (2 ** 64 - 1)) + off.view(np.uint64)).view(np.int64)
    far = rng.random(n) < 0.02
    k[far] = rng.choice(INT_KEYS, int(far.sum()))
    return k


def _u32_flags(t, cols):
    return [J.COL_SENTINEL if c is t.payload[-1] and t.dense == 2 else 0 for c in cols]


# ---- builds --------------------------------------------------------------------------------------------------
def _build_keys(n, rng, dtypes):
    cols = []
    for i, dt in enumerate(dtypes):
        if dt == R.I64:
            v = rng.integers(-5, max(n // 3, 2), n).astype(np.int64)
            e = rng.random(n) < 0.05
            v[e] = rng.choice(INT_KEYS, int(e.sum()))
        else:
            v = rng.choice(FLOAT_KEYS, n) if n else np.zeros(0)
        cols.append(R.Column(v, (rng.random(n) < 0.07) if i % 2 == 0 else None, dt))
    return cols


KEY_SETS = [[R.I64], [R.F64], [R.F64, R.I64], [R.I64, R.F64, R.I64, R.F64]]


@pytest.mark.parametrize("n", SIZES)
def test_join_build_chains(n):
    """b2_join_build at cap 1, 2, 64 and pow2 >= 2n over 1-4 keys of mixed dtype with NULL bitmaps, NaN of several
    payloads, ±0.0, ±inf and INT64_MIN / MAX: every chain invariant the probe relies on"""
    import torch
    L = _L()
    rng = np.random.default_rng(100 + n)
    for dtypes in KEY_SETS:
        keys = _build_keys(n, rng, dtypes)
        for cap in (1, 2, 64, 1 << max(1, (2 * n - 1).bit_length())):
            keep = []
            arr = col_array(keys, keep)
            head = torch.full((cap,), -1, dtype=torch.int32, device=_dev())
            nxt = torch.full((max(n, 1),), 0x5A5A5A5A, dtype=torch.int32, device=_dev())
            L.join_build(arr, len(keys), n, _ptr(head), _ptr(nxt), cap, _stream())
            err = J.check_chains(_np(head), _np(nxt)[:n], keys)
            assert err is None, f"n={n} keys={dtypes} cap={cap}: {err}"


def _dense_keys(n, rng, kmin, rng_):
    """unique in-range keys (range >= n), a tenth of the rows just outside the range, some NULL"""
    k = n - n // 10
    offs = rng.permutation(rng_)[:k].astype(np.uint64)
    keys = (np.uint64(kmin & (2 ** 64 - 1)) + offs).view(np.int64)
    out = np.array([kmin - 1 if kmin != MIN else MAX, kmin + rng_ if kmin <= MAX - rng_ else MIN], np.int64)
    rest = n - k
    keys = np.concatenate([keys, rng.choice(out, rest) if rest else np.zeros(0, np.int64)])
    null = rng.random(n) < 0.05
    return R.Column(keys, null, R.I64)


def run_build_dense(key, kmin, rng_):
    import torch
    L = _L()
    keep = []
    lookup = torch.full((rng_,), -1, dtype=torch.int32, device=_dev())
    flags = _zeros(1)
    L.join_build_dense(C.byref(col_struct(key, keep)), key.n, kmin, rng_, _ptr(lookup), _ptr(flags), _stream())
    return _np(lookup), int(_np(flags)[0])


@pytest.mark.parametrize("n", SIZES)
def test_join_build_dense(n):
    """lookup word for word and flag 0 on unique keys; flag 1 and lookup[d] one of the duplicates' rows with one
    and with many duplicated keys; kmin = INT64_MIN and kmin + range - 1 = INT64_MAX; NULL and out-of-range keys"""
    rng = np.random.default_rng(200 + n)
    rng_ = max(n + n // 3, 40)
    for kmin in (-1000, MIN, MAX - rng_ + 1):
        key = _dense_keys(n, rng, kmin, rng_)
        lookup, flag = run_build_dense(key, kmin, rng_)
        exp, dup, _ = J.dense_build(key, kmin, rng_)
        assert dup == 0
        _assert_words(lookup, exp, f"n={n} kmin={kmin}: lookup")
        assert flag == 0, f"n={n} kmin={kmin}: duplicate flag set on unique keys"
        if n < 2:
            continue
        for ndup in (1, max(1, n // 4)):
            vals = key.values.copy()
            null = key.null.copy()
            live = np.flatnonzero(~null & J.offsets(key, kmin, rng_)[1])
            if len(live) < 2:
                continue
            src = rng.choice(live, min(ndup, len(live) - 1), replace=False)
            dst = rng.choice(np.setdiff1d(live, src), len(src), replace=len(src) > len(live) - len(src))
            vals[dst] = vals[src]
            dkey = R.Column(vals, null, R.I64)
            lookup, flag = run_build_dense(dkey, kmin, rng_)
            exp, dup, dups = J.dense_build(dkey, kmin, rng_)
            assert flag == 1 == dup, f"n={n} kmin={kmin} ndup={ndup}: duplicate flag {flag}"
            dmask = np.zeros(rng_, bool)
            dmask[list(dups)] = True
            _assert_words(lookup[~dmask], exp[~dmask], f"n={n} kmin={kmin} ndup={ndup}: unique offsets")
            for o, rows in dups.items():
                assert lookup[o] in rows, f"offset {o}: lookup {lookup[o]} is none of the rows {rows}"


def run_key_layout(key, kmin, rng_, col, out_dtype, base, out_init, with_valid, with_present):
    import torch
    L = _L()
    keep = []
    out = None
    if out_init is not None:
        out = _t(out_init.view(np.int32) if out_init.dtype == np.uint32 else out_init)
    valid = _zeros(_words(rng_) + 1) if with_valid else None
    present = _zeros(_words(rng_) + 1) if with_present else None
    cs = C.byref(col_struct(col, keep)) if col is not None else None
    L.join_key_layout(C.byref(col_struct(key, keep)), key.n, kmin, rng_, cs, out_dtype, base, _ptr(out),
                      _ptr(valid), _ptr(present), _stream())
    torch.cuda.synchronize()
    o = None if out is None else (_np(out).view(np.uint32) if out_init.dtype == np.uint32 else _np(out))
    return (o, None if valid is None else _np(valid).view(np.uint32),
            None if present is None else _np(present).view(np.uint32))


@pytest.mark.parametrize("n", SIZES)
def test_join_key_layout(n):
    """I64 -> I64 (nullable), I64 -> U32 with base at the value minimum over value ranges 2^32 - 2, 2^32 - 1 and
    2^32 (wraps to 0), F64 bits (NaN payloads, -0.0), U8, and presence only; offsets without a build row keep the
    garbage (or the 0xFFFFFFFF sentinel fill)"""
    rng = np.random.default_rng(300 + n)
    rng_ = max(n + n // 2, 70)
    kmin = MIN if n % 2 else 12345
    key = _dense_keys(n, rng, kmin, rng_)
    nw = _words(rng_) + 1
    pf = rng.choice(np.concatenate([FLOAT_KEYS, [3.25, -7.5]]), n) if n else np.zeros(0)
    cases = [("i64", R.Column(rng.choice(INT_KEYS, n) if n else np.zeros(0, np.int64), rng.random(n) < 0.2, R.I64),
              R.I64, 0, np.full(rng_, GARBAGE, np.int64)),
             ("f64", R.Column(pf, rng.random(n) < 0.1, R.F64), R.F64, 0, np.full(rng_, GARBAGE, np.int64)),
             ("u8", R.Column(rng.integers(0, 256, n).astype(np.uint8), rng.random(n) < 0.1, R.U8), R.U8, 0,
              np.full(rng_, 0x5A, np.uint8))]
    for span in (2 ** 32 - 2, 2 ** 32 - 1, 2 ** 32):
        base = -2 ** 45 + span
        v = base + rng.integers(0, span + 1, n, dtype=np.int64)
        if n:
            v[0] = base
        if n > 1:
            v[1] = base + span
        fill = np.uint32(0xFFFFFFFF) if span < 2 ** 32 - 1 else np.uint32(0xA5A5A5A5)
        cases.append((f"u32 span {span}", R.Column(v, None, R.I64), J.U32, base, np.full(rng_, fill, np.uint32)))
        cases.append((f"u32 span {span} nullable", R.Column(v, rng.random(n) < 0.1, R.I64), J.U32, base,
                      np.full(rng_, 0xA5A5A5A5, np.uint32)))
    for name, col, out_dtype, base, init in cases:
        for with_valid, with_present in ((True, True), (False, False)):
            got, gv, gp = run_key_layout(key, kmin, rng_, col, out_dtype, base, init, with_valid, with_present)
            exp, ev, ep = J.key_layout(key, kmin, rng_, col, out_dtype, base, init,
                                       np.zeros(nw, np.uint32) if with_valid else None,
                                       np.zeros(nw, np.uint32) if with_present else None)
            what = f"n={n} {name} valid={with_valid}"
            _assert_words(got, exp, f"{what}: out_data")
            if with_valid:
                _assert_words(gv, ev, f"{what}: out_valid")
            if with_present:
                _assert_words(gp, ep, f"{what}: present")
    _, _, gp = run_key_layout(key, kmin, rng_, None, 0, 0, None, False, True)
    _, _, ep = J.key_layout(key, kmin, rng_, None, 0, 0, None, None, np.zeros(nw, np.uint32))
    _assert_words(gp, ep, f"n={n} presence only")


# ---- the two-pass probe ----------------------------------------------------------------------------------------
def make_table(kind, n, rng):
    if kind == "chained":
        t = chained_table(n, rng)
        k0, k1 = chained_probe_keys(n, t, rng)
        cols = probe_cols(n, rng, k0, k1)
        return t, cols, [K0, K1]
    dense = 1 if kind == "dense1" else 2
    t = direct_table(dense, n, rng, MIN if n % 2 else -1000)
    cols = probe_cols(n, rng, direct_probe_keys(n, t, rng))
    return t, cols, [K0]


def _kmid(cols):
    v = np.sort(cols[KN].values)
    return int(v[len(v) // 2]) if len(v) else 0


def build_gather_cols(t, config):
    """(columns, flags) of the build side for a gather configuration"""
    if config == "full":
        cols = t.payload[:3] + (t.payload[4:6] if t.dense == 2 else t.payload[3:4])
    else:
        cols = [t.payload[2], t.payload[0], t.payload[1]]
    return cols, _u32_flags(t, cols)


def check_rows_and_gathers(what, t, e: J.Emitted, got_p, got_b, pg=None, pgc=(), bg=None, bgc=()):
    """probe indices exact, build runs as sets, every gathered word against the indices emitted beside it.
    Without a build index output a chained table's indices come from the gathered row id column (row + 1, so
    0 for none); a direct-address probe emits at most one row per probe row, so its runs are exact."""
    total = e.total
    if got_p is not None:
        _assert_words(got_p[:total].astype(np.int64), e.probe, f"{what}: probe indices")
    gb = e.build
    if got_b is not None:
        gb = got_b[:total].astype(np.int64)
    elif t.dense == 0 and any(c is t.payload[0] for c in bgc):
        gb = _np(bg.data[[c is t.payload[0] for c in bgc].index(True)])[:total] - 1
    _assert_words(J.sort_runs(e.probe, gb), e.build, f"{what}: build runs")
    for k, c in enumerate(pgc):
        vals, valid = J.gather_probe(c, e.probe)
        pg.check(k, total, vals, valid, f"{what}: probe")
    for k, c in enumerate(bgc):
        vals, valid = J.gather_build(c, gb, getattr(t, "u32_base", 0))
        bg.check(k, total, vals, valid, f"{what}: build")


def run_two_pass(t, pcols, key_cols, terms, mode, what):
    """b2_join_count, then b2_join_write and the two gather configurations"""
    import torch
    L = _L()
    n = pcols[0].n
    scan = scan_of(pcols, terms)
    pk = (C.c_int32 * len(key_cols))(*key_cols)
    passing = R.eval_terms(pcols, terms, n)
    e = J.emit(mode, passing, t.matches(pcols, passing, key_cols))
    ntiles = L.num_tiles(n)
    off = torch.full((ntiles + 1,), GARBAGE, dtype=torch.int64, device=_dev())
    L.join_count(C.byref(scan), pk, C.byref(t.jt), mode, _ptr(off), _stream())
    _assert_words(_np(off), J.tile_off(e.count, n), f"{what}: tile_off")
    total = e.total
    inner_left = mode in (J.JOIN_INNER, J.JOIN_LEFT)

    # indices only, with build_matched
    op = torch.full((total + SLACK,), -7, dtype=torch.int32, device=_dev())
    ob = torch.full((total + SLACK,), -7, dtype=torch.int32, device=_dev())
    bm = _zeros(t.nb + 8, torch.uint8) if inner_left else None
    L.join_write(C.byref(scan), pk, C.byref(t.jt), mode, _ptr(off), _ptr(op), _ptr(ob), _ptr(bm), _stream())
    got_p, got_b = _np(op), _np(ob)
    _assert_words(got_p[total:], np.full(SLACK, -7, np.int32), f"{what}: probe indices past the total")
    _assert_words(got_b[total:], np.full(SLACK, -7, np.int32), f"{what}: build indices past the total")
    check_rows_and_gathers(what + " write", t, e, got_p, got_b)
    if bm is not None:
        exp = np.zeros(t.nb + 8, np.uint8)
        exp[: t.nb] = J.build_matched(mode, e, t.nb)
        _assert_words(_np(bm)[: t.nb + 8], exp, f"{what}: build_matched")

    for config in ("full", "bare"):
        full = config == "full"
        pgi = (PID, K0, PF, PU) if full else (PU, PF, PID)
        pgc = [pcols[i] for i in pgi]
        bgc, flags = build_gather_cols(t, config) if inner_left else ([], [])
        pg = Gathered([_out_dtype(c) for c in pgc], total, full)
        bg = Gathered([_out_dtype(c) for c in bgc], total, full)
        keep = []
        bcols = col_array(bgc, keep, flags)
        op = torch.full((total + SLACK,), -7, dtype=torch.int32, device=_dev()) if full else None
        ob = torch.full((total + SLACK,), -7, dtype=torch.int32, device=_dev()) if full else None
        pc = (C.c_int32 * len(pgi))(*pgi)
        args = (C.byref(scan), pk, C.byref(t.jt), mode, _ptr(off), _ptr(op), _ptr(ob), None, len(pgc), pc, pg.out,
                pg.vptr(), len(bgc), bcols)
        if t.dense == 2:
            base = (C.c_int64 * max(1, len(bgc)))(*[t.u32_base] * len(bgc))
            L.join_write_gather_keyed(*args, base, bg.out, bg.vptr(), _stream())
        else:
            L.join_write_gather(*args, bg.out, bg.vptr(), _stream())
        check_rows_and_gathers(f"{what} gather {config}", t, e, _np(op) if full else None,
                               _np(ob) if full else None, pg, pgc, bg, bgc)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["chained", "dense1", "dense2"])
def test_join_two_pass(kind, n):
    """{chained, direct-address, key-ordered} x 4 modes x {no term, a term on another column, on the key, an F64
    term}: tile_off, probe indices, build runs, gathered I64 / F64 / U8 (/ U32) columns of both sides with and
    without validity outputs, build_matched; probe rows with 5000 matches beside single matches in one warp"""
    rng = np.random.default_rng(400 + n)
    t, pcols, key_cols = make_table(kind, n, rng)
    for terms in (T_NONE, T_OTHER, t_key(_kmid(pcols)), T_F64):
        for mode in MODES:
            run_two_pass(t, pcols, key_cols, terms, mode, f"{kind} n={n} mode={mode} terms={terms}")


# ---- b2_join_onepass ---------------------------------------------------------------------------------------------
ONEPASS_CONFIGS = [
    # (probe columns, build payload indices, validity outputs): first other 8-byte probe column held from trip 1,
    # first build column fetched speculatively (I64 / U32) or not (U8)
    ((K0, PID, PF, PU), (4, 1, 2, 0), True),
    ((PU, PF), (2, 0, 1), False),
    ((), (0,), False),
]


def run_onepass(t, pcols, key_cols, terms, mode, lookback, pgi, bgi, with_valid, what, order="probe"):
    """b2_join_onepass with outputs allocated at n rows of garbage; order "probe" compares row for row, "batch"
    sorts by the gathered row id (which must be the first probe column) and checks the per-batch order"""
    import torch
    L = _L()
    n = pcols[0].n
    scan = scan_of(pcols, terms)
    pk = (C.c_int32 * len(key_cols))(*key_cols)
    passing = R.eval_terms(pcols, terms, n)
    e = J.emit(mode, passing, t.matches(pcols, passing, key_cols))
    pgc = [pcols[i] for i in pgi]
    bgc = [t.payload[i] for i in bgi if t.dense == 2 or i < 4] if mode in (J.JOIN_INNER, J.JOIN_LEFT) else []
    flags = _u32_flags(t, bgc)
    pg = Gathered([_out_dtype(c) for c in pgc], n, with_valid)
    bg = Gathered([_out_dtype(c) for c in bgc], n, with_valid)
    keep = []
    bcols = col_array(bgc, keep, flags)
    base = (C.c_int64 * max(1, len(bgc)))(*[getattr(t, "u32_base", 0)] * len(bgc))
    ws = torch.zeros(L.join_onepass_ws_bytes(n) // 8 + 1, dtype=torch.int64, device=_dev())
    pc = (C.c_int32 * max(1, len(pgc)))(*list(pgi))
    L.join_onepass(C.byref(scan), pk, C.byref(t.jt), mode, lookback, _ptr(ws), len(pgc), pc, pg.out, pg.vptr(),
                   len(bgc), bcols, base, bg.out, bg.vptr(), _stream())
    total = int(_np(ws)[0])
    assert total == e.total, f"{what}: ws[0] = {total} rows, expected {e.total}"
    if order == "probe":
        perm = np.arange(total)
    else:
        got_pid = _np(pg.data[0])[:total]
        batch = 2048 if order == "tile" else 256
        check_batch_order(got_pid, batch, what)
        perm = np.argsort(got_pid, kind="stable")
    for k, c in enumerate(pgc):
        vals, valid = J.gather_probe(c, e.probe)
        check_permuted(pg, k, total, perm, vals, valid, f"{what}: probe")
    for k, c in enumerate(bgc):
        vals, valid = J.gather_build(c, e.build, getattr(t, "u32_base", 0))
        check_permuted(bg, k, total, perm, vals, valid, f"{what}: build")
    return pg, bg, total


def check_permuted(g: Gathered, k, total, perm, vals, valid, what):
    """output column k, read in the order `perm`, against the reference; rows past the total unchanged"""
    got = _np(g.data[k])
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    u8 = g.dtypes[k] == R.U8
    exp = np.asarray(vals, got.dtype)
    _assert_words(got[:total][perm], exp, f"{what}: column {k} values")
    _assert_words(got[total:], np.full(len(got) - total, 0x5A if u8 else GARBAGE, got.dtype),
                  f"{what}: column {k} rows past the {total} emitted")
    if g.valid[k] is not None:
        w = _np(g.valid[k]).view(np.uint32)
        v = np.asarray(valid, bool)[inv] if total else np.zeros(0, bool)
        _assert_words(w, J.valid_words(v, len(w)), f"{what}: column {k} validity words")


def check_batch_order(pid, batch, what):
    """rows of one `batch`-row probe batch are contiguous in the output and in probe order"""
    pid = np.asarray(pid, np.int64)
    if not len(pid):
        return
    b = pid // batch
    same = b[1:] == b[:-1]
    assert (pid[1:][same] > pid[:-1][same]).all(), f"{what}: a batch's rows are out of probe order"
    starts = b[np.concatenate([[True], ~same])]
    assert len(np.unique(starts)) == len(starts), f"{what}: a batch's rows are split"


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("lookback", [0, 1])
@pytest.mark.parametrize("dense", [1, 2])
def test_join_onepass_ordered(dense, lookback, n):
    """counted (lookback 0) and decoupled look-back (1) probes of direct-address and key-ordered tables: row for
    row in probe order in all four modes, ws[0] the total, garbage past it untouched"""
    rng = np.random.default_rng(500 + n)
    t, pcols, key_cols = make_table("dense1" if dense == 1 else "dense2", n, rng)
    for terms in (T_NONE, T_OTHER, t_key(_kmid(pcols))):
        for mode in MODES:
            for pgi, bgi, wv in ONEPASS_CONFIGS:
                run_onepass(t, pcols, key_cols, terms, mode, lookback, pgi, bgi, wv,
                            f"dense={dense} lookback={lookback} n={n} mode={mode} terms={terms} probe={pgi}")


# the 30 launchable instances of b2_join_stream_kernel<HAS_P, BMODE, OUT_KEY, CTA_RES>, per reservation
STREAM_INSTANCES = [(hp, bm, ok) for hp in (False, True) for bm in range(4) for ok in (False, True)
                    if hp or bm or ok]
STREAM_PAYLOAD = {1: 0, 2: 4, 3: 5}     # BMODE -> key-ordered payload: I64 row id, U32 + base, U32 sentinel


def run_stream(t, pcols, terms, mode, pgi, bgi, what, tile_order):
    """b2_join_onepass(lookback = 2); with the row id gathered (first probe column) the output is sorted by it
    and compared exactly, otherwise compared as a multiset of rows"""
    import torch
    L = _L()
    n = pcols[0].n
    scan = scan_of(pcols, terms)
    pk = (C.c_int32 * 1)(KN)
    passing = R.eval_terms(pcols, terms, n)
    e = J.emit(mode, passing, t.matches(pcols, passing, [KN]))
    pgc = [pcols[i] for i in pgi]
    bgc = [t.payload[i] for i in bgi]
    pg = Gathered([R.I64] * len(pgc), n, False)
    bg = Gathered([_out_dtype(c) for c in bgc], n, False)
    keep = []
    bcols = col_array(bgc, keep, _u32_flags(t, bgc))
    base = (C.c_int64 * max(1, len(bgc)))(*[t.u32_base] * len(bgc))
    ws = torch.zeros(L.join_onepass_ws_bytes(n) // 8 + 1, dtype=torch.int64, device=_dev())
    pc = (C.c_int32 * max(1, len(pgc)))(*list(pgi))
    L.join_onepass(C.byref(scan), pk, C.byref(t.jt), mode, 2, _ptr(ws), len(pgc), pc, pg.out, None, len(bgc), bcols,
                   base, bg.out, None, _stream())
    total = int(_np(ws)[0])
    assert total == e.total, f"{what}: ws[0] = {total} rows, expected {e.total}"
    exp = [J.gather_probe(c, e.probe)[0] for c in pgc] + [J.gather_build(c, e.build, t.u32_base)[0] for c in bgc]
    got = [_np(x) for x in pg.data + bg.data]
    for k, g in enumerate(got):
        _assert_words(g[total:], np.full(len(g) - total, GARBAGE, g.dtype), f"{what}: column {k} past the total")
    got = [g[:total] for g in got]
    if pgi and pgi[0] == PID:
        check_batch_order(got[0], 2048 if tile_order else 256, what)
        perm = np.argsort(got[0], kind="stable")
        for k, (g, x) in enumerate(zip(got, exp)):
            _assert_words(g[perm], np.asarray(x, np.int64), f"{what}: column {k}")
    else:
        gs = np.stack(got, axis=1) if got else np.zeros((total, 0), np.int64)
        xs = np.stack([np.asarray(x, np.int64) for x in exp], axis=1)
        gs, xs = gs[np.lexsort(gs.T[::-1])] if len(gs) else gs, xs[np.lexsort(xs.T[::-1])] if len(xs) else xs
        _assert_words(gs.reshape(-1), xs.reshape(-1), f"{what}: rows as a multiset")


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("reserve", ["cta", "warp"])
def test_join_onepass_stream(reserve, n):
    """lookback = 2 reaches every instance of the streaming kernel (extra probe column, build payload mode 0-3,
    key output) under B200SQL_JOIN_RESERVE=cta / warp, and every shape that falls back to the generic kernel:
    nullable key, U8 column, validity output, LEFT / ANTI, two build columns, three probe columns, a direct-address
    (not key-ordered) table.  CTA reservation keeps each 2048-row tile's rows together and in probe order, warp
    reservation and the generic kernel each 256-row warp batch's."""
    rng = np.random.default_rng(600 + n)
    t, pcols, _ = make_table("dense2", n, rng)
    t1, p1, _ = make_table("dense1", n, rng)
    with env(B200SQL_JOIN_RESERVE=reserve):
        for terms in (T_NONE, T_OTHER):
            for hp, bm, ok in STREAM_INSTANCES:
                pgi = ([PID] if hp else []) + ([KN] if ok else [])
                bgi = [STREAM_PAYLOAD[bm]] if bm else []
                for mode in (J.JOIN_INNER, J.JOIN_SEMI) if not bm else (J.JOIN_INNER,):
                    run_stream(t, pcols, terms, mode, pgi, bgi,
                               f"stream {reserve} n={n} hp={hp} bmode={bm} key={ok} mode={mode} terms={terms}",
                               reserve == "cta")
            # fallbacks to the generic kernel (one atomic per warp batch): row id first, so sorted compare
            what = f"generic {reserve} n={n} terms={terms}"
            for name, key_cols, pgi, bgi, mode, wv in [
                    ("nullable key", [K0], (PID,), (0,), J.JOIN_INNER, False),
                    ("U8 probe column", [KN], (PID, PU), (0,), J.JOIN_INNER, False),
                    ("U8 build column", [KN], (PID,), (2,), J.JOIN_INNER, False),
                    ("validity output", [KN], (PID, KN), (4,), J.JOIN_INNER, True),
                    ("LEFT", [KN], (PID, KN), (0,), J.JOIN_LEFT, False),
                    ("ANTI", [KN], (PID,), (), J.JOIN_ANTI, False),
                    ("two build columns", [KN], (PID,), (0, 4), J.JOIN_INNER, False),
                    ("three probe columns", [KN], (PID, KN, P), (5,), J.JOIN_INNER, False)]:
                run_onepass(t, pcols, key_cols, terms, mode, 2, pgi, bgi, wv, f"{what} {name}", order="batch")
            run_onepass(t1, p1, [KN], terms, J.JOIN_INNER, 2, (PID, KN), (0,), False, f"{what} dense 1", order="batch")


# ---- one run per probe kernel with wrapping tile loops -------------------------------------------------------------
def test_join_probes_wrap_their_tile_loops():
    """2112 x 4096 + 1 probe rows: more than two waves of resident blocks for 4096- and 2048-row tiles, look-back
    over more than 32 predecessors and a partial last tile, for the two-pass probe (chained and direct-address),
    the counted and look-back one-pass probes, the streaming kernel under both reservations and the generic one"""
    n = BIG_N
    rng = np.random.default_rng(700)
    for kind in ("chained", "dense1"):
        if kind == "chained":
            t = chained_table(40_000, rng, nkeys=1, hot=False)
            k = rng.integers(-2, t.nb // 2 + 4, n).astype(np.int64)
            pcols = probe_cols(n, rng, k, np.zeros(n))
        else:
            t = direct_table(1, 40_000, rng, -1000)
            pcols = probe_cols(n, rng, direct_probe_keys(n, t, rng))
        run_two_pass_big(t, pcols, kind)
    t = direct_table(2, 40_000, rng, -1000)
    pcols = probe_cols(n, rng, direct_probe_keys(n, t, rng))
    for lookback in (0, 1):
        run_onepass(t, pcols, [K0], T_OTHER, J.JOIN_LEFT, lookback, (PID, PF), (4, 1), True,
                    f"big onepass lookback={lookback}")
    for reserve in ("cta", "warp"):
        with env(B200SQL_JOIN_RESERVE=reserve):
            run_stream(t, pcols, T_OTHER, J.JOIN_INNER, [PID, KN], [4], f"big stream {reserve}", reserve == "cta")
    run_onepass(t, pcols, [K0], T_OTHER, J.JOIN_INNER, 2, (PID,), (0,), False, "big generic", order="batch")


def run_two_pass_big(t, pcols, kind):
    import torch
    L = _L()
    n = pcols[0].n
    scan = scan_of(pcols, T_OTHER)
    pk = (C.c_int32 * 1)(K0)
    passing = R.eval_terms(pcols, T_OTHER, n)
    e = J.emit(J.JOIN_LEFT, passing, t.matches(pcols, passing, [K0]))
    ntiles = L.num_tiles(n)
    off = torch.full((ntiles + 1,), GARBAGE, dtype=torch.int64, device=_dev())
    L.join_count(C.byref(scan), pk, C.byref(t.jt), J.JOIN_LEFT, _ptr(off), _stream())
    _assert_words(_np(off), J.tile_off(e.count, n), f"big {kind}: tile_off")
    total = e.total
    pgc, bgc = [pcols[PID]], [t.payload[0], t.payload[1]]
    pg, bg = Gathered([R.I64], total, True), Gathered([R.I64, R.I64], total, True)
    ob = torch.full((total + SLACK,), -7, dtype=torch.int32, device=_dev())
    keep = []
    bcols = col_array(bgc, keep)
    pc = (C.c_int32 * 1)(PID)
    L.join_write_gather(C.byref(scan), pk, C.byref(t.jt), J.JOIN_LEFT, _ptr(off), None, _ptr(ob), None, 1, pc, pg.out,
                        pg.vptr(), 2, bcols, bg.out, bg.vptr(), _stream())
    check_rows_and_gathers(f"big {kind}", t, e, None, _np(ob), pg, pgc, bg, bgc)


# ---- argument errors -----------------------------------------------------------------------------------------------
class ArgCase:
    """a small probe (one tile) whose every buffer is sized for what an unchecked launch would touch: outputs
    of n rows (one tile emits at most n rows at any offset the zeroed tile_off gives), U8 key buffers of 8 n
    bytes, probe keys within the first words of the table"""
    N = 64

    def __init__(self):
        import torch
        L = _L()
        n = self.N
        self.keep = []
        ids = np.arange(n, dtype=np.int64)
        self.cols = [R.Column(ids, None, R.I64), R.Column(ids.astype(np.float64), None, R.F64),
                     R.Column(np.zeros(8 * n, np.uint8), None, R.U8)]
        self.scan = L.Scan()
        self.scan.ncols, self.scan.nterms, self.scan.n = 3, 0, n
        for i, c in enumerate(self.cols):
            self.scan.cols[i] = col_struct(c, self.keep)
        self.lookup = torch.full((4 * n,), -1, dtype=torch.int32, device=_dev())
        self.lookup[: n].copy_(torch.arange(n, dtype=torch.int32))
        self.present = torch.full((4 * n,), -1, dtype=torch.int32, device=_dev())
        self.head = torch.full((n,), -1, dtype=torch.int32, device=_dev())
        self.next = torch.full((n,), -1, dtype=torch.int32, device=_dev())
        self.off = _zeros(8, torch.int64)
        self.outp = _zeros(n)
        self.outb = _zeros(n)
        self.matched = _zeros(4 * n, torch.uint8)
        self.ws = torch.zeros(L.join_onepass_ws_bytes(n) // 8 + 1, dtype=torch.int64, device=_dev())
        self.gout = _zeros(4 * n, torch.int64)
        self.gval = _zeros(n)
        self.bcol = col_struct(R.Column(np.arange(4 * n, dtype=np.int64), None, R.I64), self.keep)

    def table(self, dense, key_col=0, rng_=None):
        jt = _L().JoinTable()
        jt.nkeys, jt.dense = 1, dense
        jt.keys[0] = self.scan.cols[key_col]
        if dense:
            jt.lookup = self.present.data_ptr() if dense == 2 else self.lookup.data_ptr()
            jt.kmin, jt.range = 0, rng_ or self.N
        else:
            jt.head, jt.next, jt.cap = self.head.data_ptr(), self.next.data_ptr(), self.N
        return jt

    def probes(self, jt, key_col, mode=J.JOIN_INNER, nbuild=0, matched=False, nprobe=0):
        """rc of every probe entry point that takes the arguments (b2_join_count takes no gather columns and no
        build_matched)"""
        lib = _L()._lib
        pk = (C.c_int32 * 4)(key_col, key_col, key_col, key_col)
        gcols = (C.c_int32 * 9)(*[0] * 9)
        gout = _ptrs([self.gout] * 9)
        gval = _ptrs([self.gval] * 9)
        bcols = (_L().Col * 9)(*[self.bcol] * 9)
        base = (C.c_int64 * 9)(*[0] * 9)
        mp = _ptr(self.matched) if matched else None
        s, st = C.byref(self.scan), _stream()
        rcs = {}
        if not nbuild and not nprobe and not matched:
            rcs["count"] = lib.b2_join_count(s, pk, C.byref(jt), mode, _ptr(self.off), st)
        self.off.zero_()
        if not nbuild and not nprobe:
            rcs["write"] = lib.b2_join_write(s, pk, C.byref(jt), mode, _ptr(self.off), _ptr(self.outp), _ptr(self.outb),
                                             mp, st)
        self.off.zero_()
        rcs["write_gather"] = lib.b2_join_write_gather(s, pk, C.byref(jt), mode, _ptr(self.off), _ptr(self.outp),
                                                       _ptr(self.outb), mp, nprobe, gcols, gout, gval, nbuild, bcols,
                                                       gout, gval, st)
        self.off.zero_()
        rcs["write_gather_keyed"] = lib.b2_join_write_gather_keyed(
            s, pk, C.byref(jt), mode, _ptr(self.off), _ptr(self.outp), _ptr(self.outb), mp, nprobe, gcols, gout, gval,
            nbuild, bcols, base, gout, gval, st)
        if jt.dense and not matched:
            self.ws.zero_()
            rcs["onepass"] = lib.b2_join_onepass(s, pk, C.byref(jt), mode, 1, _ptr(self.ws), nprobe, gcols, gout, gval,
                                                 nbuild, bcols, base, gout, gval, st)
        _np(self.off)
        return rcs


def _all_rejected(rcs, what, wrong=None):
    """every rc B2_ERR_ARG (-2); with `wrong` the misses are collected there instead of raised"""
    bad = {k: v for k, v in rcs.items() if v != -2}
    if wrong is not None and bad:
        wrong.append(f"{what}: {bad}")
    assert wrong is not None or not bad, f"{what}: expected B2_ERR_ARG (-2) from every entry point, got {bad}"


def _report(wrong):
    assert not wrong, "accepted, expected B2_ERR_ARG (-2):\n  " + "\n  ".join(wrong)


def test_join_rejects_semi_anti_build_columns_and_matched_flags():
    """build gather columns and build_matched are for INNER / LEFT only: the chained SEMI probe fills build
    columns with NULL and flags only the first partner, the direct-address probes gather the partner"""
    a = ArgCase()
    wrong = []
    for dense in (0, 1, 2):
        jt = a.table(dense)
        for mode in (J.JOIN_SEMI, J.JOIN_ANTI):
            _all_rejected(a.probes(jt, 0, mode, nbuild=1), f"dense={dense} mode={mode} with a build column", wrong)
            _all_rejected(a.probes(jt, 0, mode, matched=True), f"dense={dense} mode={mode} with build_matched", wrong)
        for mode in (J.JOIN_INNER, J.JOIN_LEFT):
            for kw in ({"nbuild": 1}, {"matched": True}):
                rcs = a.probes(jt, 0, mode, **kw)
                assert all(v == 0 for v in rcs.values()), f"dense={dense} mode={mode} {kw}: {rcs}"
    _report(wrong)


def test_join_rejects_bad_tables():
    """U8 keys, a table kind outside {0, 1, 2}, an F64 key on a direct-address table, a key-ordered range >= 2^31"""
    a = ArgCase()
    wrong = []
    for dense in (0, 1, 2):
        _all_rejected(a.probes(a.table(dense, key_col=2), 2), f"dense={dense}: U8 key", wrong)
    for dense in (-1, 3):
        _all_rejected(a.probes(a.table(dense), 0), f"dense={dense}", wrong)
    for dense in (1, 2):
        _all_rejected(a.probes(a.table(dense, key_col=1), 1), f"dense={dense}: F64 key", wrong)
    for rng_ in (1 << 31, 1 << 33):
        _all_rejected(a.probes(a.table(2, rng_=rng_), 0), f"key-ordered range {rng_}", wrong)
    assert all(v == 0 for v in a.probes(a.table(1, rng_=1 << 31), 0).values()), "a direct-address range >= 2^31"
    _report(wrong)


def test_join_rejects_bad_arguments():
    """the existing checks: nkeys 0 / 5, cap not a power of two, mode 4, more than 8 gather columns, a U32
    payload on a table that is not key-ordered, a key layout over range >= 2^31"""
    import torch
    L = _L()
    lib = L._lib
    a = ArgCase()
    st = _stream()
    keys = (L.Col * 5)(*[a.scan.cols[0]] * 5)
    for nkeys in (0, 5):
        assert lib.b2_join_build(keys, nkeys, a.N, _ptr(a.head), _ptr(a.next), a.N, st) == -2, f"build nkeys {nkeys}"
        jt = a.table(0)
        jt.nkeys = nkeys
        _all_rejected(a.probes(jt, 0), f"table nkeys {nkeys}")
    assert lib.b2_join_build(keys, 1, a.N, _ptr(a.head), _ptr(a.next), 3, st) == -2, "cap 3"
    jt = a.table(0)
    jt.cap = 3
    _all_rejected(a.probes(jt, 0), "table cap 3")
    _all_rejected(a.probes(a.table(1), 0, mode=4), "mode 4")
    _all_rejected(a.probes(a.table(1), 0, nprobe=9), "9 probe gather columns")
    _all_rejected(a.probes(a.table(1), 0, nbuild=9), "9 build gather columns")
    u32 = L.Col()
    u32.data, u32.dtype = a.bcol.data, L.U32
    lib_rc = lib.b2_join_write_gather_keyed(
        C.byref(a.scan), (C.c_int32 * 1)(0), C.byref(a.table(1)), J.JOIN_INNER, _ptr(a.off), None, None, None, 0,
        None, None, None, 1, (L.Col * 1)(u32), (C.c_int64 * 1)(0), _ptrs([a.gout]), None, st)
    assert lib_rc == -2, "U32 payload on a direct-address table"
    out = _zeros(4 * a.N, torch.int64)
    for rng_ in (1 << 31, 1 << 32):
        rc = lib.b2_join_key_layout(C.byref(a.scan.cols[0]), a.N, 0, rng_, C.byref(a.scan.cols[0]), L.I64, 0,
                                    _ptr(out), None, _ptr(a.present), st)
        assert rc == -2, f"key layout range {rng_}"
    torch.cuda.synchronize()
