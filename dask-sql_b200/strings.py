"""VARCHAR columns as dictionary codes: the only module that knows the dictionary rules.

A VARCHAR column is an int64 code column (plus the usual validity bitmap: NULL is the bitmap) into a
per-column dictionary that holds the column's distinct non-NULL values sorted by their UTF-8 bytes --
code-point order, which is Python's `str` order.  Code order is therefore string order, and `=`, `<`,
BETWEEN, IN, prefix LIKE, GROUP BY, DISTINCT, MIN / MAX, ORDER BY and joins run on the int64 kernels.

The dictionary travels with the column inside its logical type: `Varchar` is a `str` whose value is
"category" (so every place that copies a column's logical type copies the dictionary too) and which
carries `.dictionary`.  Where two code columns meet, their dictionaries are compared by content digest,
never by the logical string.

Per-entry device work (a general LIKE, translating one dictionary into another) runs once per
dictionary entry (b2_str_like / b2_str_lower_bound) into a table that B2_OP_MAP looks up per row.
"""
import hashlib
import weakref
from typing import Optional

import numpy as np

from . import _lib as L
from .expr import Expr, Lit, Call, I64, U8

LOGICAL = "category"


# ---------------------------------------------------------------------------------------------
# dictionaries
# ---------------------------------------------------------------------------------------------
class Dictionary:
    """Sorted unique UTF-8 strings: host `large_string` array plus a lazily uploaded device copy
    (int64 offsets, uint8 chars) per device.  Equal contents give the same object (`intern`)."""

    def __init__(self, values):
        import pyarrow as pa
        values = values.cast(pa.large_string())
        n = len(values)
        bufs = values.buffers()
        off = np.frombuffer(bufs[1], dtype=np.int64)[values.offset: values.offset + n + 1] if n else \
            np.zeros(1, dtype=np.int64)
        start, end = int(off[0]), int(off[-1])
        chars = bytes(memoryview(bufs[2])[start:end]) if n and bufs[2] is not None else b""
        self._setup(np.ascontiguousarray(off - start), chars)

    def _setup(self, offsets, chars, digest=None):
        import pyarrow as pa
        self.offsets, self.chars = offsets, chars
        n = len(offsets) - 1
        self.values = pa.LargeStringArray.from_buffers(n, pa.py_buffer(offsets.tobytes()), pa.py_buffer(chars))
        if digest is None:
            h = hashlib.blake2b(digest_size=16)
            h.update(offsets.tobytes())
            h.update(chars)
            digest = h.digest()
        self.digest = digest
        self._device = {}          # per-device copies and host caches: rebuilt where needed, never pickled
        self._categories = None
        self._objects = None

    def __reduce__(self):
        # what travels between ranks (merge.broadcast_part pickles logical types): the host arrays and the
        # digest only; the receiver reuses an equal dictionary it already holds
        return (_restore, (self.offsets, self.chars, self.digest))

    def __len__(self):
        return int(self.offsets.shape[0]) - 1

    def __repr__(self):
        return f"Dictionary({len(self)} entries, {self.digest.hex()[:8]})"

    def entry(self, i: int) -> bytes:
        return self.chars[self.offsets[i]: self.offsets[i + 1]]

    def lower_bound(self, key: bytes) -> int:
        """first code whose entry is >= key (bytes order)"""
        lo, hi = 0, len(self)
        while lo < hi:
            mid = (lo + hi) // 2
            if self.entry(mid) < key:
                lo = mid + 1
            else:
                hi = mid
        return lo

    def upper_bound(self, key: bytes) -> int:
        """first code whose entry is > key"""
        lb = self.lower_bound(key)
        return lb + 1 if lb < len(self) and self.entry(lb) == key else lb

    def code_of(self, s: str) -> Optional[int]:
        key = s.encode("utf-8")
        lb = self.lower_bound(key)
        return lb if lb < len(self) and self.entry(lb) == key else None

    def to_list(self):
        return self.values.to_pylist()

    def sorted_objects(self) -> np.ndarray:
        """the entries as a sorted numpy object array (Python str order is the dictionary's order), built once"""
        if self._objects is None:
            self._objects = np.array(self.to_list(), dtype=object)
        return self._objects

    def categories(self):
        """the dictionary as the pandas Index of a result's categories (built once)"""
        if self._categories is None:
            import pandas as pd
            self._categories = pd.Index(self.to_list(), dtype=object)
        return self._categories

    def device(self, dev):
        """(offsets int64[n + 1], chars uint8) on `dev`, uploaded on first use"""
        import torch
        key = dev.index
        if key not in self._device:
            off = torch.from_numpy(self.offsets.copy()).to(dev)
            chars = torch.frombuffer(bytearray(self.chars or b"\0"), dtype=torch.uint8).to(dev)
            self._device[key] = (off, chars)
        return self._device[key]


_INTERN = weakref.WeakValueDictionary()


def _restore(offsets, chars, digest) -> "Dictionary":
    got = _INTERN.get(digest)
    if got is None:
        got = Dictionary.__new__(Dictionary)
        got._setup(offsets, chars, digest)
        _INTERN[digest] = got
    return got


def intern(d: Dictionary) -> Dictionary:
    got = _INTERN.get(d.digest)
    if got is None:
        _INTERN[d.digest] = got = d
    return got


def same(a: Dictionary, b: Dictionary) -> bool:
    return a is b or a.digest == b.digest


class Varchar(str):
    """Logical type of a VARCHAR column: equal to "category" (what pandas calls it) and carrying the
    column's Dictionary."""

    def __new__(cls, dictionary: Dictionary):
        obj = str.__new__(cls, LOGICAL)
        obj.dictionary = dictionary
        return obj

    def __reduce__(self):
        return (Varchar, (self.dictionary,))


def is_varchar(x) -> bool:
    lg = x.logical if isinstance(x, Expr) else x
    return isinstance(lg, Varchar)


def dictionary_of(x) -> Dictionary:
    return (x.logical if isinstance(x, Expr) else x).dictionary


# ---------------------------------------------------------------------------------------------
# ingest: Arrow / pandas input -> (codes, NULL mask, logical)
# ---------------------------------------------------------------------------------------------
def is_string_type(t) -> bool:
    import pyarrow as pa
    return pa.types.is_string(t) or pa.types.is_large_string(t)


def is_string_dictionary_type(t) -> bool:
    import pyarrow as pa
    return pa.types.is_dictionary(t) and is_string_type(t.value_type)


def encode_arrow(arr):
    """A string or dictionary<int*, string> Arrow array (or chunked array, whose chunks may carry
    different dictionaries) -> (int64 codes, bool NULL mask or None, Varchar).

    The dictionary is the sorted unique non-NULL values that occur; input codes are remapped onto it
    with one host gather.  Duplicate Arrow dictionary entries map to one code, a NULL entry to NULL,
    and unused entries are dropped.  An ordered categorical's own order is ignored: SQL compares bytes."""
    import pyarrow as pa
    import pyarrow.compute as pc

    if isinstance(arr, pa.ChunkedArray):
        if pa.types.is_dictionary(arr.type) and arr.num_chunks > 1:
            arr = arr.cast(arr.type.value_type)          # chunks with different dictionaries: decode once
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    t = arr.type
    if pa.types.is_dictionary(t):
        if not is_string_type(t.value_type):
            raise NotImplementedError(f"dictionary column of {t.value_type}: only string dictionaries (VARCHAR) "
                                      "are supported")
    elif is_string_type(t):
        arr = pc.dictionary_encode(arr)
    else:
        raise NotImplementedError(f"column type {t} is not a string type")
    n = len(arr)
    idx = arr.indices.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64, copy=False)
    in_null = arr.is_null().to_numpy(zero_copy_only=False) if arr.null_count else None
    words = arr.dictionary
    used = np.zeros(len(words), dtype=bool)
    live = idx if in_null is None else idx[~in_null]
    used[live] = True
    used &= ~words.is_null().to_numpy(zero_copy_only=False)
    present = words.filter(pa.array(used))
    uniq = pc.unique(present.cast(pa.large_string()))
    uniq = uniq.take(pc.array_sort_indices(uniq))
    d = intern(Dictionary(uniq))
    remap = pc.index_in(words.cast(pa.large_string()), value_set=d.values)   # NULL entry / unused -> NULL
    remap_np = remap.fill_null(-1).to_numpy(zero_copy_only=False).astype(np.int64) if len(words) else \
        np.full(1, -1, dtype=np.int64)
    codes = remap_np[idx] if n else np.zeros(0, dtype=np.int64)
    null = codes < 0
    if in_null is not None:
        null |= in_null
    codes = np.where(null, 0, codes).astype(np.int64)
    return codes, (null if null.any() else None), Varchar(d)


def encode_into(arr, logical: Varchar):
    """A string / string-dictionary Arrow array whose values all occur in logical.dictionary ->
    (codes, NULL mask or None, logical): one row group of a lazy Parquet table.  Only the chunk's own
    distinct values are looked up (a binary search each in the sorted dictionary), then gathered by the
    chunk's indices: the cost follows the row group, not the size of the table's dictionary."""
    import pyarrow as pa
    import pyarrow.compute as pc
    if isinstance(arr, pa.ChunkedArray):
        if pa.types.is_dictionary(arr.type) and arr.num_chunks > 1:
            arr = arr.cast(arr.type.value_type)
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    if not pa.types.is_dictionary(arr.type):
        arr = pc.dictionary_encode(arr)
    words = arr.dictionary.to_pylist()
    table = logical.dictionary.sorted_objects()
    remap = np.full(max(len(words), 1), -1, dtype=np.int64)
    live = [i for i, w in enumerate(words) if w is not None]
    if live and len(table):
        keys = np.array([words[i] for i in live], dtype=object)
        pos = np.minimum(np.searchsorted(table, keys), len(table) - 1)
        hit = table[pos] == keys
        remap[np.array(live)[hit]] = pos[hit]
    idx = arr.indices.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64, copy=False)
    codes = remap[idx] if len(arr) else np.zeros(0, dtype=np.int64)
    null = codes < 0
    if arr.null_count:
        null |= arr.is_null().to_numpy(zero_copy_only=False)
    codes = np.where(null, 0, codes)
    return codes, (null if null.any() else None), logical


def stat_to_codes(d: Dictionary, lo, hi):
    """Parquet min / max statistics of a string column -> code bounds; a truncated min is <= the true
    minimum and a truncated max >= the true maximum, so the bounds stay conservative"""
    as_bytes = lambda v: v if isinstance(v, bytes) else str(v).encode("utf-8")     # noqa: E731
    return d.lower_bound(as_bytes(lo)), d.upper_bound(as_bytes(hi)) - 1


def encode_pandas(series):
    """pandas `category` Series with string categories -> (codes, NULL mask or None, Varchar)"""
    import pandas as pd
    import pyarrow as pa

    cats = series.cat.categories
    if len(cats) and not (pd.api.types.is_string_dtype(cats.dtype) and all(isinstance(c, str) for c in cats)):
        raise NotImplementedError(f"category column {series.name!r} has non-string categories ({cats.dtype}); "
                                  "only string categories are VARCHAR")
    codes = series.cat.codes.to_numpy()
    arr = pa.DictionaryArray.from_arrays(pa.array(codes, type=pa.int32(), mask=codes < 0),
                                         pa.array(list(cats), type=pa.large_string()))
    return encode_arrow(arr)


def plain_string_error(what) -> NotImplementedError:
    return NotImplementedError(
        f"column {what} holds plain strings, which are outside the int64/float64/bool hot path; register it as "
        "VARCHAR with series.astype('category') or create_table(..., dictionary=[column, ...])")


def check_distribution(distribution, schema):
    """Each rank would build its own dictionary from its own rows; only replicated data agrees."""
    if distribution in ("sharded", "root"):
        bad = [n for n, _, lg in schema if is_varchar(lg)]
        if bad:
            raise NotImplementedError(f"VARCHAR columns {bad} in a '{distribution}' table: every rank would hold a "
                                      "different dictionary; register the table as 'replicated' or 'local'")


# ---------------------------------------------------------------------------------------------
# output
# ---------------------------------------------------------------------------------------------
def to_host(codes: np.ndarray, null: Optional[np.ndarray], logical: Varchar):
    """codes -> pandas Categorical whose categories are the dictionary (NaN for NULL)"""
    import pandas as pd
    c = codes.astype(np.int64, copy=True)
    if null is not None:
        c[null] = -1
    return pd.Categorical.from_codes(c, dtype=pd.CategoricalDtype(logical.dictionary.categories()), validate=False)


# ---------------------------------------------------------------------------------------------
# predicates: literals -> int64 terms on the codes (host only)
# ---------------------------------------------------------------------------------------------
_FLIP = {"eq": "eq", "ne": "ne", "lt": "gt", "le": "ge", "gt": "lt", "ge": "le"}
_NO_CODE = -1      # no row holds it: `code = -1` is false for every non-NULL row and NULL for NULL rows


def _cmp(op, e, v):
    return Call(op, [e, Lit(int(v))], U8)


def _any_code(e):
    """true for every non-NULL code, NULL for a NULL row (so NOT of it stays NULL, as SQL asks)"""
    return _cmp("ge", e, 0)


def compare_literal(op: str, e: Expr, lit: str) -> Expr:
    """`e <op> 'lit'` for a VARCHAR expression e: one or two code terms, exact for present and absent
    literals because the dictionary is sorted."""
    d = dictionary_of(e)
    key = lit.encode("utf-8")
    if op in ("eq", "ne"):
        code = d.code_of(lit)
        if code is None:
            return _cmp("eq", e, _NO_CODE) if op == "eq" else _any_code(e)
        return _cmp(op, e, code)
    if op == "lt":
        return _cmp("lt", e, d.lower_bound(key))
    if op == "le":
        return _cmp("lt", e, d.upper_bound(key))
    if op == "gt":
        return _cmp("ge", e, d.upper_bound(key))
    if op == "ge":
        return _cmp("ge", e, d.lower_bound(key))
    raise NotImplementedError(f"operator {op} on VARCHAR")


def binop(op: str, a, b) -> Expr:
    """A comparison with at least one VARCHAR operand (expr.binop routes it here)."""
    if op not in _FLIP:
        raise NotImplementedError(f"operator {op} on VARCHAR: only comparisons, [NOT] LIKE / ILIKE and IN apply")
    if not is_varchar(a):
        a, b, op = b, a, _FLIP[op]
    if isinstance(b, str):
        return compare_literal(op, a, b)
    if b is None or (isinstance(b, Lit) and b.value is None):
        return Call(op, [a, Lit(None, I64)], U8)
    if not is_varchar(b):
        raise NotImplementedError(f"comparison of a VARCHAR with {getattr(b, 'logical', type(b).__name__)}")
    da, db = dictionary_of(a), dictionary_of(b)
    if same(da, db):
        return Call(op, [a, b], U8)
    # different dictionaries: 2 * code_a against b's lower bound in a's dictionary (odd when absent)
    two_a = Call("mul", [a, Lit(2)], I64)
    return Call(op, [two_a, map_codes(b, OrderTable(da, db))], U8)


# -- LIKE ------------------------------------------------------------------------------------
def like_tokens(pattern: str, escape: Optional[str]):
    """pattern -> [("%" | "_" | "lit", text)]: escaped characters are literals, and so is everything else"""
    out = []
    i = 0
    while i < len(pattern):
        ch = pattern[i]
        if escape is not None and ch == escape and i + 1 < len(pattern):
            out.append(("lit", pattern[i + 1]))
            i += 2
            continue
        out.append((ch, ch) if ch in "%_" else ("lit", ch))
        i += 1
    return out


def like_shape(pattern: str, escape: Optional[str]):
    """("eq", text) for a pattern without wildcards, ("prefix", p) for `p%...%`, else ("general", None)"""
    toks = like_tokens(pattern, escape)
    k = len(toks)
    while k and toks[k - 1][0] == "%":
        k -= 1
    head = toks[:k]
    if any(t != "lit" for t, _ in head):
        return "general", None
    text = "".join(v for _, v in head)
    return ("eq", text) if k == len(toks) else ("prefix", text)


def like_host(s: str, pattern: str, escape: Optional[str], ilike=False) -> bool:
    """The kernel's LIKE rule on one host string (constant folding)"""
    import re
    rx = "".join(".*" if t == "%" else "." if t == "_" else re.escape(v) for t, v in like_tokens(pattern, escape))
    return re.fullmatch(rx, s, re.DOTALL | ((re.IGNORECASE | re.ASCII) if ilike else 0)) is not None


def successor(key: bytes) -> bytes:
    """the least byte string greater than every string that starts with `key` (UTF-8 never holds 0xFF)"""
    return key[:-1] + bytes([key[-1] + 1])


def like(e: Expr, pattern: str, escape: Optional[str] = "\\", ilike=False) -> Expr:
    """`e [I]LIKE pattern`: code terms when the pattern is an equality or a prefix range, else a per-entry
    match table looked up per row (B2_OP_MAP)."""
    if escape is not None and len(escape) != 1:
        raise ValueError(f"ESCAPE takes one character, not {escape!r}")
    d = dictionary_of(e)
    if not ilike:
        kind, text = like_shape(pattern, escape)
        if kind == "eq":
            return compare_literal("eq", e, text)
        if kind == "prefix":
            if text == "":
                return _any_code(e)
            key = text.encode("utf-8")
            return Call("and", [_cmp("ge", e, d.lower_bound(key)), _cmp("lt", e, d.lower_bound(successor(key)))], U8)
    return map_codes(e, LikeTable(d, pattern, escape, ilike))


# ---------------------------------------------------------------------------------------------
# per-entry tables for B2_OP_MAP
# ---------------------------------------------------------------------------------------------
class MapTable:
    """A table indexed by the codes of one dictionary, computed on the device on first use.
    .column(device) -> DeviceColumn of len(self) entries; dtype is I64 or U8."""
    dtype = I64

    def __init__(self, n):
        self.n = n
        self._cols = {}

    def __len__(self):
        return self.n

    def column(self, dev):
        if dev.index not in self._cols:
            self._cols[dev.index] = self._compute(dev)
        return self._cols[dev.index]


class LikeTable(MapTable):
    dtype = U8

    def __init__(self, d: Dictionary, pattern: str, escape: Optional[str], ilike: bool):
        super().__init__(len(d))
        self.d, self.pattern, self.escape, self.ilike = d, pattern, escape, ilike

    def __repr__(self):
        return f"{'ilike' if self.ilike else 'like'}({self.pattern!r} escape {self.escape!r} on {self.d!r})"

    def _compute(self, dev):
        return like_table(self.d, self.pattern, self.escape, self.ilike, dev)


class MatchTable(MapTable):
    """code in dictionary `b` -> code of the same string in `a`, NULL when `a` lacks it"""

    def __init__(self, a: Dictionary, b: Dictionary):
        super().__init__(len(b))
        self.a, self.b = a, b

    def __repr__(self):
        return f"match({self.b!r} in {self.a!r})"

    def _compute(self, dev):
        return lower_bound_table(self.a, self.b, L.STR_LB_MATCH, dev)


class OrderTable(MatchTable):
    """code in `b` -> 2 * lower bound in `a` - (1 if absent): comparable with 2 * a's codes"""

    def __repr__(self):
        return f"order({self.b!r} in {self.a!r})"

    def _compute(self, dev):
        return lower_bound_table(self.a, self.b, L.STR_LB_ORDER, dev)


def map_codes(e: Expr, table: MapTable) -> Expr:
    return Call("map", [e], table.dtype, param=table)


def translate_key(e: Expr, into: Dictionary) -> Expr:
    """e's codes rewritten as codes of `into` (NULL where `into` lacks the string): a join key that meets
    a column of another dictionary"""
    return map_codes(e, MatchTable(into, dictionary_of(e)))


def join_keys(a: Expr, b: Expr, translate_a: bool):
    """Equi-join keys a = b with a VARCHAR on either side -> key expressions on one code space.  Equal
    dictionaries join on their codes; otherwise one side (a when translate_a) is translated into the
    other's dictionary, where a string the other side lacks becomes NULL and so matches nothing."""
    if not (is_varchar(a) and is_varchar(b)):
        raise NotImplementedError("a join of a VARCHAR key with a non-VARCHAR key")
    if same(dictionary_of(a), dictionary_of(b)):
        return a, b
    if translate_a:
        return translate_key(a, dictionary_of(b)), b
    return a, translate_key(b, dictionary_of(a))


# ---------------------------------------------------------------------------------------------
# device calls
# ---------------------------------------------------------------------------------------------
def like_table(d: Dictionary, pattern: str, escape: Optional[str], ilike: bool, dev):
    """b2_str_like over every entry of d -> DeviceColumn U8[len(d)]"""
    import torch
    from .device import DeviceColumn, ptr, stream_ptr
    off, chars = d.device(dev)
    pat = pattern.encode("utf-8")
    pbuf = torch.frombuffer(bytearray(pat or b"\0"), dtype=torch.uint8).to(dev)
    out = torch.empty(max(len(d), 1), dtype=torch.uint8, device=dev)
    esc = 0xFFFFFFFF if escape is None else ord(escape)
    L.str_like(ptr(off), ptr(chars), len(d), ptr(pbuf), len(pat), esc, L.STR_ILIKE if ilike else 0,
               ptr(out), stream_ptr())
    return DeviceColumn(out[: len(d)], None, U8)


def lower_bound_table(a: Dictionary, b: Dictionary, mode: int, dev):
    """b2_str_lower_bound of b's entries in a -> DeviceColumn I64[len(b)] (with validity for MATCH)"""
    import torch
    from .device import DeviceColumn, ptr, stream_ptr, bitmap_words
    ao, ac = a.device(dev)
    bo, bc = b.device(dev)
    out = torch.empty(max(len(b), 1), dtype=torch.int64, device=dev)
    valid = torch.empty(max(bitmap_words(len(b)), 1), dtype=torch.int32, device=dev) \
        if mode == L.STR_LB_MATCH else None
    L.str_lower_bound(ptr(ao), ptr(ac), len(a), ptr(bo), ptr(bc), len(b), mode, ptr(out), ptr(valid), stream_ptr())
    return DeviceColumn(out[: len(b)], valid, I64)

