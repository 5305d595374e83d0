"""Device-resident Arrow-layout columns and the Python face of the C-ABI kernels.

PyTorch is used only as plumbing: device memory (caching allocator), streams, and
torch.distributed.  All arithmetic on column data happens in libb200sql.so.
"""
import ctypes as C
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib as L
from . import strings as S
from . import temporal as T
from .expr import int_literal_is_exact

I64, F64, U8 = L.I64, L.F64, L.U8
_TORCH_DTYPE = {I64: torch.int64, F64: torch.float64, U8: torch.uint8}


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("dask_sql_b200 executes on a CUDA device (H100, sm_90a); no CPU fallback exists")


_stream = [None, None, None]


def cur_stream():
    """The current torch stream, looked up once per query.  torch.cuda.current_stream() walks through
    torch._utils._get_available_device_type() on every call (measured ~100 us per call in a
    torch.distributed job), and Event.record() / wait_event() call it when no stream is passed -- dozens
    of times per query.  Cached until reset_stream() (the executor calls that on entry to every query
    and before resolving a pending result); events are always recorded on an explicit stream."""
    s = _stream[1]
    if s is None:
        s = _stream[1] = torch.cuda.current_stream()
    return s


def stream_ptr():
    """The same stream as a C pointer for the C-ABI calls."""
    s = _stream[0]
    if s is None:
        s = _stream[0] = C.c_void_p(cur_stream().cuda_stream)
    return s


def cur_device():
    """torch.device of the current CUDA device, looked up once per query (see cur_stream)."""
    d = _stream[2]
    if d is None:
        require_cuda()
        d = _stream[2] = torch.device("cuda", torch.cuda.current_device())
    return d


def reset_stream():
    _stream[0] = _stream[1] = _stream[2] = None


def ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() > 0 else C.c_void_p(0)


def bitmap_words(n):
    return (n + 31) // 32


@dataclass
class Stats:
    """min/max over non-null values (python int / float), null count (bitmap NULLs + NaNs), and
    `repeat`: the share of sampled rows that have an equal value among the 31 rows next to them
    (0 for keys that rarely collide inside a warp, > 0.3 for Zipf(1.1))."""
    vmin: object
    vmax: object
    nulls: int
    repeat: float = 0.0


NARROW_HEADROOM = 1 << 30     # device bytes an image must leave free (DeviceColumn.star_image)


def narrow_base(stats: Stats, dtype) -> Optional[int]:
    """Base of the 32-bit frame-of-reference image of an int64 column with these statistics: its minimum when
    every non-NULL value lies in [vmin, vmin + 2^32), else None.  Exact: the range is taken in Python ints."""
    if dtype != I64 or stats.vmin is None:
        return None
    lo, hi = int(stats.vmin), int(stats.vmax)
    return lo if hi - lo < (1 << 32) else None


class DeviceColumn:
    """values buffer + optional Arrow validity bitmap (stored as int32 words) on one GPU."""

    __slots__ = ("data", "valid", "dtype", "logical", "n", "stats", "flags", "base", "_image")

    def __init__(self, data: torch.Tensor, valid: Optional[torch.Tensor], dtype: int, logical=None, stats=None):
        self.data = data
        self.valid = valid
        self.dtype = dtype
        self.logical = logical if logical is not None else {I64: "int64", F64: "float64", U8: "bool"}[dtype]
        self.n = int(data.shape[0])
        self.stats = stats
        self.flags = 0
        self.base = 0          # a B2_U32 image: the value of offset 0 (the star scans pass it beside the scan)
        self._image = None     # (data._version, what star_image returns) once decided

    @property
    def device(self):
        return self.data.device

    def as_struct(self) -> L.Col:
        c = L.Col()
        c.data = self.data.data_ptr() if self.n else 0
        c.valid = self.valid.data_ptr() if self.valid is not None and self.n else 0
        c.dtype = self.dtype
        c.flags = self.flags
        return c

    def nbytes(self):
        return self.data.numel() * self.data.element_size() + (0 if self.valid is None else self.valid.numel() * 4)

    def ensure_stats(self) -> Stats:
        if self.stats is None:
            self.stats = col_stats(self)
        return self.stats

    def star_image(self) -> "DeviceColumn":
        """What a star scan streams for this column: its 32-bit image when the column is int64 and its values
        span less than 2^32 (narrow_base; b2_narrow_image: uint32 offsets from `base`, 0 for a NULL row, this
        column's bitmap), else the column itself.  4 bytes per row instead of 8 in the scans, 4 more per row of
        HBM while the image is kept.  Made on first use, on the current stream, unless the device would be left
        with less than NARROW_HEADROOM free; kept with the column and made again, from fresh statistics, once a
        write to the values moves the tensor's version counter.  B200SQL_NO_NARROW=1: always the column."""
        if self.dtype != I64 or self.n == 0 or os.environ.get("B200SQL_NO_NARROW") == "1":
            return self
        version = self.data._version
        if self._image is not None:
            if self._image[0] == version:
                return self._image[1]
            self.stats = None              # they describe the values the old image was made of
        base = narrow_base(self.ensure_stats(), self.dtype)
        img = self
        if base is not None and torch.cuda.mem_get_info(self.device)[0] >= 4 * self.n + NARROW_HEADROOM:
            out = torch.empty(self.n, dtype=torch.int32, device=self.device)
            st = self.as_struct()
            L.narrow_image(C.byref(st), self.n, base, ptr(out), stream_ptr())
            img = DeviceColumn(out, self.valid, L.U32, self.logical)
            img.base = base
        self._image = (version, img)
        return img

    def slice(self, lo, hi):
        """Row-range view.  Only valid for lo % 32 == 0 when the column has a validity bitmap."""
        v = None
        if self.valid is not None:
            assert lo % 32 == 0
            v = self.valid[lo // 32: (hi + 31) // 32]
        return DeviceColumn(self.data[lo:hi], v, self.dtype, self.logical)


# ---------------------------------------------------------------------------------------------
# host <-> device
# ---------------------------------------------------------------------------------------------
def _pack_valid(mask_null: np.ndarray) -> np.ndarray:
    n = mask_null.shape[0]
    bits = np.packbits(~mask_null, bitorder="little")
    out = np.zeros(bitmap_words(n) * 4, dtype=np.uint8)
    out[: bits.shape[0]] = bits
    return out.view(np.int32)


def column_from_host(values, device, pin=False) -> DeviceColumn:
    """pandas Series / numpy array -> DeviceColumn (PandasLikeInputPlugin.to_dc,
    input_utils/pandaslike.py:18-38, is where host columns enter in the reference)."""
    import pandas as pd

    logical = str(getattr(values, "dtype", "float64"))
    mask = None
    if isinstance(values, pd.Series):
        arr = values.array
        if isinstance(arr, pd.arrays.BooleanArray):
            mask, vals = np.asarray(arr._mask), np.asarray(arr._data).astype(np.uint8)
        elif isinstance(arr, (pd.arrays.IntegerArray, pd.arrays.FloatingArray)):
            mask, vals = np.asarray(arr._mask), np.asarray(arr._data)
        else:
            vals = values.to_numpy()
    else:
        vals = np.asarray(values)
    kind = vals.dtype.kind
    if kind == "M":               # DATE / TIMESTAMP: int64 ticks of the input's own unit, NaT -> NULL
        vals, mask, logical = T.from_host_array(vals)
        dt = I64
    elif kind == "b":
        vals, dt = vals.astype(np.uint8), U8
    elif kind == "i" or (kind == "u" and vals.dtype.itemsize < 8):
        vals, dt = vals.astype(np.int64, copy=False), I64
    elif kind == "u" and logical in ("uint8",) and mask is not None:
        vals, dt = vals.astype(np.int64), I64
    elif kind == "f":
        vals, dt = vals.astype(np.float64, copy=False), F64
    else:
        raise NotImplementedError(
            f"column dtype {logical} is outside the int64/float64/bool hot path of this layer")
    vals = np.ascontiguousarray(vals)
    t = torch.from_numpy(vals)
    if pin:
        t = t.pin_memory()
    data = t.to(device, non_blocking=pin)
    valid = None
    if mask is not None and mask.any():
        valid = torch.from_numpy(_pack_valid(mask)).to(device)
    return DeviceColumn(data, valid, dt, logical)


def column_to_host(col: DeviceColumn):
    """DeviceColumn -> pandas array preserving the logical dtype (D2H)."""
    import pandas as pd

    vals = col.data.cpu().numpy()
    mask = None
    if col.valid is not None:
        bits = col.valid.cpu().numpy().view(np.uint8)
        mask = ~np.unpackbits(bits, bitorder="little")[: col.n].astype(bool)
        if not mask.any():
            mask = None
    lg = col.logical
    if S.is_varchar(lg):
        return S.to_host(vals, mask, lg)
    unit = T.unit_of(lg)
    if unit is not None:
        return T.to_host_array(vals, unit, mask)
    if col.dtype == U8:
        vals = vals.astype(bool)
        if mask is not None or lg == "boolean":
            return pd.array(np.where(mask, False, vals) if mask is not None else vals, dtype="boolean") \
                if mask is None else pd.arrays.BooleanArray(vals, mask)
        return vals
    if col.dtype == F64:
        if mask is not None:
            vals = vals.copy()
            vals[mask] = np.nan
        if lg.startswith("Float"):
            return pd.arrays.FloatingArray(vals, np.isnan(vals))
        if lg == "float32":
            return vals.astype(np.float32)
        return vals
    # integers
    if lg[0] in "IU" and lg != "int64":  # pandas nullable extension dtype (Int64, Int8, UInt8 ...)
        np_dt = np.dtype(lg.lower())
        return pd.arrays.IntegerArray(vals.astype(np_dt), mask if mask is not None else np.zeros(col.n, bool))
    if mask is not None:
        # numpy ints cannot hold NULL: pandas promotes to float64 + NaN (sum(min_count=1) on an
        # all-NULL group, outer-join fill), and so do we.
        out = vals.astype(np.float64)
        out[mask] = np.nan
        return out
    if lg.startswith(("int", "uint")) and lg != "int64":
        return vals.astype(np.dtype(lg))
    return vals


# ---------------------------------------------------------------------------------------------
# scan descriptors
# ---------------------------------------------------------------------------------------------
@dataclass
class TermSpec:
    col: int
    op: int
    lit: object = 0


def make_scan(cols: Sequence[DeviceColumn], terms: Sequence[TermSpec], n: Optional[int] = None) -> L.Scan:
    if len(cols) > L.MAX_COLS:
        raise ValueError(f"a fused scan reads at most {L.MAX_COLS} columns")
    if len(terms) > L.MAX_TERMS:
        raise ValueError(f"a fused scan evaluates at most {L.MAX_TERMS} predicate terms")
    s = L.Scan()
    s.ncols = len(cols)
    s.nterms = len(terms)
    s.n = int(n if n is not None else (cols[0].n if cols else 0))
    for i, c in enumerate(cols):
        s.cols[i] = c.as_struct()
    for i, t in enumerate(terms):
        tm = s.terms[i]
        tm.col, tm.op = t.col, t.op
        cd = cols[t.col].dtype
        lit = t.lit
        if t.op in (L.IS_NULL, L.IS_NOT_NULL, L.IS_TRUE):
            continue
        if cd == F64:
            tm.lit_f = float(lit)
        elif isinstance(lit, (float, np.floating)) and not int_literal_is_exact(float(lit)):
            tm.as_f64, tm.lit_f = 1, float(lit)     # compares in float64, see expr.F64_EXACT_INT
        else:
            tm.lit_i = int(lit)
    return s


def make_aggs(specs):
    arr = (L.Agg * max(1, len(specs)))()
    for i, (col, op) in enumerate(specs):
        arr[i].col, arr[i].op = col, op
    return arr


# ---------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------
_ws_cache = {}


def _workspace(device, nbytes):
    key = (device.index, cur_stream().cuda_stream)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = ws
    return ws


def col_stats(col: DeviceColumn) -> Stats:
    reset_stream()          # a blocking call anyway: also the point where table loading picks up the stream
    out = torch.empty(6, dtype=torch.int64, device=col.device)
    ws = _workspace(col.device, L.stats_ws_bytes())
    st = col.as_struct()
    L.col_stats(C.byref(st), col.n, ptr(out), ptr(ws), stream_ptr())
    mn, mx, nulls, nans, rep, sampled = out.cpu().tolist()
    repeat = rep / sampled if sampled else 0.0
    if mn == (1 << 63) - 1 and mx == -(1 << 63):
        return Stats(None, None, nulls + nans, repeat)
    if col.dtype == F64:
        mn = np.int64(mn).view(np.float64).item()
        mx = np.int64(mx).view(np.float64).item()
    return Stats(mn, mx, nulls + nans, repeat)


def expr_eval(prog: L.Prog, cols: Sequence[DeviceColumn], n: int, want_valid: bool, out=None,
              row_base: Optional[int] = None) -> DeviceColumn:
    """row_base: the base-table number of row 0, which the B2_OP_RAND_* draws are keyed on (None: the
    program draws nothing, and runs through b2_expr_eval)"""
    dev = cols[0].device if cols else cur_device()
    if out is None:
        out = torch.empty(n, dtype=_TORCH_DTYPE[prog.out_dtype], device=dev)
    valid = torch.empty(bitmap_words(n), dtype=torch.int32, device=dev) if want_valid else None
    arr = (L.Col * max(1, len(cols)))()
    for i, c in enumerate(cols):
        arr[i] = c.as_struct()
    if row_base is None:
        L.expr_eval(C.byref(prog), arr, len(cols), n, ptr(out), ptr(valid), stream_ptr())
    else:
        L.expr_eval_rows(C.byref(prog), arr, len(cols), n, row_base, ptr(out), ptr(valid), stream_ptr())
    return DeviceColumn(out, valid, prog.out_dtype)


class GlobalAgg:
    """Accumulates SELECT <aggs> FROM t WHERE ... over any number of partitions."""

    def __init__(self, device, agg_specs):
        self.specs = list(agg_specs)
        self.aggs = make_aggs(self.specs)
        k = max(1, len(self.specs))
        self.acc = torch.zeros(k, dtype=torch.int64, device=device)
        self.cnt = torch.zeros(k, dtype=torch.int64, device=device)
        self.first = True
        self.device = device

    def update(self, scan: L.Scan):
        ws = _workspace(self.device, L.scan_agg_ws_bytes())
        L.scan_agg(C.byref(scan), self.aggs, len(self.specs), ptr(self.acc), ptr(self.cnt),
                   0 if self.first else 1, ptr(ws), stream_ptr())
        self.first = False

    def result(self):
        """-> (acc raw int64 numpy, cnt numpy); float results are the int64 bit pattern."""
        if self.first:  # no partition seen: identities
            raise RuntimeError("GlobalAgg.result() before any update")
        return self.acc.cpu().numpy(), self.cnt.cpu().numpy()


def select(scan: L.Scan, device, gather_cols: Sequence[int] = (), want_idx=True, cols: Sequence[DeviceColumn] = ()):
    """Order-preserving selection of one partition -> (idx int32 tensor or None, [DeviceColumn])."""
    n = scan.n
    ntiles = L.num_tiles(n)
    tile_off = torch.empty(ntiles + 1, dtype=torch.int64, device=device)
    L.select_count(C.byref(scan), ptr(tile_off), stream_ptr())
    total = int(tile_off[ntiles].item())
    idx = torch.empty(total, dtype=torch.int32, device=device) if want_idx else None
    outs, ovalid = [], []
    for g in gather_cols:
        c = cols[g]
        outs.append(torch.empty(total, dtype=_TORCH_DTYPE[c.dtype], device=device))
        ovalid.append(torch.zeros(bitmap_words(total), dtype=torch.int32, device=device) if c.valid is not None else None)
    k = len(gather_cols)
    if total > 0:
        gc = (C.c_int32 * max(1, k))(*gather_cols)
        od = (C.c_void_p * max(1, k))(*[o.data_ptr() for o in outs])
        ov = (C.c_void_p * max(1, k))(*[(v.data_ptr() if v is not None else 0) for v in ovalid])
        L.select_write(C.byref(scan), ptr(tile_off), ptr(idx), k, gc, od, ov, stream_ptr())
    res = [DeviceColumn(o, v, cols[g].dtype, cols[g].logical) for o, v, g in zip(outs, ovalid, gather_cols)]
    return idx, res, total


trace = None      # optional [(label, cuda event)] recorded around the two launches of select_launch (diagnostics)


def _mark(label):
    if trace is not None:
        e = torch.cuda.Event(enable_timing=True)
        e.record(cur_stream())
        trace.append((label, e))


def select_launch(scan: L.Scan, device, gather_cols: Sequence[int], cols: Sequence[DeviceColumn]):
    """select() without the host round trip: outputs are allocated at their upper bound (scan.n rows),
    count and write kernels are both enqueued, and the count stays on the device.  Only for inputs
    without validity bitmaps.  -> ([output tensors of scan.n rows], 1-element int64 count tensor)"""
    n = scan.n
    ntiles = L.num_tiles(n)
    tile_off = torch.empty(ntiles + 1, dtype=torch.int64, device=device)
    _mark("select:begin")
    L.select_count(C.byref(scan), ptr(tile_off), stream_ptr())
    _mark("select:counted")
    outs = [torch.empty(n, dtype=_TORCH_DTYPE[cols[g].dtype], device=device) for g in gather_cols]
    k = len(gather_cols)
    gc = (C.c_int32 * max(1, k))(*gather_cols)
    od = (C.c_void_p * max(1, k))(*[o.data_ptr() for o in outs])
    ov = (C.c_void_p * max(1, k))(*[0] * k)
    if n > 0:
        L.select_write(C.byref(scan), ptr(tile_off), C.c_void_p(0), k, gc, od, ov, stream_ptr())
    _mark("select:written")
    return outs, tile_off[ntiles:ntiles + 1]


def gather(col: DeviceColumn, idx: torch.Tensor, nullable: bool) -> DeviceColumn:
    n = int(idx.shape[0])
    out = torch.empty(n, dtype=_TORCH_DTYPE[col.dtype], device=col.device)
    valid = torch.empty(bitmap_words(n), dtype=torch.int32, device=col.device) if (nullable or col.valid is not None) else None
    st = col.as_struct()
    L.gather(C.byref(st), ptr(idx), n, ptr(out), ptr(valid), stream_ptr())
    return DeviceColumn(out, valid, col.dtype, col.logical)


def _pow2_at_least(x):
    p = 1
    while p < x:
        p <<= 1
    return p


class GroupTable:
    """Caller-owned accumulator arrays of one group-by (dense / hash1 / hashk)."""

    def __init__(self, device, nslots, agg_specs, agg_dtypes, need_cnt, need_rows, need_present, indicator=None,
                 alloc=None, new=None):
        """alloc: number of slots to allocate (>= nslots; the kernels only ever touch the first nslots).
        A table whose partial results are reduce-scattered over the ranks is padded to a multiple of
        32 x world size so that every rank's slice -- and its share of a presence bitmap -- is aligned.

        indicator: index of a float SUM accumulator whose input is never NULL.  It starts at -0.0
        instead of +0.0; the kernels add x + 0.0 (never -0.0), so a slot still holding the -0.0 bit
        pattern (= INT64_MIN = EMPTY_KEY) received no row.  That makes the accumulator itself the
        "group exists" flag and saves the per-row presence-bitmap lookup (an L1 wavefront per row on
        a path whose bound is the SM's load/store issue rate).

        new: optional allocator `new(n, torch dtype, fill value) -> tensor` for the arrays (a prepared
        multi-GPU query places them in symmetric memory so that peers can read them over NVLink)."""
        self.fills = []      # (array, initial value) of every array: what reset() restores

        def make(n, dtype, fill):
            t = torch.full((n,), fill, dtype=dtype, device=device) if new is None else new(n, dtype, fill)
            self.fills.append((t, fill))
            return t

        self.device, self.nslots = device, nslots
        self.alloc = alloc = max(int(alloc or nslots), nslots)
        self.indicator = indicator
        self.specs = list(agg_specs)
        self.aggs = make_aggs(self.specs)
        self.state = L.AggState()
        self.acc: List[Optional[torch.Tensor]] = []
        self.cnt: List[Optional[torch.Tensor]] = []
        for a, ((col, op), dt) in enumerate(zip(self.specs, agg_dtypes)):
            acc = cnt = None
            if col >= 0 and op != L.AGG_COUNT:
                if op == L.AGG_SUMF or (op == L.AGG_SUM and dt == F64):
                    acc = make(alloc, torch.float64, -0.0 if a == indicator else 0.0)
                else:
                    acc = make(alloc, torch.int64, L.agg_identity(op))
            if col >= 0 and (op == L.AGG_COUNT or need_cnt[a]):
                cnt = make(alloc, torch.int64, 0)
            self.acc.append(acc)
            self.cnt.append(cnt)
            self.state.acc[a] = acc.data_ptr() if acc is not None else 0
            self.state.cnt[a] = cnt.data_ptr() if cnt is not None else 0
        self.rows = make(alloc, torch.int64, 0) if need_rows else None
        need_present = need_present and indicator is None
        self.present = make(bitmap_words(alloc), torch.int32, 0) if need_present else None
        self.state.rows = self.rows.data_ptr() if self.rows is not None else 0
        self.state.present = self.present.data_ptr() if self.present is not None else 0

    def reset(self):
        """Every array back to its initial value (an empty table), in stream order: a table reused run
        after run is refilled, not re-allocated."""
        for t, fill in self.fills:
            t.fill_(fill)


def groupby_dense(scan, key_col, kmin, table: GroupTable, skew=None, hot=None):
    """skew: None = one atomic per row; "warp" = per-warp match/shuffle pre-aggregation + per-CTA table
    (b2_groupby_dense_grouped); "hot" = thread-private partials for the heavy hitters listed in `hot`
    (int32[32] device tensor from hot_slots(); b2_groupby_dense_hot)."""
    args = (C.byref(scan), key_col, int(kmin), table.nslots, table.aggs, len(table.specs), C.byref(table.state))
    if skew == "hot" and hot is not None:
        L.groupby_dense_hot(*args, ptr(hot), stream_ptr())
    elif skew == "warp":
        L.groupby_dense_grouped(*args, stream_ptr())
    else:
        L.groupby_dense(*args, stream_ptr())


def hot_slots(key: DeviceColumn, kmin, nslots) -> torch.Tensor:
    """int32[32]: the heavy hitters of a dense key column (sampled), -1 padded."""
    out = torch.empty(32, dtype=torch.int32, device=key.device)
    st = key.as_struct()
    L.hot_slots(C.byref(st), key.n, int(kmin), int(nslots), ptr(out), stream_ptr())
    return out


def new_flags(device):
    return torch.zeros(4, dtype=torch.int32, device=device)


def groupby_hash1(scan, key_col, table_keys, cap, table: GroupTable, flags):
    L.groupby_hash1(C.byref(scan), key_col, ptr(table_keys), cap, table.aggs, len(table.specs),
                    C.byref(table.state), ptr(flags), stream_ptr())


def groupby_hashk(scan, key_cols, table_keys, table_nulls, table_state, cap, table: GroupTable, flags):
    kc = (C.c_int32 * len(key_cols))(*key_cols)
    L.groupby_hashk(C.byref(scan), kc, len(key_cols), ptr(table_keys), ptr(table_nulls), ptr(table_state), cap,
                    table.aggs, len(table.specs), C.byref(table.state), ptr(flags), stream_ptr())


class JoinTable:
    """Build side of a hash join (chained or direct-address); keeps its tensors alive."""

    def __init__(self, keys: Sequence[DeviceColumn], allow_dense=True):
        self.keys = list(keys)
        n = self.keys[0].n
        dev = self.keys[0].device
        self.n = n
        self.struct = L.JoinTable()
        self.struct.nkeys = len(keys)
        for i, k in enumerate(self.keys):
            self.struct.keys[i] = k.as_struct()
        self.dense = False
        self.unique = False
        if allow_dense and len(keys) == 1 and keys[0].dtype == I64 and n > 0:
            st = keys[0].ensure_stats()
            if st.vmin is not None:
                rng = st.vmax - st.vmin + 1
                if rng <= max(4 * n, 1 << 16) and rng < (1 << 31):
                    lookup = torch.full((rng,), -1, dtype=torch.int32, device=dev)
                    flags = new_flags(dev)
                    ks = keys[0].as_struct()
                    L.join_build_dense(C.byref(ks), n, st.vmin, rng, ptr(lookup), ptr(flags), stream_ptr())
                    if int(flags[0].item()) == 0:
                        self.dense, self.unique = True, True
                        self.lookup = lookup
                        self.struct.dense, self.struct.lookup = 1, lookup.data_ptr()
                        self.struct.kmin, self.struct.range = st.vmin, rng
                        return
        cap = _pow2_at_least(max(2 * n, 64))
        self.head = torch.full((cap,), -1, dtype=torch.int32, device=dev)
        self.next = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        arr = (L.Col * len(keys))(*[k.as_struct() for k in keys])
        L.join_build(arr, len(keys), n, ptr(self.head), ptr(self.next), cap, stream_ptr())
        self.struct.dense, self.struct.head, self.struct.next, self.struct.cap = 0, self.head.data_ptr(), self.next.data_ptr(), cap

    def key_layout(self, cols: Sequence[DeviceColumn]):
        """Re-lay build-side columns of a unique dense-key table in key order (b2_join_key_layout):
        the probe then fetches a payload with one random access at key-kmin, the int32 row lookup
        shrinks to a presence bitmap, and int64 payloads with a 32-bit value range are stored as
        uint32 offsets (half the L2 footprint).  After this the table matches by key offset
        (struct.dense == 2) and only join_probe_gather may be used with it."""
        assert self.dense and self.struct.dense == 1
        dev, kmin, rng, n = self.keys[0].device, self.struct.kmin, self.struct.range, self.n
        ks = self.keys[0].as_struct()
        present = torch.zeros(bitmap_words(rng), dtype=torch.int32, device=dev)
        store = {L.U32: torch.int32, I64: torch.int64, F64: torch.float64, U8: torch.uint8}
        self.keyed_cols, self.keyed_base = [], []
        first = True
        for c in cols:
            out_dtype, base = c.dtype, 0
            if c.dtype == I64:
                st = c.ensure_stats()
                if st.vmin is not None and st.vmax - st.vmin < (1 << 32):
                    out_dtype, base = L.U32, int(st.vmin)
            # a narrowed payload whose offsets leave 0xFFFFFFFF free marks absent keys itself (B2_COL_SENTINEL):
            # the streaming probe and b2_join_agg then skip the presence bitmap (one random access per row)
            sentinel = out_dtype == L.U32 and c.valid is None and st.vmax - st.vmin < (1 << 32) - 1
            if sentinel:
                out = torch.full((rng,), -1, dtype=torch.int32, device=dev)
            else:
                out = torch.empty(rng, dtype=store[out_dtype], device=dev)     # only present offsets are read
            ovalid = torch.zeros(bitmap_words(rng), dtype=torch.int32, device=dev) if c.valid is not None else None
            cs = c.as_struct()
            L.join_key_layout(C.byref(ks), n, kmin, rng, C.byref(cs), out_dtype, base, ptr(out), ptr(ovalid),
                              ptr(present) if first else None, stream_ptr())
            first = False
            kc = DeviceColumn(out, ovalid, out_dtype, c.logical)
            kc.flags = L.COL_SENTINEL if sentinel else 0
            self.keyed_cols.append(kc)
            self.keyed_base.append(base)
        if first:
            L.join_key_layout(C.byref(ks), n, kmin, rng, None, 0, 0, None, None, ptr(present), stream_ptr())
        self.present = present
        self.lookup = None
        self.struct.dense, self.struct.lookup = 2, present.data_ptr()


def join_probe_gather(scan, probe_keys, jt: JoinTable, mode, device, scan_cols, probe_gather, build_cols,
                      build_nullable, build_matched=None):
    """Probe and gather in one pass.  probe_gather: slots of scan columns to copy; build_cols: build-side
    DeviceColumns to fetch by build row.  -> (probe outputs, build outputs, total)."""
    n = scan.n
    ntiles = L.num_tiles(n)
    tile_off = torch.empty(ntiles + 1, dtype=torch.int64, device=device)
    pk = (C.c_int32 * len(probe_keys))(*probe_keys)
    L.join_count(C.byref(scan), pk, C.byref(jt.struct), mode, ptr(tile_off), stream_ptr())
    total = int(tile_off[ntiles].item())
    if total >= (1 << 31):
        raise NotImplementedError("join output of one partition exceeds 2^31 rows; use more partitions")
    pouts, pvalid, bouts, bvalid = [], [], [], []
    for sl in probe_gather:
        c = scan_cols[sl]
        pouts.append(torch.empty(total, dtype=_TORCH_DTYPE[c.dtype], device=device))
        pvalid.append(torch.zeros(bitmap_words(total), dtype=torch.int32, device=device) if c.valid is not None else None)
    for c in build_cols:
        bouts.append(torch.empty(total, dtype=_TORCH_DTYPE[c.dtype], device=device))
        bvalid.append(torch.zeros(bitmap_words(total), dtype=torch.int32, device=device)
                      if (c.valid is not None or build_nullable) else None)
    if total > 0:
        np_, nb = len(probe_gather), len(build_cols)
        pc = (C.c_int32 * max(1, np_))(*probe_gather)
        po = (C.c_void_p * max(1, np_))(*[t.data_ptr() for t in pouts])
        pv = (C.c_void_p * max(1, np_))(*[(v.data_ptr() if v is not None else 0) for v in pvalid])
        bo = (C.c_void_p * max(1, nb))(*[t.data_ptr() for t in bouts])
        bv = (C.c_void_p * max(1, nb))(*[(v.data_ptr() if v is not None else 0) for v in bvalid])
        if jt.struct.dense == 2:
            assert len(jt.keyed_cols) == nb and build_matched is None
            bc = (L.Col * max(1, nb))(*[c.as_struct() for c in jt.keyed_cols])
            bb = (C.c_int64 * max(1, nb))(*jt.keyed_base)
            L.join_write_gather_keyed(C.byref(scan), pk, C.byref(jt.struct), mode, ptr(tile_off), None, None,
                                      None, np_, pc, po, pv, nb, bc, bb, bo, bv, stream_ptr())
        else:
            bc = (L.Col * max(1, nb))(*[c.as_struct() for c in build_cols])
            L.join_write_gather(C.byref(scan), pk, C.byref(jt.struct), mode, ptr(tile_off), None, None,
                                ptr(build_matched), np_, pc, po, pv, nb, bc, bo, bv, stream_ptr())
    pres = [DeviceColumn(o, v, scan_cols[sl].dtype, scan_cols[sl].logical)
            for o, v, sl in zip(pouts, pvalid, probe_gather)]
    bres = [DeviceColumn(o, v, c.dtype, c.logical) for o, v, c in zip(bouts, bvalid, build_cols)]
    return pres, bres, total


def join_probe_onepass(scan, probe_keys, jt: JoinTable, mode, device, scan_cols, probe_gather, build_cols,
                       build_nullable):
    """join_probe_gather for direct-address tables without the counting pass and without the host
    round trip: one kernel (b2_join_onepass: each warp batch or tile reserves its output range with
    an atomic, so rows come in probe order within a batch and in unspecified order across batches),
    outputs allocated at their upper bound (one row per probe row), the row count stays on the device.
    -> (trim, 1-element int64 count tensor); `trim(total)` slices the probe and build outputs."""
    assert jt.dense
    n = scan.n
    total = torch.zeros(1, dtype=torch.int64, device=device)
    pk = (C.c_int32 * len(probe_keys))(*probe_keys)
    pouts, pvalid, bouts, bvalid = [], [], [], []
    for sl in probe_gather:
        c = scan_cols[sl]
        pouts.append(torch.empty(n, dtype=_TORCH_DTYPE[c.dtype], device=device))
        pvalid.append(torch.zeros(bitmap_words(n), dtype=torch.int32, device=device) if c.valid is not None else None)
    for c in build_cols:
        bouts.append(torch.empty(n, dtype=_TORCH_DTYPE[c.dtype], device=device))
        bvalid.append(torch.zeros(bitmap_words(n), dtype=torch.int32, device=device)
                      if (c.valid is not None or build_nullable) else None)
    np_, nb = len(probe_gather), len(build_cols)
    pc = (C.c_int32 * max(1, np_))(*probe_gather)
    po = (C.c_void_p * max(1, np_))(*[t.data_ptr() for t in pouts])
    pv = (C.c_void_p * max(1, np_))(*[(v.data_ptr() if v is not None else 0) for v in pvalid])
    bo = (C.c_void_p * max(1, nb))(*[t.data_ptr() for t in bouts])
    bv = (C.c_void_p * max(1, nb))(*[(v.data_ptr() if v is not None else 0) for v in bvalid])
    if jt.struct.dense == 2:
        assert len(jt.keyed_cols) == nb
        bc = (L.Col * max(1, nb))(*[c.as_struct() for c in jt.keyed_cols])
        bb = (C.c_int64 * max(1, nb))(*jt.keyed_base)
    else:
        bc = (L.Col * max(1, nb))(*[c.as_struct() for c in build_cols])
        bb = None
    L.join_onepass(C.byref(scan), pk, C.byref(jt.struct), mode, ptr(total), np_, pc, po, pv, nb, bc, bb, bo, bv,
                   stream_ptr())

    def trim(total):
        w = bitmap_words(total)
        pres = [DeviceColumn(o[:total], v[:w] if v is not None else None, scan_cols[sl].dtype, scan_cols[sl].logical)
                for o, v, sl in zip(pouts, pvalid, probe_gather)]
        bres = [DeviceColumn(o[:total], v[:w] if v is not None else None, c.dtype, c.logical)
                for o, v, c in zip(bouts, bvalid, build_cols)]
        return pres, bres

    return trim, total


def join_probe(scan, probe_keys, jt: JoinTable, mode, device, build_matched=None):
    """-> (probe_idx int32, build_idx int32 or None, total)."""
    assert jt.struct.dense != 2, "a key-ordered table yields key offsets, not build rows"
    n = scan.n
    ntiles = L.num_tiles(n)
    tile_off = torch.empty(ntiles + 1, dtype=torch.int64, device=device)
    pk = (C.c_int32 * len(probe_keys))(*probe_keys)
    L.join_count(C.byref(scan), pk, C.byref(jt.struct), mode, ptr(tile_off), stream_ptr())
    total = int(tile_off[ntiles].item())
    if total >= (1 << 31):
        raise NotImplementedError("join output of one partition exceeds 2^31 rows; use more partitions")
    pidx = torch.empty(total, dtype=torch.int32, device=device)
    bidx = torch.empty(total, dtype=torch.int32, device=device)
    if total > 0:
        L.join_write(C.byref(scan), pk, C.byref(jt.struct), mode, ptr(tile_off), ptr(pidx), ptr(bidx),
                     ptr(build_matched), stream_ptr())
    return pidx, bidx, total


def join_mark(scan, probe_keys, jt: JoinTable, terms, flags, device) -> DeviceColumn:
    """The three-valued mark of an IN / EXISTS subquery over the rows of `scan` (b2_join_mark).
    terms: [(probe slot, build DeviceColumn, B2 comparison)] -> a B2_U8 column with validity."""
    n = scan.n
    out = torch.empty(max(n, 1), dtype=torch.uint8, device=device)[:n]
    valid = torch.empty(bitmap_words(n), dtype=torch.int32, device=device)
    pk = (C.c_int32 * len(probe_keys))(*probe_keys)
    mt = (L.MarkTerm * max(1, len(terms)))()
    for i, (slot, col, cmp) in enumerate(terms):
        mt[i].probe_col, mt[i].build, mt[i].cmp = slot, col.as_struct(), cmp
    L.join_mark(C.byref(scan), pk, C.byref(jt.struct), mt, len(terms), flags, ptr(out), ptr(valid), stream_ptr())
    return DeviceColumn(out, valid, U8)
