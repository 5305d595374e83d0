"""Device tables: the registered relations behind Context.create_table.

A table is a list of partitions; a partition maps column name -> DeviceColumn (HBM-resident,
`persist=True`) or HostColumn (pinned host memory, streamed to the GPU per query, the
counterpart of dask's lazy partitions when `persist=False`, input_utils/convert.py:70-71).
In a multi-rank job (one process per GPU) every rank holds its own shard of a `sharded`
table; `replicated` tables hold the same rows on every rank; `root` tables hold rows on rank 0
only and are broadcast over NCCL when a join needs them as its build side.
"""
from typing import Dict, List, Optional

import numpy as np
import torch

from . import temporal as T
from .device import DeviceColumn, Stats, column_from_host, I64, F64, U8, _pack_valid


class HostColumn:
    """Pinned host copy of a column; .to_device() issues the (async) H2D copy."""

    __slots__ = ("data", "valid", "dtype", "logical", "n", "stats")

    def __init__(self, data: torch.Tensor, valid: Optional[torch.Tensor], dtype, logical):
        self.data, self.valid, self.dtype, self.logical = data, valid, dtype, logical
        self.n = int(data.shape[0])
        self.stats = None

    def to_device(self, device) -> DeviceColumn:
        d = self.data.to(device, non_blocking=True)
        v = self.valid.to(device, non_blocking=True) if self.valid is not None else None
        col = DeviceColumn(d, v, self.dtype, self.logical, self.stats)
        return col

    def nbytes(self):
        return self.data.numel() * self.data.element_size() + (0 if self.valid is None else self.valid.numel() * 4)


class ArrowColumn:
    """One column of a pyarrow.Table as plain buffers: widened values + Arrow validity bytes.

    Arrow's validity bitmap is LSB-ordered, one bit per row -- exactly the device layout -- so the
    bytes are used as they are (no unpack / repack, no pandas object in between); slices at
    multiples of 8 rows (partitions start at multiples of 32) are views."""

    __slots__ = ("values", "valid_bytes", "logical")

    def __init__(self, values: np.ndarray, valid_bytes: Optional[np.ndarray], logical: str):
        self.values, self.valid_bytes, self.logical = values, valid_bytes, logical

    def __len__(self):
        return int(self.values.shape[0])

    def __getitem__(self, sl: slice):
        lo, hi, _ = sl.indices(len(self))
        vb = None
        if self.valid_bytes is not None:
            assert lo % 8 == 0
            vb = self.valid_bytes[lo // 8: (hi + 7) // 8]
        return ArrowColumn(self.values[lo:hi], vb, self.logical)

    def valid_words(self) -> Optional[np.ndarray]:
        """int32 validity words of this slice, or None when nothing is NULL."""
        if self.valid_bytes is None:
            return None
        n = len(self)
        nbytes = (n + 7) // 8
        out = np.zeros(((n + 31) // 32) * 4, dtype=np.uint8)
        out[:nbytes] = self.valid_bytes[:nbytes]
        if n % 8:
            out[nbytes - 1] &= (1 << (n % 8)) - 1          # bits past the end belong to nobody
        bits_set = int(np.unpackbits(out[:nbytes], bitorder="little")[:n].sum()) if n else 0
        return None if bits_set == n else out.view(np.int32)


def _arrow_array_to_column(arr) -> ArrowColumn:
    import pyarrow as pa

    t = arr.type
    n = len(arr)
    # DATE: date32 (days) / date64 (ms -> days); TIMESTAMP: timestamp[unit] without a time zone
    date_or_ts = pa.types.is_date(t) or (pa.types.is_timestamp(t) and t.tz is None)
    if pa.types.is_dictionary(t) or pa.types.is_string(t) or pa.types.is_large_string(t) \
            or (pa.types.is_temporal(t) and not date_or_ts) \
            or pa.types.is_decimal(t) or pa.types.is_nested(t) or pa.types.is_uint64(t):
        raise NotImplementedError(
            f"column type {t} is outside the int64/float64/bool hot path of this layer")
    bufs = arr.buffers()
    off = arr.offset
    has_nulls = arr.null_count > 0
    valid_bytes = None
    if has_nulls:
        vb = np.frombuffer(bufs[0], dtype=np.uint8)
        if off % 8 == 0:
            valid_bytes = vb[off // 8: off // 8 + (n + 7) // 8]
        else:   # a slice that does not start on a byte boundary: realign once
            bits = np.unpackbits(vb, bitorder="little")[off: off + n]
            valid_bytes = np.packbits(bits, bitorder="little")
    if date_or_ts:
        if pa.types.is_date32(t):
            vals, unit = np.frombuffer(bufs[1], dtype=np.int32)[off: off + n].astype(np.int64), "D"
        elif pa.types.is_date64(t):
            vals, unit = np.frombuffer(bufs[1], dtype=np.int64)[off: off + n] // 86_400_000, "D"
        else:
            vals, unit = np.frombuffer(bufs[1], dtype=np.int64)[off: off + n], t.unit
        return ArrowColumn(vals, valid_bytes, T.logical_of(unit))
    if pa.types.is_boolean(t):
        bits = np.unpackbits(np.frombuffer(bufs[1], dtype=np.uint8), bitorder="little")[off: off + n]
        return ArrowColumn(np.ascontiguousarray(bits, dtype=np.uint8).view(np.bool_), valid_bytes,
                           "boolean" if has_nulls else "bool")
    if pa.types.is_integer(t):
        np_dt = np.dtype(t.to_pandas_dtype())
        vals = np.frombuffer(bufs[1], dtype=np_dt)[off: off + n]
        name = np_dt.name
        return ArrowColumn(vals.astype(np.int64, copy=False), valid_bytes,
                           (name[0].upper() + name[1:]).replace("Uint", "UInt") if has_nulls else name)
    if pa.types.is_floating(t):
        np_dt = np.dtype(t.to_pandas_dtype())
        vals = np.frombuffer(bufs[1], dtype=np_dt)[off: off + n].astype(np.float64, copy=False)
        if has_nulls:   # NULL float = NaN, the reference's (pandas') convention
            vals = vals.copy()
            vals[np.unpackbits(valid_bytes, bitorder="little")[:n] == 0] = np.nan
        return ArrowColumn(vals, None, np_dt.name)
    raise NotImplementedError(f"column type {t} is outside the int64/float64/bool hot path of this layer")


def arrow_columns(table) -> Dict[str, ArrowColumn]:
    """pyarrow.Table -> {name: ArrowColumn}.  Multi-chunk columns are concatenated once (Arrow
    does that in C++); single-chunk columns are zero-copy views of the Arrow buffers."""
    import pyarrow as pa

    out = {}
    for name in table.column_names:
        col = table.column(name)
        arr = col.chunk(0) if col.num_chunks == 1 else (col.combine_chunks() if col.num_chunks else
                                                       pa.array([], type=col.type))
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.chunk(0) if arr.num_chunks == 1 else pa.concat_arrays(arr.chunks)
        out[str(name)] = _arrow_array_to_column(arr)
    return out


def location_format(location: str, format: Optional[str] = None) -> str:
    import os
    if format is None:
        format = os.path.splitext(location.rstrip("/"))[1].lstrip(".").lower() or "parquet"
    return format.lower()


def read_location(location: str, format: Optional[str] = None, **kwargs):
    """Parquet / CSV file (or directory of Parquet files) -> pyarrow.Table
    (the reference: input_utils/location.py:27-54, dd.read_<format>(location, **kwargs))."""
    import os

    if format is None:
        ext = os.path.splitext(location.rstrip("/"))[1].lstrip(".").lower()
        format = ext or "parquet"
    format = format.lower()
    columns = kwargs.pop("columns", None)
    kwargs.pop("gpu", None)
    if kwargs:
        raise TypeError(f"unsupported options for reading {location!r}: {sorted(kwargs)}")
    if format == "parquet":
        import pyarrow.parquet as pq
        return pq.read_table(location, columns=list(columns) if columns is not None else None)
    if format == "csv":
        import pyarrow.csv as pcsv
        t = pcsv.read_csv(location)
        return t.select(list(columns)) if columns is not None else t
    raise AttributeError(f"Do not understand the input format {format!r} (supported here: parquet, csv)")


def _host_column(values, pin=True) -> HostColumn:
    import pandas as pd

    logical = str(getattr(values, "dtype", "float64"))
    mask = None
    words = None
    if isinstance(values, ArrowColumn):
        vals, logical, words = values.values, values.logical, values.valid_words()
    elif isinstance(values, pd.Series):
        arr = values.array
        if isinstance(arr, pd.arrays.BooleanArray):
            mask, vals = np.asarray(arr._mask), np.asarray(arr._data).astype(np.uint8)
        elif isinstance(arr, (pd.arrays.IntegerArray, pd.arrays.FloatingArray)):
            mask, vals = np.asarray(arr._mask), np.asarray(arr._data)
        else:
            vals = values.to_numpy()
    elif isinstance(values, torch.Tensor):
        vals = values
    else:
        vals = np.asarray(values)
    if not isinstance(vals, torch.Tensor) and vals.dtype.kind == "M":
        vals, mask, logical = T.from_host_array(vals)      # DATE / TIMESTAMP ticks, NaT -> NULL
    if isinstance(vals, torch.Tensor):
        t = vals
        dt = {torch.int64: I64, torch.float64: F64, torch.uint8: U8, torch.bool: U8}[t.dtype]
        if t.dtype == torch.bool:
            t = t.to(torch.uint8)
        logical = {I64: "int64", F64: "float64", U8: "bool"}[dt]
    else:
        kind = vals.dtype.kind
        if kind == "b":
            vals, dt = vals.astype(np.uint8), U8
        elif T.is_temporal(logical):
            dt = I64
        elif kind in "iu" and not (kind == "u" and vals.dtype.itemsize == 8):
            vals, dt = vals.astype(np.int64, copy=False), I64
        elif kind == "f":
            vals, dt = vals.astype(np.float64, copy=False), F64
        else:
            raise NotImplementedError(
                f"column dtype {logical} is outside the int64/float64/bool hot path of this layer")
        import warnings
        with warnings.catch_warnings():
            # pandas hands out read-only views; the tensor is only ever read (H2D source), so the
            # zero-copy view is what we want
            warnings.simplefilter("ignore", UserWarning)
            t = torch.from_numpy(np.ascontiguousarray(vals))
    if pin and torch.cuda.is_available() and not t.is_pinned():
        t = t.pin_memory()
    v = None
    if words is not None:
        v = torch.from_numpy(np.ascontiguousarray(words))
    elif mask is not None and mask.any():
        v = torch.from_numpy(_pack_valid(mask))
    if v is not None and pin and torch.cuda.is_available():
        v = v.pin_memory()
    return HostColumn(t, v, dt, logical)


class DeviceTable:
    def __init__(self, partitions: List[Dict[str, object]], distribution="local", name=None):
        self.partitions = partitions
        self.distribution = distribution
        self.name = name
        self._schema = None

    def schema(self):
        if self._schema is None:
            p0 = self.partitions[0]
            self._schema = [(n, c.dtype, c.logical) for n, c in p0.items()]
        return self._schema

    @property
    def columns(self):
        return [n for n, _, _ in self.schema()]

    @property
    def nrows(self):
        return sum(next(iter(p.values())).n if p else 0 for p in self.partitions)

    @property
    def npartitions(self):
        return len(self.partitions)

    def column_nullable(self, name) -> bool:
        """does any partition of the column carry a validity bitmap?"""
        return any(p[name].valid is not None for p in self.partitions)

    def nbytes(self):
        return sum(c.nbytes() for p in self.partitions for c in p.values())

    def is_resident(self):
        return all(isinstance(c, DeviceColumn) for p in self.partitions for c in p.values())

    def column_stats(self, name) -> Stats:
        """Table-level statistics of one column (min/max/nulls), combining partitions.
        Computed on the GPU the first time a plan needs them, then cached."""
        mn = mx = None
        nulls = 0
        repeat = 0.0
        for p in self.partitions:
            c = p[name]
            if c.stats is None:
                if isinstance(c, HostColumn):
                    dev = torch.device("cuda", torch.cuda.current_device())
                    c.stats = c.to_device(dev).ensure_stats()
                else:
                    c.ensure_stats()
            st = c.stats
            nulls += st.nulls
            repeat = max(repeat, st.repeat)
            if st.vmin is not None:
                mn = st.vmin if mn is None else min(mn, st.vmin)
                mx = st.vmax if mx is None else max(mx, st.vmax)
        return Stats(mn, mx, nulls, repeat)

    # -- construction -------------------------------------------------------------------------
    @classmethod
    def from_columns(cls, columns: Dict[str, object], npartitions=1, device=None, persist=True,
                     distribution="local", name=None):
        """columns: name -> pandas Series / numpy array / torch tensor (host or device)."""
        names = list(columns)
        n = len(next(iter(columns.values()))) if names else 0
        npartitions = max(1, min(int(npartitions), max(1, n)))
        # partition boundaries on multiples of 32 rows so validity bitmaps split on word boundaries
        step = -(-n // npartitions)
        step = max(32, (step + 31) // 32 * 32)
        bounds = [(lo, min(n, lo + step)) for lo in range(0, max(n, 1), step)]
        if n == 0:
            bounds = [(0, 0)]
        parts = []
        for lo, hi in bounds:
            part = {}
            for nm in names:
                v = columns[nm]
                if isinstance(v, torch.Tensor) and v.is_cuda:
                    dt = {torch.int64: I64, torch.float64: F64, torch.uint8: U8}[v.dtype]
                    part[nm] = DeviceColumn(v[lo:hi], None, dt)
                    continue
                piece = v.iloc[lo:hi] if hasattr(v, "iloc") else v[lo:hi]
                hc = _host_column(piece, pin=not persist)
                part[nm] = hc.to_device(device) if persist else hc
            parts.append(part)
        return cls(parts, distribution, name)

    @classmethod
    def from_pandas(cls, df, npartitions=1, device=None, persist=True, distribution="local", name=None):
        return cls.from_columns({str(c): df[c] for c in df.columns}, npartitions, device, persist,
                                distribution, name)


# ---------------------------------------------------------------------------------------------
# lazy Parquet tables: row groups as partitions, pruned by the pushed-down predicate
# ---------------------------------------------------------------------------------------------
_PRUNE = None


def _prune_rule():
    """(term op) -> function(stats, literal) -> True when NO row of the row group can satisfy the term."""
    global _PRUNE
    if _PRUNE is None:
        from . import _lib as L
        _PRUNE = {
            L.EQ: lambda s, v: v < s["min"] or v > s["max"],
            L.LT: lambda s, v: s["min"] >= v,
            L.LE: lambda s, v: s["min"] > v,
            L.GT: lambda s, v: s["max"] <= v,
            L.GE: lambda s, v: s["max"] < v,
            L.IS_NULL: lambda s, v: s["nulls"] == 0,
            L.IS_NOT_NULL: lambda s, v: s["nulls"] == s["rows"],
        }
    return _PRUNE


class ParquetTable(DeviceTable):
    """A Parquet file registered with persist=False: nothing is read at create_table.  A query reads only
    the columns it references and only the row groups whose min/max/null-count statistics admit a row
    passing the pushed-down `column <cmp> literal` conjuncts -- the reference's predicate pushdown
    (physical/utils/filter.py:17 attempt_predicate_pushdown regenerates dd.read_parquet(filters=...) from
    TableScan.getDNFFilters(), table_scan.py:80-99).  Each surviving row group is one partition: Arrow
    buffers -> pinned host columns -> H2D, the kernels then apply the predicate row by row as always, so
    pruning is conservative and can only skip IO.  Decoded column chunks are kept (host memory) for the
    next query, like an OS page cache; `stats` tells how many row groups each scan skipped."""

    def __init__(self, location: str, distribution="local", name=None, columns=None):
        import pyarrow.parquet as pq
        self.location = location
        self.file = pq.ParquetFile(location)
        md = self.file.metadata
        names = [self.file.schema_arrow.names[i] for i in range(len(self.file.schema_arrow.names))]
        self._names = [n for n in names if columns is None or n in columns]
        self._nrows = md.num_rows
        import pyarrow as pa
        units = {}
        for f in self.file.schema_arrow:
            if pa.types.is_date(f.type):
                units[f.name] = "D"
            elif pa.types.is_timestamp(f.type) and f.type.tz is None:
                units[f.name] = f.type.unit
        self._groups = []                       # per row group: {"rows": n, "cols": {name: {"min","max","nulls","rows"} | None}}
        for g in range(md.num_row_groups):
            rg = md.row_group(g)
            cols = {}
            for c in range(rg.num_columns):
                col = rg.column(c)
                st = col.statistics
                nm = col.path_in_schema
                if st is not None and st.has_min_max and st.has_null_count:
                    lo, hi = st.min, st.max
                    unit = units.get(nm)
                    if unit is not None:       # datetime.date / datetime statistics -> ticks of the column's unit
                        lo, hi = T.stat_to_ticks(lo, unit), T.stat_to_ticks(hi, unit)
                    cols[nm] = {"min": lo, "max": hi, "nulls": st.null_count, "rows": rg.num_rows}
                else:
                    cols[nm] = None
            self._groups.append({"rows": rg.num_rows, "cols": cols})
        self._cache = {}                        # (row group, column) -> HostColumn
        self.stats = {"scans": 0, "row_groups_read": 0, "row_groups_skipped": 0}
        self.distribution = distribution
        self.name = name
        self._schema = None
        self._proto = None

    # -- metadata without touching the data pages
    def _prototype(self):
        """zero-row host columns: they carry every column's physical / logical type"""
        if self._proto is None:
            empty = self.file.schema_arrow.empty_table().select(self._names)
            self._proto = {n: _host_column(c, pin=False) for n, c in arrow_columns(empty).items()}
        return self._proto

    def schema(self):
        if self._schema is None:
            out = []
            for n, c in self._prototype().items():
                lg = c.logical
                if self.column_nullable(n):      # the chunks that hold NULLs arrive as pandas nullable dtypes
                    if lg.startswith(("int", "uint")):
                        lg = (lg[0].upper() + lg[1:]).replace("Uint", "UInt")
                    elif lg == "bool":
                        lg = "boolean"
                out.append((n, c.dtype, lg))
            self._schema = out
        return self._schema

    @property
    def nrows(self):
        return self._nrows

    def is_resident(self):
        return False

    @property
    def npartitions(self):
        return max(1, len(self._groups))

    def column_nullable(self, name) -> bool:
        sts = [g["cols"].get(name) for g in self._groups]
        return any(s is None or s["nulls"] > 0 for s in sts)

    def column_stats(self, name) -> Stats:
        """from the file's row-group statistics when every row group carries them, else from the data"""
        sts = [g["cols"].get(name) for g in self._groups]
        dt = dict((n, d) for n, d, _ in self.schema())[name]
        if sts and all(s is not None for s in sts) and dt != F64:       # float NaNs are not in Parquet null counts
            lo, hi = min(s["min"] for s in sts), max(s["max"] for s in sts)
            return Stats(int(lo), int(hi), sum(s["nulls"] for s in sts), 0.0)
        return super().column_stats(name)

    # -- data
    def _column(self, g: int, name: str) -> HostColumn:
        key = (g, name)
        if key not in self._cache:
            t = self.file.read_row_group(g, columns=[name])
            self._cache[key] = _host_column(arrow_columns(t)[name], pin=torch.cuda.is_available())
        return self._cache[key]

    @property
    def partitions(self):
        """every row group, every column (generic callers; scans go through scan_pruned)"""
        return [{n: self._column(g, n) for n in self._names} for g in range(len(self._groups))] or [dict(self._prototype())]

    @partitions.setter
    def partitions(self, value):          # DeviceTable.__init__ is not used; nothing to set
        pass

    def surviving_groups(self, terms):
        """row groups that may hold a row passing all `terms` = [(column, B2 op, literal)]"""
        rules = _prune_rule()
        keep = []
        for g, info in enumerate(self._groups):
            dead = False
            for name, op, lit in terms:
                st = info["cols"].get(name)
                rule = rules.get(op)
                if st is None or rule is None:
                    continue
                if isinstance(lit, float) and isinstance(st["min"], int):
                    # the kernel compares an int column with a float literal in float64, where 2^53 + 1
                    # equals 2^53 (expr.F64_EXACT_INT); Python's exact int/float comparison would prune it
                    st = dict(st, min=float(st["min"]), max=float(st["max"]))
                try:
                    if rule(st, lit):
                        dead = True
                        break
                except TypeError:               # statistics of a type that does not compare with the literal
                    continue
            if not dead:
                keep.append(g)
        return keep

    def scan_pruned(self, needed, terms):
        """[{column: HostColumn}] for the row groups that survive `terms`, restricted to `needed`"""
        keep = self.surviving_groups(terms)
        self.stats["scans"] += 1
        self.stats["row_groups_read"] += len(keep)
        self.stats["row_groups_skipped"] += len(self._groups) - len(keep)
        cols = [n for n in self._names if n in needed]
        parts = [{n: self._column(g, n) for n in cols} for g in keep if self._groups[g]["rows"] > 0]
        if not parts:
            proto = self._prototype()
            parts = [{n: proto[n] for n in cols}]
        return parts
