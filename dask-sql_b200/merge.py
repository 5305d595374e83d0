"""Cross-GPU exchange steps of the path (one process per GPU, torch.distributed):

  broadcast_part / allgather_part : join build side (dimension table) reaches every rank
  tree_merge_raw                  : hash GROUP BY partials merged along a fan-in tree

Dense group tables never come here: their accumulator arrays are all-reduced in place
(executor._allreduce_table).
"""
from collections import OrderedDict
from typing import List

import torch
import torch.distributed as dist

from . import _lib as L
from . import parallel as P
from .device import DeviceColumn, I64, F64, U8

_TORCH_DT = {I64: torch.int64, F64: torch.float64, U8: torch.uint8}


def _meta(part, names):
    return [(n, part[n].dtype, part[n].logical, part[n].valid is not None) for n in names]


def broadcast_part(part, dev, src=0):
    """Every rank receives rank `src`'s copy of `part` (NCCL broadcast per column buffer)."""
    from .executor import Part
    rank, size = P.world()
    if size == 1:
        return part
    names = list(part.keys())
    n, meta = P.broadcast_object((part.n, _meta(part, names)) if rank == src else None, src)
    out = Part({}, n)
    for name, dt, lg, has_valid in meta:
        if rank == src:
            data, valid = part[name].data.contiguous(), part[name].valid
        else:
            data = torch.empty(n, dtype=_TORCH_DT[dt], device=dev)
            valid = torch.empty((n + 31) // 32, dtype=torch.int32, device=dev) if has_valid else None
        if n:
            P.broadcast_(data, src)
            if has_valid:
                P.broadcast_(valid, src)
        out[name] = DeviceColumn(data, valid if has_valid else None, dt, lg)
    return out


def allgather_part(part, dev):
    """Concatenation (in rank order) of every rank's `part` on every rank: the build side arrives
    pre-sharded, or a key-range-sharded aggregate is needed whole.  One all-gather per column
    buffer on max-count-padded slices, not one broadcast per rank."""
    from .executor import Part, concat_columns
    rank, size = P.world()
    if size == 1:
        return part
    names = list(part.keys())
    hdr = P.all_gather_ints([part.n] + [1 if part[n].valid is not None else 0 for n in names], dev)
    counts = [h[0] for h in hdr]
    out = Part({}, sum(counts))
    for i, name in enumerate(names):
        c = part[name]
        pieces = P.all_gather_varlen(c.data.contiguous(), counts, cat=False)
        if not any(h[1 + i] for h in hdr):
            out[name] = DeviceColumn(torch.cat(pieces), None, c.dtype, c.logical)
            continue
        # some rank carries NULLs: gather the bitmap words too and re-pack row-wise on the device
        wcounts = [(n + 31) // 32 for n in counts]
        mine = c.valid if c.valid is not None else torch.full((wcounts[rank],), -1, dtype=torch.int32, device=dev)
        vpieces = P.all_gather_varlen(mine.contiguous(), wcounts, cat=False)
        cols = [DeviceColumn(d, v if hdr[r][1 + i] else None, c.dtype, c.logical)
                for r, (d, v) in enumerate(zip(pieces, vpieces)) if counts[r] > 0]
        out[name] = concat_columns(cols) if cols else DeviceColumn(torch.cat(pieces), None, c.dtype, c.logical)
    return out


def _send_part(part, names, dst):
    for n in names:
        c = part[n]
        if part.n:
            dist.send(c.data.contiguous(), dst=dst)
            if c.valid is not None:
                dist.send(c.valid.contiguous(), dst=dst)


def _recv_part(meta, n, src, dev):
    from .executor import Part
    out = Part({}, n)
    for name, dt, lg, has_valid in meta:
        data = torch.empty(n, dtype=_TORCH_DT[dt], device=dev)
        valid = torch.empty((n + 31) // 32, dtype=torch.int32, device=dev) if has_valid else None
        if n:
            dist.recv(data, src=src)
            if has_valid:
                dist.recv(valid, src=src)
        out[name] = DeviceColumn(data, valid, dt, lg)
    return out


def raw_to_part(raw):
    """RawGroups -> flat Part: keys k*, accumulators a<i>, counts c<i>, rows."""
    from .executor import Part
    cols = OrderedDict()
    for i, (name, col) in enumerate(raw.keys.items()):
        cols[f"k{i}"] = col
    for i, a in enumerate(raw.acc):
        if a is not None:
            cols[f"a{i}"] = a
    for i, c in enumerate(raw.cnt):
        if c is not None:
            cols[f"c{i}"] = c
    if raw.rows is not None:
        cols["rows"] = raw.rows
    return Part(cols, raw.n)


def part_to_raw(part, raw_like):
    from .executor import RawGroups
    keys = OrderedDict((name, part[f"k{i}"]) for i, name in enumerate(raw_like.keys))
    acc = [part.get(f"a{i}") if a is not None else None for i, a in enumerate(raw_like.acc)]
    cnt = [part.get(f"c{i}") if c is not None else None for i, c in enumerate(raw_like.cnt)]
    rows = part.get("rows") if raw_like.rows is not None else None
    return RawGroups(keys, acc, cnt, rows, part.n)


def merge_partials(parts: List, plan, nkeys: int):
    """Re-aggregate concatenated partial tables on this GPU with the same group-by kernels:
    SUM of partial sums / counts / rows, MIN of mins, MAX of maxes, AND / OR / XOR of bitwise partials."""
    from .executor import Part, concat_parts
    from .frame import LazyFrame, TableSource, AggSource
    from .table import DeviceTable

    names = list(parts[0].keys())
    whole = concat_parts(parts, names)
    table = DeviceTable([dict(whole.resolve())], "local")
    frame = LazyFrame(TableSource(table))
    aggs = []
    for n in names:
        if n.startswith("k"):
            continue
        fn = "sum"
        if n.startswith("a"):
            op = plan.kaggs[int(n[1:])].op
            fn = {L.AGG_MIN: "min", L.AGG_MAX: "max", L.AGG_AND: "bit_and", L.AGG_OR: "bit_or",
                  L.AGG_XOR: "bit_xor"}.get(op, "sum")
        aggs.append((n, n, fn))
    keys = [f"k{i}" for i in range(nkeys)]
    merged = LazyFrame(AggSource(frame, keys, aggs))
    from .executor import execute
    out = execute(merged)
    res = concat_parts(out, names)
    # partial accumulators are never NULL: drop validity bitmaps the generic path may add
    for n in names:
        if not n.startswith("k") and res[n].valid is not None:
            res[n] = DeviceColumn(res[n].data, None, res[n].dtype, res[n].logical)
    return res


def tree_merge_raw(raw, plan, options, dev):
    """Tree-reduce the per-rank partial group tables onto rank 0, then broadcast the result.
    Fan-in = sql.aggregate.split_every (default 8), like dask's groupby tree (aggregate.py:581)."""
    rank, size = P.world()
    if size == 1:
        return raw
    fan_in = int((options or {}).get("split_every") or 8)
    local = raw_to_part(raw)
    names = list(local.keys())
    nkeys = len(raw.keys)
    for rnd in P.tree_rounds(size, fan_in):
        for receiver, sender in rnd:
            if rank == sender:
                hdr = torch.tensor([local.n] + [1 if local[n].valid is not None else 0 for n in names],
                                   dtype=torch.int64, device=dev)
                dist.send(hdr, dst=receiver)
                _send_part(local, names, receiver)
            elif rank == receiver:
                hdr = torch.empty(1 + len(names), dtype=torch.int64, device=dev)
                dist.recv(hdr, src=sender)
                h = hdr.cpu().tolist()
                meta = [(n, local[n].dtype, local[n].logical, bool(v)) for n, v in zip(names, h[1:])]
                other = _recv_part(meta, h[0], sender, dev)
                local = merge_partials([local, other], plan, nkeys)
    local = broadcast_part(local, dev, src=0)
    return part_to_raw(local, raw)
