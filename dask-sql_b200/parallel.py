"""Multi-GPU plumbing: one process per GPU, torch.distributed (NCCL over NVLink/NVSwitch on
GPUs, gloo in the CPU tests).  Only the two exchange steps of the path use it (SURVEY 8e):

  * join build side   : broadcast of the dimension table's columns from its owner rank
                        (replaces dask's merge(broadcast=True), join.py:228-246)
  * group-by partials : dense tables -> merged by slot range, every rank keeps one range: ONE kernel over
                        NVLink peer memory for prepared plans (PeerArena + b2_peer_merge), else
                        ncclReduceScatter per array; hash tables -> a tree of pairwise send/recv + merge,
                        fan-in = sql.aggregate.split_every (replaces dask's tree reduction,
                        aggregate.py:321,581)
"""
from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


import os
import time

_WORLD = None        # (rank, size, backend) once a process group exists: asked dozens of times per query
coll_times = {} if os.environ.get("B200SQL_CALL_TIMES") == "1" else None     # diagnostics: name -> [calls, host s]


def _timed(name, fn, *args, **kw):
    if coll_times is None:
        return fn(*args, **kw)
    t0 = time.perf_counter()
    out = fn(*args, **kw)
    rec = coll_times.setdefault(name, [0, 0.0])
    rec[0] += 1
    rec[1] += time.perf_counter() - t0
    return out


def world() -> Tuple[int, int]:
    global _WORLD
    if _WORLD is not None:
        if dist.is_initialized():
            return _WORLD[0], _WORLD[1]
        _WORLD = None                      # the group was destroyed
    if dist.is_available() and dist.is_initialized():
        _WORLD = (dist.get_rank(), dist.get_world_size(), dist.get_backend())
        return _WORLD[0], _WORLD[1]
    return 0, 1


def shard_bounds(n: int, rank: int, size: int, align: int = 32) -> Tuple[int, int]:
    """Contiguous row range of `rank` when n rows are sharded over `size` ranks; boundaries are
    multiples of `align` rows so validity bitmaps split on word boundaries."""
    per = -(-n // size)
    per = (per + align - 1) // align * align
    lo = min(n, rank * per)
    hi = min(n, lo + per)
    return lo, hi


def allreduce_(t: torch.Tensor, op: str = "sum") -> torch.Tensor:
    if world()[1] == 1:
        return t
    rop = {"sum": dist.ReduceOp.SUM, "min": dist.ReduceOp.MIN, "max": dist.ReduceOp.MAX}[op]
    _timed(f"all_reduce[{t.dtype},{op}]", dist.all_reduce, t, op=rop)
    return t


def _backend() -> str:
    return _WORLD[2] if world()[1] > 1 else "none"


def reduce_scatter_(t: torch.Tensor, op: str = "sum", out=None) -> torch.Tensor:
    """Element-wise reduction of `t` over all ranks, of which this rank keeps only its own
    contiguous 1/size slice (t.numel() must be a multiple of the world size).  NCCL: one
    ncclReduceScatter -- (size-1)/size of the array crosses NVLink per rank instead of the
    2(size-1)/size of an all-reduce, and the consumer (compaction of the group table) then
    touches 1/size of the slots.  gloo (CPU tests) has no reduce-scatter: all-reduce + slice."""
    rank, size = world()
    if size == 1:
        return t
    n = t.numel()
    assert n % size == 0, "reduce_scatter_ needs a length that is a multiple of the world size"
    chunk = n // size
    bitwise = op in ("and", "or", "xor")
    rop = {"sum": dist.ReduceOp.SUM, "min": dist.ReduceOp.MIN, "max": dist.ReduceOp.MAX, "and": dist.ReduceOp.BAND,
           "or": dist.ReduceOp.BOR, "xor": dist.ReduceOp.BXOR}[op]
    if _backend() == "nccl" and bitwise:
        # NCCL has no bitwise reduction: every rank receives the peers' copies of its slot chunk and folds
        # them in rank order with b2_bitwise_combine (the op on 32-bit words is the op on 64-bit ones)
        from . import _lib as L
        from . import device as D
        recv = torch.empty(n, dtype=t.dtype, device=t.device)
        _timed(f"all_to_all[{t.dtype},{op}]", dist.all_to_all_single, recv, t.contiguous())
        if out is None:
            out = torch.empty(chunk, dtype=t.dtype, device=t.device)
        out.copy_(recv[:chunk])
        words = chunk * t.element_size() // 4
        code = {"and": L.AGG_AND, "or": L.AGG_OR, "xor": L.AGG_XOR}[op]
        for r in range(1, size):
            L.bitwise_combine(out.data_ptr(), recv[r * chunk:(r + 1) * chunk].data_ptr(), words, code, D.stream_ptr())
        return out
    if _backend() == "nccl":
        if out is None:
            out = torch.empty(chunk, dtype=t.dtype, device=t.device)
        _timed(f"reduce_scatter[{t.dtype},{op}]", dist.reduce_scatter_tensor, out, t, op=rop)
        return out
    dist.all_reduce(t, op=rop)
    return t[rank * chunk:(rank + 1) * chunk].clone()


def all_gather_varlen(t: torch.Tensor, counts: Sequence[int], cat: bool = True):
    """Concatenation over ranks of the first counts[r] elements of every rank's 1-D `t`
    (ONE collective on max(counts)-padded buffers instead of one broadcast per rank).
    cat=False returns the per-rank pieces (views of the receive buffer) instead."""
    rank, size = world()
    if size == 1:
        return t[: counts[0]] if cat else [t[: counts[0]]]
    m = max(max(counts), 1)
    send = t
    if t.numel() != m:
        send = torch.zeros(m, dtype=t.dtype, device=t.device)
        send[: counts[rank]] = t[: counts[rank]]
    if _backend() == "nccl":
        recv = torch.empty(size * m, dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(recv, send.contiguous())
        pieces = [recv[r * m: r * m + counts[r]] for r in range(size)]
    else:
        bufs = [torch.empty(m, dtype=t.dtype, device=t.device) for _ in range(size)]
        dist.all_gather(bufs, send.contiguous())
        pieces = [bufs[r][: counts[r]] for r in range(size)]
    if not cat:
        return pieces
    return torch.cat(pieces)


def all_gather_ints(values: Sequence[int], device) -> List[List[int]]:
    """Every rank's small list of integers on every rank (one tiny all-gather + one host read)."""
    rank, size = world()
    if size == 1:
        return [list(values)]
    t = torch.tensor(list(values), dtype=torch.int64, device=device)
    bufs = [torch.empty_like(t) for _ in range(size)]
    dist.all_gather(bufs, t)
    return torch.stack(bufs).cpu().tolist()


class PeerArena:
    """One allocation per rank that EVERY rank of the job has mapped (NVLink / NVSwitch peer memory):
    torch.distributed._symmetric_memory allocates it with the CUDA VMM API and exchanges the handles
    through the process group's store -- memory and mapping only, no torch kernel ever touches it.
    carve() hands out 256-byte aligned views of this rank's copy; `base[p]` is rank p's copy as mapped
    into this process (what b2_peer_merge dereferences); offsets are identical on all ranks because
    every rank carves in the same order."""

    ALIGN = 256

    def __init__(self, nbytes: int, device):
        import torch.distributed._symmetric_memory as symm
        nbytes = (int(nbytes) + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.buf = symm.empty(nbytes, dtype=torch.uint8, device=device)
        self.buf.zero_()
        self.hdl = symm.rendezvous(self.buf, dist.group.WORLD)
        self.base = [int(p) for p in self.hdl.buffer_ptrs]
        rank, size = world()
        if len(self.base) != size or self.base[rank] != self.buf.data_ptr():
            raise RuntimeError("symmetric memory rendezvous returned an unexpected mapping")
        self.nbytes, self.used = nbytes, 0
        torch.cuda.synchronize(device)
        dist.barrier()                     # every rank's copy is zeroed before anyone signals into it

    def carve(self, n: int, dtype, fill=0):
        """(view of n elements of `dtype` in this rank's copy, filled; its byte offset in every copy)"""
        width = torch.empty((), dtype=dtype).element_size()
        off = self.used
        nb = (n * width + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        if off + nb > self.nbytes:
            raise MemoryError("peer arena exhausted")
        self.used = off + nb
        t = self.buf[off: off + n * width].view(dtype)
        t.fill_(fill)
        return t, off


def peer_memory_available() -> bool:
    """NCCL job on one node whose torch build has symmetric memory; B200SQL_PEER_MERGE=0 turns it off."""
    if os.environ.get("B200SQL_PEER_MERGE") == "0" or world()[1] < 2 or _backend() != "nccl":
        return False
    try:
        import torch.distributed._symmetric_memory  # noqa: F401
    except Exception:
        return False
    return True


def broadcast_(t: torch.Tensor, src: int = 0) -> torch.Tensor:
    if world()[1] > 1:
        _timed("broadcast", dist.broadcast, t, src=src)
    return t


def broadcast_object(obj, src: int = 0):
    if world()[1] == 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=src)
    return box[0]


def tree_rounds(size: int, fan_in: int = 2) -> List[List[Tuple[int, int]]]:
    """Merge schedule of a fan-in-`fan_in` reduction tree onto rank 0.
    Returns rounds; each round is a list of (receiver, sender) pairs that can run concurrently.
    With fan_in = split_every this mirrors dask's tree of partial-aggregate concatenations."""
    fan_in = max(2, int(fan_in))
    rounds = []
    stride = 1
    while stride < size:
        pairs = []
        group = stride * fan_in
        for base in range(0, size, group):
            for k in range(1, fan_in):
                s = base + k * stride
                if s < size:
                    pairs.append((base, s))
        # senders within one group target the same receiver: serialise them into sub-rounds
        sub = {}
        for r, s in pairs:
            sub.setdefault(r, []).append(s)
        depth = max(len(v) for v in sub.values())
        for d in range(depth):
            rounds.append([(r, v[d]) for r, v in sub.items() if d < len(v)])
        stride = group
    return rounds


def send_tensors(tensors: Sequence[torch.Tensor], dst: int):
    for t in tensors:
        dist.send(t.contiguous(), dst=dst)


def recv_tensors(shapes_dtypes, src: int, device) -> List[torch.Tensor]:
    out = []
    for shape, dtype in shapes_dtypes:
        t = torch.empty(shape, dtype=dtype, device=device)
        dist.recv(t, src=src)
        out.append(t)
    return out
