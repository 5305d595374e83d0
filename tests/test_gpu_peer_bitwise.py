"""b2_peer_merge's AND / OR / XOR arrays on ONE GPU, the way tests/test_gpu_peer.py checks the sums and
extrema: `world` buffers stand in for the ranks' symmetric copies, every "rank" runs its kernel on its own
stream, and each merged slice must equal the sequential rank-order fold bit for bit."""
import ctypes as C

import pytest

from tests.test_gpu_peer import ALIGN, _carve

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_peer_merge_bitwise(world):
    import torch
    from dask_sql_b200 import _lib as L

    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev)
    g.manual_seed(7 * world)
    chunk = 32 * 37
    alloc = chunk * world
    names = ["and", "or", "xor", "rows"]
    ops = [L.PEER_AND_I64, L.PEER_OR_I64, L.PEER_XOR_I64, L.PEER_SUM_I64]
    ident = {"and": -1, "or": 0, "xor": 0, "rows": 0}
    edges = torch.tensor([-2**63, -1, 0, 2**63 - 1, -2, 1], dtype=torch.int64, device=dev)
    bufs = [torch.zeros(len(names) * alloc * 8 + 8 * ALIGN, dtype=torch.uint8, device=dev) for _ in range(world)]
    tabs = []
    for r in range(world):
        used = 0
        _, sig_off, used = _carve(bufs[r], used, L.MAX_PEERS, torch.int64)
        arrs, offs = {}, {}
        for name in names:
            arrs[name], offs[name], used = _carve(bufs[r], used, alloc, torch.int64)
        hit = torch.rand(alloc, device=dev, generator=g) < 0.5
        ints = torch.randint(-2**63, 2**63 - 1, (alloc,), dtype=torch.int64, device=dev, generator=g)
        pick = torch.randint(0, len(edges), (alloc,), device=dev, generator=g)
        ints = torch.where(torch.rand(alloc, device=dev, generator=g) < 0.3, edges[pick], ints)
        for name in ("and", "or", "xor"):
            arrs[name].copy_(torch.where(hit, ints, torch.full_like(ints, ident[name])))
        arrs["rows"].copy_(hit.to(torch.int64))
        tabs.append((arrs, hit))
    ready = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    outs, press, descs = [], [], []
    for r in range(world):
        m = L.PeerMerge()
        m.world, m.rank, m.narrays = world, r, len(names)
        m.lo, m.count, m.signal_off = r * chunk, chunk, sig_off
        m.local_ready = ready[r].data_ptr()
        for p in range(world):
            m.peer_base[p] = bufs[p].data_ptr()
        o = {}
        for a, (name, op) in enumerate(zip(names, ops)):
            m.ops[a], m.array_off[a] = op, offs[name]
            o[name] = torch.empty(chunk, dtype=torch.int64, device=dev)
            m.out[a] = o[name].data_ptr()
        pres = torch.full((chunk,), 7, dtype=torch.uint8, device=dev)
        m.out_present = pres.data_ptr()
        m.presence_kind, m.presence_array = L.PEER_PRESENT_ROWS, 3
        outs.append(o), press.append(pres), descs.append(m)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    for epoch in (1, 2):
        for r in reversed(range(world)):
            descs[r].epoch = epoch
            L.peer_merge(C.byref(descs[r]), C.c_void_p(streams[r].cuda_stream))
        torch.cuda.synchronize()
    any_hit = torch.stack([h for _, h in tabs]).any(0)
    for r in range(world):
        sl = slice(r * chunk, (r + 1) * chunk)
        exp = {n: tabs[0][0][n][sl].clone() for n in names}
        for p in range(1, world):
            a = tabs[p][0]
            exp["and"] &= a["and"][sl]
            exp["or"] |= a["or"][sl]
            exp["xor"] ^= a["xor"][sl]
            exp["rows"] += a["rows"][sl]
        for n in names:
            assert torch.equal(outs[r][n], exp[n]), (n, r)
        assert torch.equal(press[r], any_hit[sl].to(torch.uint8)), r
