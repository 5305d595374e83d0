"""VARCHAR columns between ranks on CPU (gloo): a replicated table's dictionary travels as its host arrays
and digest only -- never its per-device copies or host caches -- and every rank decodes the same strings."""
import multiprocessing as mp
import os
import pickle
import socket

import numpy as np
import pyarrow as pa
import torch
import torch.distributed as dist

from dask_sql_b200 import strings as S


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


WORDS = ["pear", None, "apple", "", "öl", "😀", "apple"]


def test_pickled_dictionary_carries_host_arrays_only():
    codes, null, lg = S.encode_arrow(pa.array(WORDS))
    d = lg.dictionary
    d.device(torch.device("cpu"))                 # a per-device copy and the host caches exist ...
    d.categories()
    d.sorted_objects()
    blob = pickle.dumps(lg)
    assert b"torch" not in blob and b"pandas" not in blob      # ... and none of them is pickled
    back = pickle.loads(blob)
    assert S.is_varchar(back) and back == "category" and back.dictionary is d     # equal dictionary reused


def _worker(rank, size, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=size)
    try:
        from dask_sql_b200 import merge
        from dask_sql_b200.device import DeviceColumn, I64
        from dask_sql_b200.executor import Part
        dev = torch.device("cpu")
        codes, null, lg = S.encode_arrow(pa.array(WORDS))     # replicated: every rank builds the same dictionary
        lg.dictionary.device(dev)
        col = DeviceColumn(torch.from_numpy(codes), None, I64, lg)
        part = Part({"s": col}, len(codes)) if rank == 0 else Part({}, 0)
        got = merge.broadcast_part(part, dev, src=0)["s"]
        gathered = merge.allgather_part(Part({"s": col}, len(codes)), dev)["s"]
        out = []
        for c in (got, gathered):
            assert S.is_varchar(c.logical) and c.logical.dictionary.digest == lg.dictionary.digest
            d = c.logical.dictionary.to_list()
            out.append([d[i] for i in c.data.tolist()])
        out_q.put((rank, out))
    finally:
        dist.destroy_process_group()


def test_gloo_broadcast_and_allgather_of_a_varchar_column():
    size = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, size, port, q)) for r in range(size)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in range(size)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    codes, null, lg = S.encode_arrow(pa.array(WORDS))
    d = lg.dictionary.to_list()
    want = [d[c] for c in codes]            # NULL rows hold code 0 (the bitmap carries NULL)
    for _, (bcast, gathered) in results:
        assert bcast == want and gathered == want * size
    assert np.array_equal(null, [w is None for w in WORDS])
