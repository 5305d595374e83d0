"""ANALYZE TABLE ... COMPUTE STATISTICS on a C2-shaped table: `--rows` rows (default 200M) in 8 partitions, `key`
int64 uniform on [0, 1M), `val` float64 uniform on [0, 1).  For each column:

- the passes of the radix select (b2_select_hist) and each pass's kernel time (CUDA events around the pass's
  launches over every partition, after `--warmup` warm-up selects, averaged over `--steps` selects);
- the bytes each pass reads (8 per row it scans; a compacting pass also writes 8 per row it keeps) and that over
  the kernel time as a share of the H100 SXM data sheet's 3.35 TB/s;
- the end-to-end `ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS <col>` time (host clock; the statement ends in
  a device-to-host copy), warmed up, averaged over `--steps`, and the same for its two parts: the select driver
  (executor.column_quantiles) and `SELECT AVG(col), STDDEV_SAMP(col) FROM t`;
- for comparison, b2_sort_by on the same column as one 200M-row array (CUDA events).

Prints one JSON line with the card's name, power limit and max SM clock, read in the same process.  Writes
nothing.
usage: python scripts/bench_analyze.py [--rows 200000000] [--steps 5] [--warmup 2]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

HBM_PEAK_GBS = 3350.0        # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import numpy as np
    import pandas as pd
    import torch
    from bench_bitwise import card
    from dask_sql_b200 import Context, executor
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.rows
    g = torch.Generator(device=dev)
    g.manual_seed(2)
    key = torch.randint(0, 1_000_000, (n,), dtype=torch.int64, device=dev, generator=g)
    val = torch.rand(n, dtype=torch.float64, device=dev, generator=g)
    c = Context()
    c.create_table("t", {"key": key, "val": val}, npartitions=8, persist=True)
    table = c.schema["root"].tables["t"].df.source.table
    out = {"card": card(), "rows": n, "partitions": table.npartitions, "steps": args.steps, "warmup": args.warmup,
           "columns": {}}

    for name, col in (("key", key), ("val", val)):
        dt = L.I64 if col.dtype == torch.int64 else L.F64
        st = table.column_stats(name)
        passes = -(-(executor.select_image(st.vmin, dt) ^ executor.select_image(st.vmax, dt)).bit_length() // 11)
        for _ in range(args.warmup):
            executor.column_quantiles(table, name)
        torch.cuda.synchronize()
        executor.kernel_events = []
        for _ in range(args.steps):
            executor.column_quantiles(table, name)
        torch.cuda.synchronize()
        evs, executor.kernel_events = executor.kernel_events, None
        assert len(evs) == passes * args.steps, (len(evs), passes)
        per_pass = []
        for p in range(passes):
            mine = evs[p::passes]
            ms = sum(e0.elapsed_time(e1) for _, _, e0, e1 in mine) / len(mine)
            kind, rows = mine[0][0], mine[0][1]
            read = 8 * rows
            written = 0
            if kind == "b2_select_hist_compact":
                # the rows it keeps are what the next pass reads
                written = 8 * evs[p + 1][1] if p + 1 < passes else 0
            gbs = (read + written) / ms / 1e6
            per_pass.append({"kernel": kind, "rows_scanned": rows, "bytes_read": read, "bytes_written": written,
                             "ms": round(ms, 4), "GBps": round(gbs, 1), "hbm_share": round(gbs / HBM_PEAK_GBS, 3)})

        def host_ms(fn):
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                r = fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / args.steps, r

        analyze_ms, res = host_ms(lambda: c.sql(f"ANALYZE TABLE t COMPUTE STATISTICS FOR COLUMNS {name}"))
        # its two parts: the select driver, and the AVG / STDDEV_SAMP query it runs for mean and std
        quantiles_ms, _ = host_ms(lambda: executor.column_quantiles(table, name))
        moments_ms, _ = host_ms(lambda: c.sql(f"SELECT AVG({name}) AS m, STDDEV_SAMP({name}) AS s FROM t",
                                              return_futures=False))

        # the quantiles against torch's own sort of the column (a check of the numbers being timed, not a timing)
        srt = torch.sort(col).values
        m = n - 1
        for q, row in ((0.25, "25%"), (0.5, "50%"), (0.75, "75%")):
            lo = int(np.floor(q * m))
            a, b = srt[lo].item(), srt[min(lo + 1, m)].item()
            want = pd.Series([a, b], dtype=np.int64 if dt == L.I64 else np.float64).quantile(q * m - lo)
            assert res.at[row, name] == want, (name, row, res.at[row, name], want)
        del srt

        # b2_sort_by over the same column as one array
        whole = D.DeviceColumn(col, None, dt)
        idx = torch.empty(n, dtype=torch.int32, device=dev)
        ws = torch.empty(L.sort_ws_bytes(n), dtype=torch.uint8, device=dev)
        cs = whole.as_struct()
        sort_ms = []
        for i in range(args.warmup + args.steps):
            L.iota(D.ptr(idx), n, D.stream_ptr())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            L.sort_by(C.byref(cs), n, 0, 0, D.ptr(idx), D.ptr(ws), D.stream_ptr())
            e1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                sort_ms.append(e0.elapsed_time(e1))
        del ws, idx
        out["columns"][name] = {
            "passes": passes, "per_pass": per_pass,
            "select_kernel_ms_total": round(sum(p["ms"] for p in per_pass), 4),
            "analyze_ms": round(analyze_ms, 3),
            "quantiles_host_ms": round(quantiles_ms, 3),
            "avg_stddev_query_ms": round(moments_ms, 3),
            "sort_by_ms": round(sum(sort_ms) / len(sort_ms), 3),
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
