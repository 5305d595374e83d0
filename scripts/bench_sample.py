"""Measure b2_sample_mask, TABLESAMPLE and RAND on the GPU (DESIGN.md section 4).

  python scripts/bench_sample.py [--rows 2e8] [--reps 20] [--out FILE]

- b2_sample_mask alone over 2e8 and 1e9 rows: CUDA events around `reps` launches; rows/s, and the bytes the
  kernel must store (1 B per row) over its time against 3.35 TB/s.
- A filtered global aggregate (C1-shaped) and a dense GROUP BY (C2-shaped) over `rows` resident rows in 8
  partitions, at BERNOULLI 1, 10 and 50 % and without a sample, the arms alternating; C2 also at SYSTEM 10 %.
- SUM(RAND(1)) per row.
Prints the card's name and power limit first, and one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:            # no nvidia-smi: the name from torch
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def time_mask(n, reps):
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    th = int(round(0.1 * 2 ** 32))
    for _ in range(3):
        L.sample_mask(n, 12345, 7, 1, th, out.data_ptr(), D.stream_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(D.cur_stream())
    for _ in range(reps):
        L.sample_mask(n, 12345, 7, 1, th, out.data_ptr(), D.stream_ptr())
    e1.record(D.cur_stream())
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    kept = int(out.sum(dtype=torch.int64).item())
    del out
    torch.cuda.empty_cache()
    return {"what": "b2_sample_mask", "rows": n, "ms": round(ms, 4), "rows_per_s": n / ms * 1e3,
            "store_share_of_3.35TBps": round(n / (ms * 1e-3) / 3.35e12, 3), "kept_frac": kept / n}


def time_query(c, sql, reps):
    c.sql(sql).compute()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        c.sql(sql).compute()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=2e8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from dask_sql_b200 import Context
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    for n in (int(2e8), int(1e9)):
        emit(time_mask(n, a.reps))

    n = int(a.rows)
    rng = np.random.default_rng(0)
    df = pd.DataFrame({"k": rng.integers(0, 1000, n), "h": rng.integers(-2 ** 31, 2 ** 31, n), "x": rng.random(n)})
    c = Context()
    c.create_table("t", df, npartitions=8, persist=True)
    del df
    shapes = {"C1": "SELECT SUM(h) AS s, COUNT(*) AS n FROM t{} WHERE x < 0.5",
              "C2": "SELECT k, SUM(h) AS s, COUNT(*) AS n FROM t{} GROUP BY k"}
    arms = [("none", ""), ("bernoulli1", " TABLESAMPLE BERNOULLI (1) REPEATABLE (1)"),
            ("bernoulli10", " TABLESAMPLE BERNOULLI (10) REPEATABLE (1)"),
            ("bernoulli50", " TABLESAMPLE BERNOULLI (50) REPEATABLE (1)"),
            ("system10", " TABLESAMPLE SYSTEM (10) REPEATABLE (1)")]
    for shape, sql in shapes.items():
        res = {name: [] for name, _ in arms}
        for _ in range(3):                       # alternate the arms
            for name, clause in arms:
                if name == "system10" and shape == "C1":
                    continue
                res[name] += time_query(c, sql.format(clause), max(1, a.reps // 4))
        for name, ts in res.items():
            if ts:
                emit({"what": shape, "arm": name, "rows": n, "median_ms": round(float(np.median(ts)), 3),
                      "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3)})
    ts = time_query(c, "SELECT SUM(RAND(1)) AS s FROM t", a.reps)
    base = time_query(c, "SELECT SUM(x) AS s FROM t", a.reps)
    emit({"what": "SUM(RAND(1))", "rows": n, "median_ms": round(float(np.median(ts)), 3),
          "ns_per_row": round(float(np.median(ts)) * 1e6 / n, 4), "SUM(x)_median_ms": round(float(np.median(base)), 3)})
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
