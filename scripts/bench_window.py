"""Measure the window functions on one GPU (DESIGN.md section 4, "Window functions").

  python scripts/bench_window.py [--rows 1e8] [--keys 1e6] [--steps 5] [--warmup 2] [--check-rows 1e6]
                                 [--out FILE]

Table: `rows` rows, int64 partition key k with `keys` distinct values, int64 order key t, float64 v (seeded).
Queries:
  ROW_NUMBER() OVER (PARTITION BY k ORDER BY t)
  SUM(v) OVER (PARTITION BY k ORDER BY t ROWS 10 PRECEDING)
  MAX(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 1000 PRECEDING AND CURRENT ROW)
For each: the step time (host clock around a query that ends in a device synchronise), split into the sort, the
window kernels and the scatter back to input order by CUDA events (executor.kernel_events); the bytes per row
the window kernels move, from the shapes (window_bytes_per_row), and that traffic over the window-kernel time
against the data sheet's 3.35 TB/s.  Before timing, the same queries run over the first `check-rows` rows of
the same seed and are compared with tests/window_ref.py.  Prints the card's name and power limit, then one
JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
QUERIES = {
    "row_number": ("ROW_NUMBER() OVER (PARTITION BY k ORDER BY t)", ("ROW_NUMBER", None, None)),
    "sum_rows10": ("SUM(v) OVER (PARTITION BY k ORDER BY t ROWS 10 PRECEDING)", ("SUM", "v", (False, -10, 0))),
    "max_rows1000": ("MAX(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 1000 PRECEDING AND CURRENT ROW)",
                     ("MAX", "v", (False, -1000, 0))),
}


def make_table(rows, keys, seed=0):
    rng = np.random.default_rng(seed)
    return pd.DataFrame({"k": rng.integers(0, keys, rows), "t": rng.integers(0, 1 << 40, rows),
                         "v": rng.normal(0, 1, rows)})


def window_bytes_per_row(query):
    """Bytes per row the window kernels read and write (not the sort, not the scatter), from the shapes:
    heads per key 4 (row id) + 2 x 8 (key at i and i-1) + 2 x 1 (flags); positions 2 x 1 (flags, two passes) +
    1 (next flag) + 3 x 4 (ps, qs, dn) + 2 x 4 (ends, at most); frame kernel 2 x 4 (ps, pend) + the result.
    SUM adds the argument's gather (4 + 8 + 8), its scan (2 x 8 read, 8 + 8 + 3 x 4 written) and the frame's
    reads of the prefix at lo-1 and hi (2 x 32); MAX adds the gather, the running scan (2 x 8 read, 8 + 4
    written) and a sparse table of L = 10 levels (8 read + 8 written at level 0, 16 read + 8 written above),
    read twice (2 x 8) by the frame.  Reads of neighbours that hit a cache line another thread loaded are
    counted once per row."""
    heads = 2 * (4 + 16 + 2)
    positions = 2 + 1 + 12 + 8
    frame = 8
    if query == "row_number":
        return heads + positions + frame + 8
    gather = 4 + 8 + 8
    if query == "sum_rows10":
        return heads + positions + gather + (16 + 8 + 8 + 12) + frame + 64 + 8 + 1 / 8
    levels = 10
    return heads + positions + gather + (16 + 12) + (16 + 24 * (levels - 1)) + frame + 16 + 4 + 8 + 1 / 8


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        import torch
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def reference(df, query):
    from tests import query_ref as Q
    from tests import window_ref as W
    fn, arg, frame = QUERIES[query][1]
    kind, cells = W.window(Q.table(df), ["k"], [("t", True, False)], fn, arg, frame or (True, float("-inf"), 0))
    return kind, cells


def check(c, df, query):
    from tests import query_ref as Q
    kind, exp = reference(df, query)
    got = c.sql(f"SELECT {QUERIES[query][0]} AS o FROM w").compute()["o"]
    cells = [None if pd.isna(x) else (float(x) if kind in ("float", "bounded") else int(x)) for x in got]
    if kind in ("float", "bounded"):
        cells = [float("nan") if x is None else x for x in cells]
    Q.assert_result({"o": cells}, Q.Result({"o": exp}, {"o": kind}), what=f"{query} on {len(df)} rows")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--keys", type=float, default=1e6)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check-rows", type=float, default=1e6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows, keys, check_rows = int(a.rows), int(a.keys), int(min(a.check_rows, a.rows))
    # the sample keeps the table's rows per partition: its keys scale with it
    sample = make_table(check_rows, max(1, keys * check_rows // rows))
    for q in QUERIES:                                  # the reference runs before any device call
        reference(sample.head(min(len(sample), 64)), q)

    import torch
    from dask_sql_b200 import Context
    from dask_sql_b200 import executor as X
    torch.cuda.set_device(0)
    info = card()
    print(info, flush=True)
    c = Context()
    c.create_table("w", sample)
    for q in QUERIES:
        check(c, sample, q)
    del sample
    c.create_table("w", make_table(rows, keys))
    results = {}
    for q, (call, _) in QUERIES.items():
        sql = f"SELECT {call} AS o FROM w"
        for _ in range(a.warmup):
            c.sql(sql).persist()
        torch.cuda.synchronize()
        steps, split = [], {"window_sort": 0.0, "window_kernels": 0.0, "window_scatter": 0.0}
        for _ in range(a.steps):
            X.kernel_events = []
            t0 = time.perf_counter()
            c.sql(sql).persist()                       # the result stays on the device
            torch.cuda.synchronize()
            steps.append((time.perf_counter() - t0) * 1e3)
            for name, _, e0, e1 in X.kernel_events:
                if name in split:
                    split[name] += e0.elapsed_time(e1) / a.steps
            X.kernel_events = None
        bpr = window_bytes_per_row(q)
        kms = split["window_kernels"]
        results[q] = {"step_ms_median": round(float(np.median(steps)), 3), "step_ms": [round(s, 3) for s in steps],
                      "sort_ms": round(split["window_sort"], 3), "window_kernels_ms": round(kms, 3),
                      "scatter_ms": round(split["window_scatter"], 3), "window_bytes_per_row": round(bpr, 1),
                      "window_kernels_share_of_3.35TBps": round(bpr * rows / (kms * 1e-3) / HBM_BYTES_PER_S, 3)
                      if kms > 0 else None}
    line = json.dumps({"card": info, "rows": rows, "keys": keys, "checked_rows": check_rows, "verified": True,
                       "queries": results})
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
