"""Measure IN / EXISTS subqueries on one GPU (DESIGN.md section 4, "Subquery marks").

  python scripts/bench_subquery.py [--rows 1e8] [--inner 2.5e7] [--steps 3] [--warmup 1] [--check-rows 1e6]
                                   [--out FILE]

Tables (seeded): o (`rows` rows: int64 key a over rows/4 values, int64 b, int64 c) and i (`inner` rows: int64 x
over the same key range, int64 y, int64 z).  Queries, each ending in a COUNT(*):
  q4   EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.y < o.b)                 a Q4-shaped pair term
  q21  EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.z <> o.c)                a Q21-shaped <> pair term
  q16  o.a NOT IN (SELECT x FROM i WHERE y > 90)                              a Q16-shaped NOT IN
  q17  o.b < (SELECT 0.5 * AVG(y) FROM i WHERE i.x = o.a)                    a Q17-shaped correlated AVG, run as
                                                                             a LEFT JOIN on the grouped body (no mark)
For each: the step time (host clock around a query that ends in a device synchronise) and the b2_join_mark time
by CUDA events (executor.kernel_events); the bytes per probe row the mark moves, modelled from the shapes
(mark_bytes_per_row), and that model over the mark time as a share of the data sheet's 3.35 TB/s.  Before
timing, each query runs on the first `check-rows` outer rows and is compared with sqlite3.  Prints the card's
name, power limit and SM clock, then one JSON line."""
import argparse
import json
import os
import sqlite3
import subprocess
import sys
import time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
QUERIES = {
    "q4": ("EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.y < o.b)", 1),
    "q21": ("EXISTS (SELECT * FROM i WHERE i.x = o.a AND i.z <> o.c)", 1),
    "q16": ("o.a NOT IN (SELECT x FROM i WHERE y > 90)", 0),
    "q17": ("o.b < (SELECT 0.5 * AVG(y) FROM i WHERE i.x = o.a)", None),
}


def make_tables(rows, inner, seed=0):
    rng = np.random.default_rng(seed)
    keys = max(1, rows // 4)
    o = pd.DataFrame({"a": rng.integers(0, keys, rows), "b": rng.integers(0, 100, rows),
                      "c": rng.integers(0, 10, rows)})
    i = pd.DataFrame({"x": rng.integers(0, keys, inner), "y": rng.integers(0, 100, inner),
                      "z": rng.integers(0, 10, inner)})
    return o, i


def mark_bytes_per_row(nterms, inner, keys):
    """model: the probe key (8 B) and each pair term's probe value (8 B), the mark byte and 1/8 of a validity
    byte, one chain head (4 B), and per candidate (inner / keys on average) a next link (4 B), its key (8 B) and
    its pair-term values (8 B each) -- every candidate visited, no cache reuse."""
    cand = inner / keys
    return 8 + 8 * nterms + 1 + 1 / 8 + 4 + cand * (4 + 8 + 8 * nterms)


def card():
    q = "name,power.limit,clocks.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def sql_of(pred):
    return f"SELECT COUNT(*) AS n FROM o WHERE {pred}"


def check(Context, rows, inner):
    o, i = make_tables(rows, inner, seed=1)
    c = Context()
    c.create_table("o", o, npartitions=4)
    c.create_table("i", i)
    db = sqlite3.connect(":memory:")
    o.to_sql("o", db, index=False)
    i.to_sql("i", db, index=False)
    db.execute("CREATE INDEX ix ON i (x)")
    for name, (pred, _) in QUERIES.items():
        got = int(c.sql(sql_of(pred), return_futures=False)["n"].iloc[0])
        want = db.execute(sql_of(pred)).fetchone()[0]
        if got != want:
            raise SystemExit(f"{name}: {got} rows, sqlite {want}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--inner", type=float, default=2.5e7)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check-rows", type=float, default=1e6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_subquery.py measures on a CUDA device; none is visible")
    from dask_sql_b200 import Context, executor

    gpu = card()
    print(gpu)
    check(Context, int(args.check_rows), int(args.check_rows) // 4)
    rows, inner = int(args.rows), int(args.inner)
    o, i = make_tables(rows, inner)
    c = Context()
    c.create_table("o", o, persist=True, npartitions=8)
    c.create_table("i", i, persist=True)
    del o, i
    result = {"card": gpu, "rows": rows, "inner": inner, "queries": {}}
    for name, (pred, nterms) in QUERIES.items():
        sql = sql_of(pred)
        for _ in range(args.warmup):
            c.sql(sql, return_futures=False)
        steps, marks = [], []
        for _ in range(args.steps):
            executor.kernel_events = []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            c.sql(sql, return_futures=False)
            torch.cuda.synchronize()
            steps.append(time.perf_counter() - t0)
            marks.append(sum(s.elapsed_time(e) / 1e3 for k, _, s, e in executor.kernel_events if k == "b2_join_mark"))
            executor.kernel_events = None
        step, mark = float(np.median(steps)), float(np.median(marks))
        if nterms is None:
            result["queries"][name] = {"step_s": step}
            print(f"{name}: step {step * 1e3:.1f} ms")
            continue
        bpr = mark_bytes_per_row(nterms, inner, max(1, rows // 4))
        result["queries"][name] = {"step_s": step, "mark_s": mark, "model_bytes_per_row": bpr,
                                   "model_share_of_3.35TBps": bpr * rows / mark / HBM_BYTES_PER_S if mark else None}
        print(f"{name}: step {step * 1e3:.1f} ms, b2_join_mark {mark * 1e3:.1f} ms, model {bpr:.1f} B/row")
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
