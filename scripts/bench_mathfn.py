"""Throughput of the numeric SQL functions in b2_expr_eval, and what they cost inside queries.

1. Per function: b2_expr_eval over N doubles (LOAD, function) timed with CUDA events, as ms per launch, G rows/s
   and the fraction of 3.35 TB/s (the H100 SXM's HBM3 data-sheet bandwidth) at 16 B/row (8 B read, 8 B written;
   the validity words are 1/32 of that and left out).
2. Two query pairs through Context.sql(), timed alternately for three rounds: SUM(ROUND(v, 2)) against SUM(v),
   and WHERE LN(x) > 0 against WHERE x > 1.
Prints the card's name and power limit first.  Usage: python scripts/bench_mathfn.py [--rows 2e8] [--iters 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BYTES = 3.35e12
FUNCS = ["ceil", "floor", "truncate", "round", "sign", "degrees", "radians", "sqrt", "exp", "ln", "log10", "cbrt",
         "sin", "cos", "tan", "cot", "asin", "acos", "atan", "atan2", "power", "mod", "power_i"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def program(name):
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import expr as E
    x, y = E.ColRef("x", E.F64), E.ColRef("y", E.F64)
    if name == "power_i":
        e = E.math("power", [E.ColRef("i", E.I64), 3])
    elif name in ("atan2", "power", "mod"):
        e = E.math(name, [x, y])
    else:
        e = E.math(name, [x], 2 if name == "round" else 0)
    return E.compile_expr(e, ["x", "y", "i"]), L


def kernel_table(rows, iters):
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(rows, generator=g, device=dev, dtype=torch.float64) * 2.0 - 0.5
    y = torch.rand(rows, generator=g, device=dev, dtype=torch.float64) * 3.0 + 0.25
    i = torch.randint(-1000, 1000, (rows,), generator=g, device=dev, dtype=torch.int64)
    out = torch.empty(rows, device=dev, dtype=torch.int64)
    valid = torch.empty((rows + 31) // 32, device=dev, dtype=torch.int32)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = []
    for name in FUNCS:
        p, L = program(name)
        cols = (L.Col * 3)()
        for k, t in enumerate((x, y, i)):
            cols[k].data, cols[k].valid, cols[k].dtype = t.data_ptr(), 0, L.I64 if t.dtype == torch.int64 else L.F64

        def launch():
            L.expr_eval(C.byref(p), cols, 3, rows, C.c_void_p(out.data_ptr()), C.c_void_p(valid.data_ptr()), stream)
        for _ in range(3):
            launch()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(iters):
            launch()
        stop.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(stop) / iters
        nread = 16 if name in ("atan2", "power", "mod") else 8
        res.append(dict(fn=name, ms=round(ms, 3), grows_s=round(rows / ms / 1e6, 2),
                        hbm_frac_16B=round(16 * rows / (ms * 1e-3) / PEAK_BYTES, 3), bytes_per_row=nread + 8))
        print(json.dumps(res[-1]), flush=True)
    return res


def query_pairs(rows, rounds):
    import pandas as pd
    import torch
    from dask_sql_b200 import Context
    rng = np.random.default_rng(1)
    t = pd.DataFrame({"v": rng.uniform(-100, 100, rows), "x": rng.uniform(0.0, 2.0, rows)})
    c = Context()
    c.create_table("t", t, npartitions=1)
    pairs = [("SELECT SUM(ROUND(v, 2)) AS s FROM t", "SELECT SUM(v) AS s FROM t"),
             ("SELECT COUNT(*) AS n FROM t WHERE LN(x) > 0", "SELECT COUNT(*) AS n FROM t WHERE x > 1")]
    out = []
    for a, b in pairs:
        for q in (a, b):
            c.sql(q).compute()
        times = {a: [], b: []}
        for _ in range(rounds):
            for q in (a, b):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(5):
                    c.sql(q).compute()
                torch.cuda.synchronize()
                times[q].append((time.perf_counter() - t0) / 5 * 1e3)
        out.append({"query": a, "ms": [round(v, 2) for v in times[a]],
                    "baseline": b, "baseline_ms": [round(v, 2) for v in times[b]]})
        print(json.dumps(out[-1]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=2e8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--query-rows", type=float, default=5e7)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mathfn.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    kernel_table(int(args.rows), args.iters)
    query_pairs(int(args.query_rows), args.rounds)


if __name__ == "__main__":
    main()
