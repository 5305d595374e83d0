"""DATE / TIMESTAMP on the device, three comparisons in one process, each pair alternated `--runs` times and
timed like bench.py (bench._time_query: CUDA events around `--steps` executions after `--warmup`):

1. C4 with DATE columns against C4 on the same day numbers as int64.  bench.py's C4 tables (seed 4): the
   fact's x in [-2^31, 2^31) is a DATE (days since 1970-01-01; x > DATE '1970-01-01' passes ~50 %, like
   x > 0) and the dim's flag in [0, 10) is a DATE (flag < DATE '1970-01-06' passes ~50 %, like flag < 5).
   The device bytes are the same tensors, so the same kernels should run in the same time.  Reports ms per
   step and b2_star_agg_kernel ms; grp must be identical and rev equal to the int64 run's.
2. SELECT y, SUM(val) ... GROUP BY y with y = EXTRACT(YEAR FROM ts) over `--rows` timestamp[us] rows: the
   b2_expr_eval pass alone (16 B/row: 8 in, 8 out) against 3.35 TB/s, and the whole query, against the same
   group-by over a precomputed year column.
3. WHERE EXTRACT(YEAR FROM ts) = 1995 against the hand-written range on ts: the rewrite makes both the same
   fused scan.

Prints one JSON line with the card's name, power limit and max SM clock.  Writes nothing.
usage: python scripts/bench_temporal.py [--steps 10] [--warmup 3] [--runs 3] [--rows 200000000]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

HBM_PEAK_GBS = 3350.0        # H100 SXM data sheet


def _relabel(table, logical):
    """The same device buffers under another logical type (DATE / TIMESTAMP ticks are int64 bytes)."""
    for part in table.partitions:
        for name, lg in logical.items():
            part[name].logical = lg
    table._schema = None
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--rows", type=int, default=200_000_000)
    ap.add_argument("--c4-rows", type=int, default=1_000_000_000)
    args = ap.parse_args()

    import torch
    import bench
    from bench import _time_query
    from bench_bitwise import card
    from dask_sql_b200 import Context, executor
    from dask_sql_b200 import expr as E
    from dask_sql_b200 import device as D
    from dask_sql_b200 import temporal as T
    from dask_sql_b200.table import DeviceTable

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    out = {"card": card(), "steps": args.steps, "warmup": args.warmup, "runs": args.runs}

    # ---- 1. C4: DATE columns against int64, the same tensors (bench.py's generator, seed 4)
    n = args.c4_rows
    g = torch.Generator(device=dev)
    g.manual_seed(4)
    fk = torch.randint(0, bench.DIM_ROWS, (n,), dtype=torch.int64, device=dev, generator=g)
    x = torch.randint(-2**31, 2**31, (n,), dtype=torch.int64, device=dev, generator=g)
    val = torch.rand(n, dtype=torch.float64, device=dev, generator=g)
    gd = torch.Generator(device=dev)
    gd.manual_seed(4)
    pk = torch.randperm(bench.DIM_ROWS, device=dev, generator=gd)
    flag = torch.randint(0, 10, (bench.DIM_ROWS,), dtype=torch.int64, device=dev, generator=gd)
    grp = torch.randint(0, bench.N_GROUPS, (bench.DIM_ROWS,), dtype=torch.int64, device=dev, generator=gd)
    c = Context()
    c.create_table("fact", {"fk": fk, "x": x, "val": val}, persist=True, npartitions=8)
    c.create_table("dim", {"pk": pk, "flag": flag, "grp": grp}, persist=True)
    c.create_table("fact_d", _relabel(DeviceTable.from_columns({"fk": fk, "x": x, "val": val}, 8),
                                      {"x": T.DATE_LOGICAL}))
    c.create_table("dim_d", _relabel(DeviceTable.from_columns({"pk": pk, "flag": flag, "grp": grp}, 1),
                                     {"flag": T.DATE_LOGICAL}))
    q_int = bench.QUERY
    q_date = ("SELECT d.grp, SUM(f.val) AS rev FROM fact_d f JOIN dim_d d ON f.fk = d.pk "
              "WHERE f.x > DATE '1970-01-01' AND d.flag < DATE '1970-01-06' GROUP BY d.grp")
    res = {"int64": {"ms": [], "b2_star_agg_kernel_ms": []}, "date": {"ms": [], "b2_star_agg_kernel_ms": []}}
    last = {}
    for _ in range(args.runs):
        for name, q in (("int64", q_int), ("date", q_date)):
            before = executor.stats["star_fused"]
            t, _, parts, launches = _time_query(torch, executor, c, q, args.steps, args.warmup, ())
            res[name]["ms"].append(round(t, 4))
            res[name]["b2_star_agg_kernel_ms"].append(_time_query.breakdown.get("b2_star_agg_kernel"))
            res[name]["star_fused"] = executor.stats["star_fused"] > before
            res[name]["launches_per_step"] = launches
            p = parts[0]
            order = torch.argsort(p["grp"].data)
            last[name] = (p["grp"].data[order], p["rev"].data[order])
    same_grp = bool(torch.equal(last["int64"][0], last["date"][0]))
    rel = float(((last["int64"][1] - last["date"][1]).abs() / last["int64"][1].abs().clamp_min(1e-300)).max().item())
    out["c4"] = {"fact_rows": n, "dim_rows": bench.DIM_ROWS, "query_date": q_date, "query_int64": q_int,
                 **res, "grp_identical": same_grp, "rev_max_rel_diff": rel}
    del c, fk, x, val, pk, flag, grp, last
    torch.cuda.empty_cache()

    # ---- 2. EXTRACT(YEAR FROM ts) GROUP BY over timestamp[us]
    m = args.rows
    g.manual_seed(7)
    lo = int(T.parse_timestamp("1980-01-01").ticks)
    hi = int(T.parse_timestamp("2030-01-01").ticks)
    ts = torch.randint(lo, hi, (m,), dtype=torch.int64, device=dev, generator=g)
    v = torch.rand(m, dtype=torch.float64, device=dev, generator=g)
    year_expr = T.extract("YEAR", E.ColRef("ts", E.I64, "datetime64[us]"))
    prog = E.compile_expr(year_expr, ["ts"])
    col = D.DeviceColumn(ts, None, E.I64, "datetime64[us]")
    year = D.expr_eval(prog, [col], m, False).data.clone()
    c = Context()
    c.create_table("t", _relabel(DeviceTable.from_columns({"ts": ts, "val": v}, 8), {"ts": "datetime64[us]"}))
    c.create_table("ty", {"y": year, "val": v}, persist=True, npartitions=8)
    ex_ms = []
    for _ in range(args.runs):
        outbuf = torch.empty(m, dtype=torch.int64, device=dev)
        for _ in range(args.warmup):
            D.expr_eval(prog, [col], m, False, out=outbuf)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            D.expr_eval(prog, [col], m, False, out=outbuf)
        e1.record()
        torch.cuda.synchronize()
        ex_ms.append(round(e0.elapsed_time(e1) / args.steps, 4))
    assert torch.equal(outbuf, year)
    q_ext = "SELECT y, SUM(val) AS s FROM (SELECT EXTRACT(YEAR FROM ts) AS y, val FROM t) AS q GROUP BY y"
    q_pre = "SELECT y, SUM(val) AS s FROM ty GROUP BY y"
    g_ms = {"extract": [], "precomputed": []}
    g_breakdown = {}
    got = {}
    for _ in range(args.runs):
        for name, q in (("extract", q_ext), ("precomputed", q_pre)):
            t, _, parts, _ = _time_query(torch, executor, c, q, args.steps, args.warmup, ())
            g_ms[name].append(round(t, 4))
            g_breakdown[name] = _time_query.breakdown
            p = parts[0]
            order = torch.argsort(p["y"].data)
            got[name] = (p["y"].data[order], p["s"].data[order])
    best = min(ex_ms)
    out["extract_year_groupby"] = {
        "rows": m, "unit": "us", "expr_eval_ms": ex_ms,
        "expr_eval_gbs_best": round(16 * m / (best * 1e-3) / 1e9, 1), "hbm_peak_gbs": HBM_PEAK_GBS,
        "expr_eval_frac_of_peak_best": round(16 * m / (best * 1e-3) / 1e9 / HBM_PEAK_GBS, 3),
        "query_ms": g_ms, "breakdown_last_run": g_breakdown,
        "groups_identical": bool(torch.equal(got["extract"][0], got["precomputed"][0])),
        "sums_max_rel_diff": float(((got["extract"][1] - got["precomputed"][1]).abs()
                                    / got["precomputed"][1].abs()).max().item())}

    # ---- 3. WHERE EXTRACT(YEAR FROM ts) = 1995 against the hand-written range
    y0, y1 = T.parse_timestamp("1995-01-01").ticks, T.parse_timestamp("1996-01-01").ticks
    q_year = "SELECT SUM(val) AS s, COUNT(*) AS n FROM t WHERE EXTRACT(YEAR FROM ts) = 1995"
    q_range = ("SELECT SUM(val) AS s, COUNT(*) AS n FROM t WHERE ts >= TIMESTAMP '1995-01-01 00:00:00' "
               "AND ts < TIMESTAMP '1996-01-01 00:00:00'")
    f_ms = {"year": [], "range": []}
    f_breakdown, f_launches, f_got = {}, {}, {}
    for _ in range(args.runs):
        for name, q in (("year", q_year), ("range", q_range)):
            t, _, parts, launches = _time_query(torch, executor, c, q, args.steps, args.warmup, ())
            f_ms[name].append(round(t, 4))
            f_breakdown[name] = _time_query.breakdown
            f_launches[name] = launches
            f_got[name] = (float(parts[0]["s"].data[0].item()), int(parts[0]["n"].data[0].item()))
    want_n = int(((ts >= y0) & (ts < y1)).sum().item())
    out["year_filter"] = {"rows": m, "query_year": q_year, "query_range": q_range, "ms": f_ms,
                          "breakdown_last_run": f_breakdown, "launches_per_step": f_launches,
                          "identical": f_got["year"] == f_got["range"], "count_ok": f_got["year"][1] == want_n}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
