#!/usr/bin/env python
"""Where a C4 step goes on one GPU: the bench.py headline query (same generator and seeds, 1e9 fact rows
in 8 partitions, 10M dim rows, 1M groups) timed with CUDA events per phase of PreparedStar.run (build /
scan / ...) and per launch of the ranked-bitmap build (the memsets, every mark, the rank, every fill, and the pack of the
staged 21-bit slots), next to the step time and the b2_star_agg_kernel time: one launch per step over all 8
fact partitions (b2_star_agg_multi), or one per partition with B200SQL_STAR_PER_PART=1, whose fill updates
the packed slots in place by CAS and has no pack.  One JSON line per phase and per launch, in ms
per step and per call, each carrying the card's name and power limit; then one "bytes" line: the bytes per
fact and per dim row that the prepared plan's scans physically read (int64 columns streamed as their 32-bit
images, DeviceColumn.star_image, unless B200SQL_NO_NARROW=1) against the logical 24 B per fact row that
bench.py's roofline divides by, and the probe's physical bandwidth from the b2_star_agg_kernel time.

    python scripts/star_step_breakdown.py --steps 10 --warmup 3
    B200SQL_STAR_PER_PART=1 python scripts/star_step_breakdown.py --steps 10 --warmup 3
    B200SQL_NO_NARROW=1 python scripts/star_step_breakdown.py --steps 10 --warmup 3

B200SQL_LIB selects another build of libb200sql.so (the C-ABI is the same), so two builds can be
compared by the same Python."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

QUERY = ("SELECT d.grp, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fk = d.pk "
         "WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp")
DIM_ROWS = 10_000_000
N_GROUPS = 1_000_000
PARTITIONS = 8


def card(index):
    """(name, power limit in W) of the device, read through NVML"""
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(index)
        name = nv.nvmlDeviceGetName(h)
        return (name.decode() if isinstance(name, bytes) else name), nv.nvmlDeviceGetPowerManagementLimit(h) / 1000
    except Exception as e:  # noqa: BLE001 -- the timings stand without it; say why it is missing
        return f"unknown ({type(e).__name__})", None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--label", default=os.environ.get("B200SQL_LIB", "in-tree") +
                    (" int64" if os.environ.get("B200SQL_NO_NARROW") == "1" else " images") +
                    (" per-partition" if os.environ.get("B200SQL_STAR_PER_PART") == "1" else ""))
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")

    import torch
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    from dask_sql_b200 import Context, executor
    from dask_sql_b200 import _lib as L

    # the tables of bench.py at one GPU
    n = int(args.rows)
    g = torch.Generator(device=dev)
    g.manual_seed(4)
    fk = torch.randint(0, DIM_ROWS, (n,), dtype=torch.int64, device=dev, generator=g)
    x = torch.randint(-2**31, 2**31, (n,), dtype=torch.int64, device=dev, generator=g)
    val = torch.rand(n, dtype=torch.float64, device=dev, generator=g)
    gd = torch.Generator(device=dev)
    gd.manual_seed(4)
    pk = torch.randperm(DIM_ROWS, device=dev, generator=gd)
    flag = torch.randint(0, 10, (DIM_ROWS,), dtype=torch.int64, device=dev, generator=gd)
    grp = torch.randint(0, N_GROUPS, (DIM_ROWS,), dtype=torch.int64, device=dev, generator=gd)
    c = Context()
    c.create_table("fact", {"fk": fk, "x": x, "val": val}, persist=True, npartitions=PARTITIONS, distribution="local")
    c.create_table("dim", {"pk": pk, "flag": flag, "grp": grp}, persist=True, distribution="local")

    # CUDA events around every launch of the lookup build; `launches` is None outside the timed steps
    launches = None
    in_build = [False]

    def timed(name, fn):
        def call(*a):
            if launches is None or not in_build[0]:
                return fn(*a)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*a)
            e1.record()
            launches.append((name, e0, e1))
            return rc
        return call

    for attr, name in (("memset", "memset"), ("star_build_mark_narrow", "mark"), ("star_build_rank", "rank"),
                       ("star_build_fill_narrow", "fill"), ("star_build_pack", "pack")):
        setattr(L, attr, timed(name, getattr(L, attr)))
    build = executor._star_bitmap_build

    def build_flagged(*a):
        in_build[0] = True
        try:
            return build(*a)
        finally:
            in_build[0] = False

    executor._star_bitmap_build = build_flagged

    def step():
        return executor.execute(c.sql(QUERY), top=True)

    for _ in range(args.warmup):
        parts = step()
    torch.cuda.synchronize()
    launches = []
    executor.phase_events = []
    executor.kernel_events = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        parts = step()
    e1.record()
    torch.cuda.synchronize()
    pev, kev = executor.phase_events, executor.kernel_events
    executor.phase_events = executor.kernel_events = None
    assert executor.stats["star_fused"] > 0, "the query did not run the fused star pipeline"

    gpu, watts = card(0)
    common = {"label": args.label, "gpu": gpu, "power_limit_w": watts, "steps": args.steps, "rows": n,
              "groups_out": int(parts[0].n)}

    def emit(kind, name, ms, count):
        print(json.dumps({"kind": kind, "name": name, "ms_per_step": round(ms / args.steps, 4),
                          "calls_per_step": count / args.steps, "ms_per_call": round(ms / count, 4), **common}),
              flush=True)

    emit("step", "step", e0.elapsed_time(e1), args.steps)
    for kind, recs in (("phase", [(r[0], r[1], r[2]) for r in pev]), ("launch", launches),
                       ("kernel", [(r[0], r[2], r[3]) for r in kev])):
        tot, cnt = {}, {}
        for name, a, b in recs:
            tot[name] = tot.get(name, 0.0) + a.elapsed_time(b)
            cnt[name] = cnt.get(name, 0) + 1
        for name in tot:
            emit(kind, name, tot[name], cnt[name])

    # bytes per row as the plan's scan descriptors point at them (validity bitmaps: 1/8 B per row)
    width = {L.I64: 8, L.F64: 8, L.U8: 1, L.U32: 4}
    prep = executor.PreparedStar._live[-1]

    def row_bytes(launches):
        s = launches[0][0]
        return sum(width[s.cols[i].dtype] + (0.125 if s.cols[i].valid else 0) for i in range(s.ncols))

    images = [(s.cols[i].dtype == L.U32) for s, *_ in prep.fact_launch + prep.dim_launch for i in range(s.ncols)]
    fact_b = row_bytes(prep.fact_launch)
    probe_ms = sum(r[2].elapsed_time(r[3]) for r in kev if r[0] == "b2_star_agg_kernel") / args.steps
    print(json.dumps({"kind": "bytes", "fact_bytes_per_row": fact_b, "fact_bytes_per_row_logical": 24,
                      "dim_bytes_per_row": row_bytes(prep.dim_launch), "image_columns": sum(images),
                      "scan_columns": len(images), "probe_gbs_physical": round(n * fact_b / probe_ms / 1e6, 1),
                      "probe_frac_of_3350_gbs": round(n * fact_b / probe_ms / 1e6 / 3350, 3),
                      "hbm_allocated_gb": round(torch.cuda.memory_allocated(dev) / 1e9, 2), **common}), flush=True)


if __name__ == "__main__":
    main()
