"""VARCHAR measurements (DESIGN.md section 4), printed with the card's name and power limit:

1. The Q3 shape with a VARCHAR predicate (`segment = 'BUILDING'`) and VARCHAR group key against its
   int64-coded twin: launches and step times, the two alternating.
2. `WHERE comment NOT LIKE '%special%requests%'` over a high-cardinality column: b2_str_like over the
   dictionary (bytes read / time / 3.35e12) and the B2_OP_MAP mask pass over the rows.
3. A string-key join with different dictionaries against the same join on int64 keys, with the
   translation kernel (b2_str_lower_bound) and its MAP pass timed on their own.

    python scripts/bench_strings.py [--scale 1.0]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps / 1e3


def random_strings(n, lo, hi, rng, inject=None, rate=0.0):
    """n random lowercase strings of lo..hi bytes as a large_string array (optionally with `inject` spliced in)"""
    import pyarrow as pa
    lens = rng.integers(lo, hi + 1, n)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    chars = rng.integers(97, 123, int(off[-1]), dtype=np.uint8)
    if inject is not None:
        w = np.frombuffer(inject.encode(), dtype=np.uint8)
        rows = np.nonzero((rng.random(n) < rate) & (lens >= len(w)))[0]
        for r in rows:
            chars[off[r]: off[r] + len(w)] = w
    return pa.LargeStringArray.from_buffers(n, pa.py_buffer(off.tobytes()), pa.py_buffer(chars.tobytes()))


def q3(scale, steps):
    import pandas as pd
    import torch
    from dask_sql_b200 import Context, executor
    rng = np.random.default_rng(0)
    nd, nf = int(1.5e6 * scale), int(1e8 * scale)
    segs = np.array(["AUTOMOBILE", "BUILDING", "FURNITURE", "HOUSEHOLD", "MACHINERY"], dtype=object)
    seg_i, grp_i = rng.integers(0, 5, nd), rng.integers(0, 1000, nd)
    grp_words = np.array(["group-%04d" % i for i in range(1000)], dtype=object)
    dim = pd.DataFrame({"pk": rng.permutation(nd), "seg_i": seg_i, "grp_i": grp_i,
                        "segment": pd.Series(segs[seg_i]).astype("category"),
                        "grp": pd.Series(grp_words[grp_i]).astype("category")})
    fact = pd.DataFrame({"fk": rng.integers(0, nd, nf), "x": rng.integers(-2**31, 2**31, nf), "val": rng.random(nf)})
    c = Context()
    c.create_table("fact", fact, persist=True)
    c.create_table("dim", dim, persist=True)
    base = "SELECT d.{g}, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fk = d.pk WHERE f.x > 0 AND {w} GROUP BY d.{g}"
    qs = {"varchar": base.format(g="grp", w="d.segment = 'BUILDING'"),
          "int64": base.format(g="grp_i", w="d.seg_i = 1")}
    out = {k: {"ms": [], "launches": None, "star_fused": None} for k in qs}
    res = {}
    for k, q in qs.items():               # warm-up, plan cache, results
        res[k] = c.sql(q).compute()
    for _ in range(steps):
        for k, q in qs.items():
            l0, s0 = executor.stats["launches"], executor.stats["star_fused"]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            c.sql(q).compute()
            torch.cuda.synchronize()
            out[k]["ms"].append((time.perf_counter() - t0) * 1e3)
            out[k]["launches"], out[k]["star_fused"] = executor.stats["launches"] - l0, executor.stats["star_fused"] - s0
    a = res["varchar"].assign(g=lambda d: d["grp"].astype(str)).sort_values("g")["rev"].to_numpy()
    b = res["int64"].assign(g=lambda d: d["grp_i"].map(lambda i: "group-%04d" % i)).sort_values("g")["rev"].to_numpy()
    for k in out:
        ms = sorted(out[k]["ms"])
        out[k]["median_ms"], out[k]["min_ms"], out[k]["max_ms"] = ms[len(ms) // 2], ms[0], ms[-1]
        del out[k]["ms"]
    out["same_result"] = bool(len(a) == len(b) and np.allclose(a, b, rtol=1e-9))
    out["rows"] = {"fact": nf, "dim": nd}
    return out


def like(scale, reps):
    import torch
    from dask_sql_b200 import expr as E
    from dask_sql_b200 import strings as S
    from dask_sql_b200 import executor
    from dask_sql_b200.device import DeviceColumn
    from dask_sql_b200.executor import Part, eval_expr
    from dask_sql_b200.expr import ColRef
    import pyarrow.compute as pc
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(1)
    nd, nrows = int(1e7 * scale), int(5e7 * scale)
    arr = random_strings(nd, 30, 90, rng, inject="specialxxrequests", rate=0.01)
    arr = pc.unique(arr)
    d = S.Dictionary(arr.take(pc.array_sort_indices(arr)))
    lg = S.Varchar(d)
    off, chars = d.device(dev)
    nbytes = int(d.offsets[-1]) + 8 * (len(d) + 1)
    t_like = timed(lambda: S.like_table(d, "%special%requests%", "\\", False, dev), reps)
    codes = torch.randint(0, len(d), (nrows,), device=dev, dtype=torch.int64)
    part = Part({"c": DeviceColumn(codes, None, 0, lg)}, nrows)
    e = E.unop("not", S.like(ColRef("c", 0, lg), "%special%requests%"))
    e.args[0].param.column(dev)            # the per-entry table is computed once per plan, outside the row pass
    t_map = timed(lambda: eval_expr(part, e), reps)
    hits = int(S.like_table(d, "%special%requests%", "\\", False, dev).data.sum().item())
    return {"dict_entries": len(d), "avg_bytes": int(d.offsets[-1]) / max(1, len(d)), "rows": nrows,
            "matching_entries": hits,
            "b2_str_like_ms": t_like * 1e3, "b2_str_like_bytes": nbytes,
            "b2_str_like_share_of_hbm_peak": nbytes / t_like / 3.35e12,
            "map_pass_ms": t_map * 1e3, "map_pass_bytes": nrows * 8 + nrows + len(d),
            "launches": executor.stats["launches"]}


def join(scale, steps):
    import pyarrow as pa
    import torch
    from dask_sql_b200 import Context
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import strings as S
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(2)
    nb, npr = int(1e6 * scale), int(1e8 * scale)
    words = [("key-%08d" % i) for i in range(int(1.5 * nb))]
    dim_words = pa.array(words[: nb], type=pa.large_string())                 # partly overlapping
    fact_words = pa.array(words[nb // 2:], type=pa.large_string())
    dd, fd = S.Dictionary(dim_words), S.Dictionary(fact_words)
    dim_codes = np.arange(nb)
    fact_codes = rng.integers(0, len(fd), npr)
    c = Context()
    c.create_table("dim", pa.table({"s": pa.DictionaryArray.from_arrays(pa.array(dim_codes), dim_words),
                                    "k": words_to_int(dim_words, 0), "v": rng.random(nb)}), persist=True)
    c.create_table("fact", pa.table({"s": pa.DictionaryArray.from_arrays(pa.array(fact_codes), fact_words),
                                     "k": fact_codes + nb // 2, "x": rng.integers(0, 100, npr)}), persist=True)
    qs = {"varchar": "SELECT f.x, d.v FROM fact f JOIN dim d ON f.s = d.s",
          "int64": "SELECT f.x, d.v FROM fact f JOIN dim d ON f.k = d.k"}
    ms = {k: [] for k in qs}
    rows = {}
    for k, q in qs.items():
        rows[k] = len(c.sql(q).compute())
    for _ in range(steps):
        for k, q in qs.items():
            frame = c.sql(q)
            from dask_sql_b200.executor import execute
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            parts = execute(frame)
            n = sum(p.n for p in parts)
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3)
            assert n == rows[k]
    t_lb = timed(lambda: S.lower_bound_table(fd, dd, L.STR_LB_MATCH, dev), 20)
    return {"probe_rows": npr, "build_rows": nb, "rows_out": rows,
            "median_ms": {k: sorted(v)[len(v) // 2] for k, v in ms.items()},
            "translate_b2_str_lower_bound_ms": t_lb * 1e3,
            "note": "the smaller (build) side's key is translated: its MAP pass runs over build_rows"}


def words_to_int(words, base):
    return np.arange(len(words), dtype=np.int64) + base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--only", default="q3,like,join")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    res = {"card": card()}
    for name in args.only.split(","):
        res[name] = {"q3": q3, "like": like, "join": join}[name](args.scale, args.steps)
        print(json.dumps({name: res[name]}), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
