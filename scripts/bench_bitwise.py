"""C2b against C2i on the same data: GROUP BY key over 200M rows, 1M uniform keys, int64 values in [-1000, 1000],
8 partitions (bench.py's C2i, same seed), as  SUM(val)  and as  BIT_OR(val).  The SUM takes one REDG.E.ADD.64 per
row, the BIT_OR one REDG.E.OR.64: does the L2 serve the bitwise reduction at the same rate?

Both queries run in the same process, alternating `--runs` times, timed like bench.py (CUDA events around
`--steps` executions after `--warmup`).  Every group of both results is checked on the full data with plain torch:
the SUM against index_add_, and bit b of the BIT_OR set iff the index_add_ of (val >> b) & 1 over the group is
> 0.  Prints one JSON line with the card's name and power limit.  Writes nothing.
usage: python scripts/bench_bitwise.py [--steps 10] [--warmup 3] [--runs 3] [--scale 1.0]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BITS = (0, 1, 2, 5, 9, 10, 11, 63)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()

    import torch
    from bench import _time_query
    from dask_sql_b200 import Context, executor

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    n, nkeys = int(2e8 * args.scale), 1_000_000
    g = torch.Generator(device=dev)
    g.manual_seed(2)
    key = torch.randint(0, nkeys, (n,), dtype=torch.int64, device=dev, generator=g)
    val = torch.randint(-1000, 1001, (n,), dtype=torch.int64, device=dev, generator=g)
    c = Context()
    c.create_table("t", {"key": key, "val": val}, persist=True, npartitions=8)
    queries = {"C2i": "SELECT key, SUM(val) AS s FROM t GROUP BY key",
               "C2b": "SELECT key, BIT_OR(val) AS s FROM t GROUP BY key"}

    cnt = torch.bincount(key, minlength=nkeys)
    present = cnt > 0
    want_keys = torch.nonzero(present).reshape(-1)
    exp_sum = torch.zeros(nkeys, dtype=torch.int64, device=dev).index_add_(0, key, val)[present]
    ms = {name: [] for name in queries}
    verified = {}
    for _ in range(args.runs):
        for name, q in queries.items():
            t, _, parts, _ = _time_query(torch, executor, c, q, args.steps, args.warmup, ())
            ms[name].append(t)
            k_out, s_out = parts[0]["key"].data, parts[0]["s"].data
            ok = bool(torch.equal(k_out, want_keys))
            if ok and name == "C2i":
                ok = bool(torch.equal(s_out, exp_sum))
            elif ok:
                for b in BITS:
                    nb = torch.zeros(nkeys, dtype=torch.int64, device=dev).index_add_(0, key, (val >> b) & 1)
                    ok = ok and bool(torch.equal((s_out >> b) & 1, (nb[present] > 0).to(torch.int64)))
            verified[name] = verified.get(name, True) and ok
    print(json.dumps({"card": card(), "rows": n, "keys": nkeys, "partitions": 8, "steps": args.steps,
                      "warmup": args.warmup, "ms_per_step": ms, "verified": verified,
                      "checked": {"C2i": "every group against torch index_add_",
                                  "C2b": f"every group, bits {list(BITS)}: set iff index_add_ of (val >> b) & 1 > 0"},
                      "queries": queries}))


if __name__ == "__main__":
    main()
