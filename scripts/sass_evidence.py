"""<out-dir>/sass_<kernel>.txt: opcode histogram + the memory / atomic / warp-level instructions of the
hot kernels, straight from `cuobjdump -sass dask-sql_b200/libb200sql.so` (one sm_90a cubin).  Needs no GPU.
usage: python scripts/sass_evidence.py [out-dir]      (default build/sass, git-ignored)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "dask-sql_b200", "libb200sql.so")
OUT = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "build", "sass")
WANT = {
    "star_agg": r"b2_star_agg_kernel",
    "join_stream": r"b2_join_stream_kernelILb1ELi3ELb1EE",
    "join_agg_fast": r"b2_join_agg_fast_kernelILb1ELi0E",
    "part_scatter_block": r"b2_part_scatter_kernel",
    "peer_merge_w8": r"b2_peer_merge_kernelILi8E",
    "groupby_dense": r"b2_groupby_dense_kernel",
    "groupby_dense_hh": r"b2_groupby_dense_hh_kernel",
    "groupby_dense_grouped": r"b2_groupby_dense_grouped_kernel",
    "scan_agg": r"b2_scan_agg_kernelILb0E",
    "window_heads": r"b2_window_heads_kernel",
    "window_rescan_sumf": r"b2_window_rescan_kernelI14b2_win_sumf_op",
    "window_rescan_pos": r"b2_window_rescan_kernelI13b2_win_pos_op",
    "window_rmq_level": r"b2_window_rmq_level_kernel",
    "window_frame": r"b2_window_frame_kernel",
}
INTERESTING = re.compile(r"\b(LDG|STG|REDG|ATOMG|ATOMS|ATOM|RED|LDS|STS|MATCH|VOTE|SHFL|REDUX|UBLKCP|SYNCS|BAR|CCTL|LDGSTS|UTMALDG|LD|ST|NANOSLEEP|MEMBAR|ERRBAR)\b")

sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
arch = re.search(r"arch = (\S+)", sass)
funcs = re.split(r"\n\s*Function : ", sass)
by_name = {}
for f in funcs[1:]:
    name, _, body = f.partition("\n")
    by_name[name.strip()] = body

os.makedirs(OUT, exist_ok=True)
for label, pat in WANT.items():
    hits = [n for n in by_name if re.search(pat, n)]
    if not hits:
        print("missing", label)
        continue
    name = hits[0]
    ops = collections.Counter()
    lines = []
    for ln in by_name[name].splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", ln)
        if not m:
            continue
        ins = m.group(2).strip()
        parts = ins.split()
        op = parts[1] if parts[0].startswith("@") and len(parts) > 1 else parts[0]
        ops[op.split(".")[0]] += 1
        if INTERESTING.search(ins):
            lines.append(f"  /*{m.group(1)}*/ {ins}")
    total = sum(ops.values())
    out = os.path.join(OUT, f"sass_{label}.txt")
    with open(out, "w") as fh:
        fh.write(f"# {name}\n# cuobjdump -sass dask-sql_b200/libb200sql.so ({arch.group(1) if arch else '?'}); {total} SASS instructions\n")
        fh.write("# opcode histogram (static):\n")
        for op, n in ops.most_common(24):
            fh.write(f"  {op:12s} {n:6d}  {100.0 * n / total:5.1f} %\n")
        fh.write("# memory / atomic / warp-level instructions in program order:\n")
        fh.write("\n".join(lines[:400]) + "\n")
    print(out, total, "instructions;", ", ".join(f"{o} {n}" for o, n in ops.most_common(6)))
