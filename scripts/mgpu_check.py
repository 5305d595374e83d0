"""Multi-GPU parity check, run under torchrun (one process per GPU, NCCL):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29511 scripts/mgpu_check.py

Every rank holds a shard of the fact table; the dim table lives on rank 0 only ('root') and is
broadcast by the join; partial aggregates are reduce-scattered by key range (dense) or tree-merged
(hash).  Results are compared with the oracle on the full data.

The data is built so that a merge that loses group existence cannot pass: a large share of the
group slots is hit by NO row (sparse group ids, filtered-out dim rows, unreferenced keys), NULL
group keys and NULL join keys occur, and every check compares the exact set of groups."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import pandas as pd
import torch
import torch.distributed as dist

from dask_sql_b200 import Context, executor
from dask_sql_b200.parallel import shard_bounds
from oracle import pandas_oracle as O


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    rng = np.random.default_rng(7)
    nd, nf = 50_000, 2_000_000
    grp = pd.array(rng.integers(0, 20_000, nd) * 3, dtype="Int64")          # 2/3 of the slots can never be hit
    grp[rng.random(nd) < 0.02] = pd.NA                                      # NULL group keys
    dim = pd.DataFrame({"pk": rng.permutation(nd).astype(np.int64), "flag": rng.integers(0, 10, nd), "grp": grp})
    fk = pd.array(rng.integers(0, int(nd * 0.8), nf), dtype="Int64")        # 20 % of the dim rows are never referenced
    fk[rng.random(nf) < 0.01] = pd.NA                                       # NULL join keys never match
    fact = pd.DataFrame({"fk": fk, "x": rng.integers(-2**31, 2**31, nf), "val": rng.random(nf),
                         "skey": rng.integers(0, 30_000, nf) * 1_000_003 - 17,
                         "gk": rng.integers(0, 5_000, nf) * 7 + 11})
    lo, hi = shard_bounds(nf, rank, world)
    c = Context()
    c.create_table("fact", fact.iloc[lo:hi], persist=True, npartitions=3, distribution="sharded")
    c.create_table("dim", dim if rank == 0 else dim.iloc[:0], persist=True, distribution="root")

    def check(got, exp, keys, fcols, icols=()):
        got = got.sort_values(keys, na_position="last").reset_index(drop=True)
        exp = exp.sort_values(keys, na_position="last").reset_index(drop=True)
        assert len(got) == len(exp), (len(got), len(exp))
        for k in list(keys) + list(icols):
            a = got[k].astype("Float64").fillna(-1e18).tolist()
            b = exp[k].astype("Float64").fillna(-1e18).tolist()
            assert a == b, k
        for f in fcols:
            np.testing.assert_allclose(got[f].to_numpy(dtype=float), exp[f].to_numpy(dtype=float), rtol=1e-9)

    # 1. Q3: broadcast build side + fused scan + reduce-scatter of the dense partial tables
    before = executor.stats["star_fused"]
    q3 = """SELECT d.grp, SUM(f.val) AS rev FROM fact f JOIN dim d ON f.fk = d.pk
            WHERE f.x > 0 AND d.flag < 5 GROUP BY d.grp"""
    e = fact[fact.x > 0].merge(dim[dim.flag < 5], left_on="fk", right_on="pk")
    exp = e.groupby("grp", dropna=False).agg(rev=("val", "sum")).reset_index()
    assert len(exp) < 0.5 * 60_000, "the check needs never-hit group slots"
    for rep in range(5):      # repeated: the prepared plan alternates its two lookup buffers / peer tables
        got = c.sql(q3, return_futures=False)
        assert executor.stats["star_fused"] == before + 1 + rep
        check(got, exp, ["grp"], ["rev"])
    from dask_sql_b200 import parallel as P
    if P.peer_memory_available():
        assert executor.stats.get("peer_merge_plans", 0) >= 1, "the NVLink peer merge was not used"
    # the same through the NCCL reduce-scatter path (fresh Context: plans are prepared per Context)
    os.environ["B200SQL_PEER_MERGE"] = "0"
    c2 = Context()
    c2.create_table("fact", fact.iloc[lo:hi], persist=True, npartitions=3, distribution="sharded")
    c2.create_table("dim", dim if rank == 0 else dim.iloc[:0], persist=True, distribution="root")
    for rep in range(2):
        check(c2.sql(q3, return_futures=False), exp, ["grp"], ["rev"])
    del os.environ["B200SQL_PEER_MERGE"]
    # the dim table replicated on every rank (no broadcast: every rank builds its own lookup)
    c3 = Context()
    c3.create_table("fact", fact.iloc[lo:hi], persist=True, npartitions=3, distribution="sharded")
    c3.create_table("dim", dim, persist=True, distribution="replicated")
    for rep in range(3):
        check(c3.sql(q3, return_futures=False), exp, ["grp"], ["rev"])
    # 1b. the same with COUNT(*) (row counter instead of the -0.0 indicator) and an int SUM (bitmap)
    got = c.sql("""SELECT d.grp, COUNT(*) AS n, SUM(f.x) AS sx FROM fact f JOIN dim d ON f.fk = d.pk
                   WHERE d.flag < 5 GROUP BY d.grp""", return_futures=False)
    e = fact.merge(dim[dim.flag < 5], left_on="fk", right_on="pk")
    exp = e.groupby("grp", dropna=False).agg(n=("val", "size"), sx=("x", "sum")).reset_index()
    check(got, exp, ["grp"], [], ["n", "sx"])
    got = c.sql("""SELECT d.grp, MIN(f.x) AS lo FROM fact f JOIN dim d ON f.fk = d.pk
                   WHERE d.flag < 5 GROUP BY d.grp""", return_futures=False)
    check(got, e.groupby("grp", dropna=False).agg(lo=("x", "min")).reset_index(), ["grp"], [], ["lo"])
    # bitwise accumulators: AND / OR / XOR merged by the peer kernel, and by all-to-all + b2_bitwise_combine
    # under NCCL (which has no bitwise reduction)
    qb = """SELECT d.grp, BIT_AND(f.x) AS ba, BIT_OR(f.x) AS bo, BIT_XOR(f.x) AS bx FROM fact f JOIN dim d
            ON f.fk = d.pk WHERE d.flag < 5 GROUP BY d.grp"""
    bits = e.groupby("grp", dropna=False).x
    expb = pd.DataFrame({"grp": bits.apply(lambda s: 0).index,
                         "ba": bits.apply(lambda s: np.bitwise_and.reduce(s.to_numpy())).values,
                         "bo": bits.apply(lambda s: np.bitwise_or.reduce(s.to_numpy())).values,
                         "bx": bits.apply(lambda s: np.bitwise_xor.reduce(s.to_numpy())).values})
    for rep in range(3):
        check(c.sql(qb, return_futures=False), expb, ["grp"], [], ["ba", "bo", "bx"])
    os.environ["B200SQL_PEER_MERGE"] = "0"
    c4 = Context()
    c4.create_table("fact", fact.iloc[lo:hi], persist=True, npartitions=3, distribution="sharded")
    c4.create_table("dim", dim if rank == 0 else dim.iloc[:0], persist=True, distribution="root")
    for rep in range(2):
        check(c4.sql(qb, return_futures=False), expb, ["grp"], [], ["ba", "bo", "bx"])
    del os.environ["B200SQL_PEER_MERGE"]
    # 1c. composite group key on the build side: hashed slots differ per rank -> merged by key
    got = c.sql("""SELECT d.grp, d.flag, SUM(f.val) AS rev, COUNT(*) AS n FROM fact f JOIN dim d ON f.fk = d.pk
                   WHERE f.x > 0 GROUP BY d.grp, d.flag""", return_futures=False)
    e = fact[fact.x > 0].merge(dim, left_on="fk", right_on="pk")
    exp = e.groupby(["grp", "flag"], dropna=False).agg(rev=("val", "sum"), n=("val", "size")).reset_index()
    check(got, exp, ["grp", "flag"], ["rev"], ["n"])
    # 2. global aggregate
    got = c.sql("SELECT SUM(x) AS s, COUNT(*) AS n, AVG(val) AS a, MIN(x) AS lo, MAX(val) AS hi FROM fact WHERE x > 0",
                return_futures=False)
    e = fact[fact.x > 0]
    assert int(got.s[0]) == int(e.x.sum()) and int(got.n[0]) == len(e) and int(got.lo[0]) == int(e.x.min())
    np.testing.assert_allclose([got.a[0], got.hi[0]], [e.val.mean(), e.val.max()], rtol=1e-9)
    # 3. dense group-by over a key range with holes (6/7 of the slots empty) and a NULL-able key
    got = c.sql("SELECT gk, SUM(val) AS s, COUNT(*) AS n FROM fact GROUP BY gk", return_futures=False)
    exp = fact.groupby("gk").agg(s=("val", "sum"), n=("val", "size")).reset_index()
    check(got, exp, ["gk"], ["s"], ["n"])
    got = c.sql("SELECT fk, SUM(val) AS s, COUNT(*) AS n FROM fact WHERE x > 0 GROUP BY fk", return_futures=False)
    exp = fact[fact.x > 0].groupby("fk", dropna=False).agg(s=("val", "sum"), n=("val", "size")).reset_index()
    check(got, exp, ["fk"], ["s"], ["n"])
    # 3b. an operator on top of a sharded aggregate sees all groups
    got = c.sql("SELECT gk, SUM(val) AS s FROM fact GROUP BY gk ORDER BY s DESC LIMIT 10", return_futures=False)
    exp = fact.groupby("gk").agg(s=("val", "sum")).reset_index().sort_values("s", ascending=False).head(10)
    assert got.gk.tolist() == exp.gk.tolist()
    # 4. sparse keys: hash group-by + tree merge of partial tables
    before = executor.stats["hash_groupby"]
    got = c.sql("SELECT skey, SUM(val) AS s, AVG(val) AS a, MIN(x) AS lo FROM fact GROUP BY skey",
                return_futures=False, config_options={"sql.aggregate.split_every": 2})
    assert executor.stats["hash_groupby"] > before
    exp = fact.groupby("skey").agg(s=("val", "sum"), a=("val", "mean"), lo=("x", "min")).reset_index()
    check(got, exp, ["skey"], ["s", "a"], ["lo"])
    # 5. materialising joins with a broadcast build side: each rank returns its shard's rows
    got = c.sql("SELECT f.fk, f.val, d.grp FROM fact f JOIN dim d ON f.fk = d.pk WHERE d.flag = 3",
                return_futures=False)
    exp = fact.iloc[lo:hi].merge(dim[dim.flag == 3], left_on="fk", right_on="pk")[["fk", "val", "grp"]]
    check(got, exp, ["fk", "val", "grp"], [])
    got = c.sql("SELECT f.fk, f.val, d.grp FROM fact f LEFT JOIN dim d ON f.fk = d.pk AND d.flag = 3 WHERE f.x > 2000000000",
                return_futures=False)
    f2 = fact.iloc[lo:hi]
    f2 = f2[f2.x > 2000000000]
    exp = f2.merge(dim[dim.flag == 3], left_on="fk", right_on="pk", how="left")[["fk", "val", "grp"]]
    assert len(got) == len(exp) and int(got.grp.isna().sum()) == int(exp.grp.isna().sum())
    # 5b. FULL OUTER: unmatched build rows appear exactly once over all ranks
    got = c.sql("SELECT f.val, d.pk FROM fact f FULL JOIN dim d ON f.fk = d.pk", return_futures=False)
    referenced = set(fact.fk.dropna().astype(np.int64).tolist())
    n_unmatched_exp = int((~dim.pk.isin(referenced)).sum())
    assert n_unmatched_exp > 0
    t = torch.tensor([int(got.val.isna().sum()), int(got.val.notna().sum())], dtype=torch.int64, device="cuda")
    dist.all_reduce(t)
    assert int(t[0]) == n_unmatched_exp, (int(t[0]), n_unmatched_exp)
    assert int(t[1]) == nf, (int(t[1]), nf)         # every probe row appears once (NULL-fk rows unmatched)
    # 6. ANALYZE on the sharded table: the select's histograms are summed over the ranks, so every rank returns
    # the frame one GPU computes from the whole table
    sql = "ANALYZE TABLE fact COMPUTE STATISTICS FOR ALL COLUMNS"
    got = c.sql(sql)
    c5 = Context()
    c5.create_table("fact", fact, persist=True, npartitions=3)
    one = c5.sql(sql)
    frames = [None] * world
    dist.all_gather_object(frames, got)
    for f in frames:
        assert list(f.columns) == list(one.columns) and list(f.index) == list(one.index)
        for col in one.columns:
            for row in one.index:
                a, b = f.at[row, col], one.at[row, col]
                if row in ("mean", "std"):
                    assert (pd.isna(a) and pd.isna(b)) or abs(a - b) <= 1e-9 * max(1.0, abs(b)), (col, row, a, b)
                else:
                    assert (pd.isna(a) and pd.isna(b)) or a == b, (col, row, a, b)
    # 7. RAND and TABLESAMPLE BERNOULLI on a sharded table: rank r numbers its rows from the rows of the ranks
    # before it, so the ranks' rows together are the sample and the column one GPU computes -- on the table cut
    # by shard_bounds, and on one cut unevenly (rank r holding a share proportional to r + 1)
    sql = "SELECT skey, gk, RAND(7) AS r FROM {} TABLESAMPLE BERNOULLI (10) REPEATABLE (3) WHERE x > 0"
    weights = np.cumsum([0] + [r + 1 for r in range(world)])
    ulo, uhi = (int(nf * weights[rank] // weights[-1]), int(nf * weights[rank + 1] // weights[-1]))
    c.create_table("fact_u", fact.iloc[ulo:uhi], persist=True, npartitions=2, distribution="sharded")
    one = c5.sql(sql.format("fact")).compute()
    for name in ("fact", "fact_u"):
        got = c.sql(sql.format(name)).compute()
        parts = [None] * world
        dist.all_gather_object(parts, got)
        check(pd.concat(parts, ignore_index=True), one, ["skey", "gk", "r"], [])
    dist.barrier()
    if rank == 0:
        print(f"mgpu_check OK on {world} GPUs")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
