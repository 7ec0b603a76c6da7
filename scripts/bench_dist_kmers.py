#!/usr/bin/env python
"""Time the distributed (k+1)-mer count and the distributed k-mers of its (k+1)-mers, phase by phase on every rank.

    python -m torch.distributed.run --nproc-per-node=N scripts/bench_dist_kmers.py [--reads 20000000] [--k 55] [--buckets 0]
    python scripts/bench_dist_kmers.py ...          (one rank, no launcher)

Every rank generates its own reads on its GPU with bench.py's generator (150 bp, 1 % substitutions, seed 42 + rank, a genome as
long as the read count) and adopts them. Before anything is timed, a small shard set (--check-reads per rank, seed 1000 + rank)
goes through both distributed steps, and rank 0 compares the ranks' k-mer shards (device checksums added / xor-ed, bucket sizes
summed) with the single-GPU k-mers of the (k+1)-mers of the union of those shards; a mismatch stops the script.
Timed: DistributedKMerCounter(k + 1).Count, then DistributedKmersFromKpomers.Count of its shard, each with a host clock around
work that ends in a device synchronise, and the phases the library records with CUDA events: histogram (level-A count), scatter,
exchange, sort (refinement + local sort + compaction). At world size 1 the single-GPU sgpu_kmers_from_kpomers_ex over the same
(k+1)-mer set runs in the same iteration, alternately before and after the distributed one, and its checksum must equal the
distributed one's. Rank 0 prints one JSON line with the card's name and power limit; peak_bytes is the context's device high-water
mark over the whole run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as BN  # noqa: E402  (the read generator of the graded bench)


def phases(t):
    return {"histogram": t["extract_count_ms"], "scatter": t["extract_scatter_ms"], "exchange": t["exchange_ms"],
            "sort": t["refine_ms"] + t["local_sort_ms"] + t["compact_ms"], "passes": t["passes"]}


def reduce_checks(torch, dist, st, dev, world):
    """(summed bucket sizes, checksum of the union) of the ranks' disjoint bucket-owned sets; dev: where the collectives run"""
    c = st.checksum()
    bsz = torch.from_numpy(st.bucket_sizes().copy()).to(dev)
    dist.all_reduce(bsz)
    t = torch.tensor([c[0], c[1] - (1 << 64) if c[1] >= (1 << 63) else c[1], c[3]], dtype=torch.int64, device=dev)   # sums wrap mod 2^64
    dist.all_reduce(t)
    xs = [None] * world
    dist.all_gather_object(xs, c[2])
    x = 0
    for v in xs:
        x ^= v
    m64 = (1 << 64) - 1
    return bsz.cpu().numpy(), [int(t[0].item()), int(t[1].item()) & m64, x, int(t[2].item()) & m64]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000, help="reads per rank")
    ap.add_argument("--k", type=int, default=55)
    ap.add_argument("--buckets", type=int, default=0, help="0 = 10 x host threads, as bench.py")
    ap.add_argument("--check-reads", type=int, default=200_000, help="reads per rank of the check against the single-GPU path")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.distributed as dist
    from spades_b200.distributed import DistributedKMerCounter, DistributedKmersFromKpomers
    from spades_b200.kmer_index import Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter
    os.environ.setdefault("RANK", "0"); os.environ.setdefault("WORLD_SIZE", "1"); os.environ.setdefault("LOCAL_RANK", "0")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29534")
    rank, world, lrank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lrank)
    dev = torch.device("cuda", lrank)
    dist.init_process_group("nccl" if world > 1 else "gloo", device_id=dev if world > 1 else None)
    k, B = args.k, args.buckets or 10 * BN.host_threads()
    stream = torch.cuda.current_stream()
    ctx = Context(lrank, stream=stream.cuda_stream)

    # ---- check: the distributed k-mers of a small shard set against one GPU over their union
    n_c = args.check_reads
    glen = max(BN.READ_LEN + 1, n_c)
    w, o, ln, nwr = BN.gen_reads_device(torch, n_c, glen, 1000 + rank, dev)
    ctx.adopt_device_reads(w.data_ptr(), n_c * nwr, o.data_ptr(), ln.data_ptr(), n_c)
    kp = DistributedKMerCounter(ctx, k + 1).Count(B)
    km = DistributedKmersFromKpomers(ctx, kp).Count(B)
    got_bsz, got = reduce_checks(torch, dist, km, dev if world > 1 else "cpu", world)
    km.free(); kp.free()
    ok, check = True, None
    if rank == 0:
        parts = [BN.gen_reads_device(torch, n_c, glen, 1000 + r, dev) for r in range(world)]
        uw = torch.cat([p[0][: n_c * nwr] for p in parts] + [torch.zeros(8, dtype=torch.int64, device=dev)])
        uo = torch.cat([p[1] + r * n_c * nwr for r, p in enumerate(parts)])
        ul = torch.cat([p[2] for p in parts])
        ctx.adopt_device_reads(uw.data_ptr(), world * n_c * nwr, uo.data_ptr(), ul.data_ptr(), world * n_c)
        kp1 = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1)).Count(B)
        km1 = KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kp1)).Count(B)
        want, want_bsz = km1.checksum(), km1.bucket_sizes()
        km1.free(); kp1.free()
        torch.cuda.synchronize()
        ok = got == want and np.array_equal(got_bsz, want_bsz)
        check = {"reads_per_rank": n_c, "distinct_kmers": want[0], "checksums_distributed": got, "checksums_single_gpu": want, "ok": ok}
        del parts, uw, uo, ul
    flag = [ok]
    dist.broadcast_object_list(flag, src=0)
    del w, o, ln
    if not flag[0]:
        raise SystemExit("bench_dist_kmers: distributed k-mers != single-GPU k-mers of the union: %s" % (check,))

    # ---- timed
    n = args.reads
    words, offs, lens, nwr = BN.gen_reads_device(torch, n, max(BN.READ_LEN + 1, n), 42 + rank, dev)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    def clock(f):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    runs = []
    for it in range(args.warmup + args.iters):
        ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
        kp, t_kp = clock(lambda: DistributedKMerCounter(ctx, k + 1).Count(B))
        ph_kp = phases(ctx.times())
        row = {"kpomers_ms": t_kp, "kpomers_phases_ms": ph_kp, "kpomers_rank": kp.total_kmers()}

        def dist_kmers():
            km, t = clock(lambda: DistributedKmersFromKpomers(ctx, kp).Count(B))
            row.update(kmers_ms=t, kmers_phases_ms=phases(ctx.times()), kmers_rank=km.total_kmers())
            c = km.checksum()
            km.free()
            return c

        def single_kmers():
            km, t = clock(lambda: KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kp)).Count(B))
            row.update(single_gpu_kmers_ms=t, single_gpu_phases_ms=phases(ctx.times()))
            c = km.checksum()
            km.free()
            return c

        if world == 1 and it % 2:
            c1 = single_kmers(); cd = dist_kmers()
        else:
            cd = dist_kmers()
            c1 = single_kmers() if world == 1 else None
        if world == 1:
            row["same_as_single_gpu"] = cd == c1
        kp.free()
        if it >= args.warmup:
            runs.append(row)
    med = lambda xs: float(np.median(xs))     # noqa: E731
    out = {"rank": rank, "world": world, "reads": n, "k": k, "buckets": B, "iters": args.iters,
           "kpomers_ms": med([r["kpomers_ms"] for r in runs]), "kmers_ms": med([r["kmers_ms"] for r in runs]),
           "kpomers_phases_ms": {p: med([r["kpomers_phases_ms"][p] for r in runs]) for p in runs[0]["kpomers_phases_ms"]},
           "kmers_phases_ms": {p: med([r["kmers_phases_ms"][p] for r in runs]) for p in runs[0]["kmers_phases_ms"]},
           "kpomers_rank": runs[-1]["kpomers_rank"], "kmers_rank": runs[-1]["kmers_rank"], "peak_bytes": ctx.times()["peak_bytes"]}
    if world == 1:
        out["single_gpu_kmers_ms"] = med([r["single_gpu_kmers_ms"] for r in runs])
        out["single_gpu_phases_ms"] = {p: med([r["single_gpu_phases_ms"][p] for r in runs]) for p in runs[0]["single_gpu_phases_ms"]}
        out["same_as_single_gpu"] = all(r["same_as_single_gpu"] for r in runs)
    out["runs"] = runs
    outs = [None] * world
    dist.all_gather_object(outs, out)
    if rank == 0:
        print(json.dumps({"gpu": BN.gpu_facts(lrank), "check": check, "ranks": outs}))
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
