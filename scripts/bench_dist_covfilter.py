#!/usr/bin/env python
"""Time the distributed coverage pre-filter (spades_b200.distributed.distributed_cov_filter) phase by phase on every rank.

    python -m torch.distributed.run --nproc-per-node=N scripts/bench_dist_covfilter.py [--reads 20000000] [--k1 56] [--threshold 2]
    python scripts/bench_dist_covfilter.py ...          (one rank, no launcher)

Every rank generates the same synthetic union on its GPU (bench.py's generator: 150 bp, 150x coverage, 1 % substitutions) and
adopts its block of it. Phases are timed with CUDA events on the stream the library runs on: hll (begin), merge (register merge,
bound, slice allocation; descriptor exchange included), fill, filter (verdicts and, with apply, the compaction). The filter runs
alternately with apply = 0 and apply = 1, so the compaction is the difference of the two. At world size 1 the single-GPU
sgpu_reads_cov_filter (apply = 1) runs on the same reads in the same process, alternated with the distributed one. Rank 0 prints
one JSON line with the card's name and power limit; the verdicts of the two paths are compared at world size 1.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402  (the read generator of the graded bench)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000)
    ap.add_argument("--k1", type=int, default=56, help="k + 1")
    ap.add_argument("--threshold", type=int, default=2)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.distributed as dist
    from spades_b200.distributed import distributed_cov_filter
    from spades_b200.kmer_index import Context
    from spades_b200.reads_io import CovFilteringWrap
    os.environ.setdefault("RANK", "0"); os.environ.setdefault("WORLD_SIZE", "1"); os.environ.setdefault("LOCAL_RANK", "0")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29533")
    rank, world, lrank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lrank)
    dist.init_process_group("gloo")
    dev = torch.device("cuda", lrank)
    n = args.reads
    words, offs, lens, nwr = B.gen_reads_device(torch, n, max(B.READ_LEN + 1, n), 42, dev)
    lo, hi = n * rank // world, n * (rank + 1) // world
    stream = torch.cuda.Stream(device=dev)
    ctx = Context(lrank, stream=stream.cuda_stream)
    torch.cuda.synchronize()

    def adopt():
        ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs[lo:].data_ptr(), lens[lo:].data_ptr(), hi - lo)

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record(stream)
        return e

    res = {"dist": [], "single": []}
    keeps = {}
    for it in range(args.iters + 1):                  # the first round warms up
        for apply in (0, 1):
            adopt()
            marks = [("start", ev())]
            keep, st = distributed_cov_filter(ctx, args.k1, args.threshold, apply=bool(apply),
                                              phase_done=lambda name: marks.append((name, ev())))
            stream.synchronize()
            t = {name: marks[i - 1][1].elapsed_time(e) for i, (name, e) in enumerate(marks) if i}
            t["total"] = marks[0][1].elapsed_time(marks[-1][1])
            t["apply"] = apply
            if it:
                res["dist"].append(t)
            keeps["dist"], stats = keep, st
        if world == 1:
            adopt()
            e0 = ev()
            keep, sst = CovFilteringWrap(ctx, args.k1, args.threshold, apply=True)
            e1 = ev()
            stream.synchronize()
            if it:
                res["single"].append(e0.elapsed_time(e1))
            keeps["single"], single_stats = keep, sst
    med = lambda xs: float(np.median(xs)) if xs else None     # noqa: E731
    out = {"rank": rank, "world": world, "reads": n, "k_plus_one": args.k1, "threshold": args.threshold, "iters": args.iters,
           "bound": stats["cardinality_upper_bound"], "key_bits": stats["key_bits"], "distinct_keys": stats["distinct_keys"],
           "kept_rank": stats["kept"]}
    for apply in (0, 1):
        rows = [t for t in res["dist"] if t["apply"] == apply]
        out["dist_apply%d_ms" % apply] = {p: med([t[p] for t in rows]) for p in ("hll", "merge", "fill", "filter", "total")}
    out["dist_compact_ms_difference"] = out["dist_apply1_ms"]["filter"] - out["dist_apply0_ms"]["filter"]
    if world == 1:
        out["single_gpu_apply1_ms"] = med(res["single"])
        out["single_gpu_runs_ms"] = res["single"]
        out["same_verdicts_as_single_gpu"] = bool(np.array_equal(keeps["dist"], keeps["single"])) and \
            [single_stats[k] for k in ("cardinality_upper_bound", "key_bits", "distinct_keys", "kept")] == \
            [stats[k] for k in ("cardinality_upper_bound", "key_bits", "distinct_keys", "kept")]
    out["dist_runs_ms"] = res["dist"]
    outs = [None] * world
    dist.all_gather_object(outs, out)
    if rank == 0:
        print(json.dumps({"gpu": B.gpu_facts(lrank), "ranks": outs}))
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
