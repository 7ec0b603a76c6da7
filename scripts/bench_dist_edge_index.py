#!/usr/bin/env python
"""Time the distributed EdgeIndex refill (DistributedEdgeIndex) next to the single-GPU EdgeIndex over the same graph, at world size
1 on one GPU: every peer mapping is then this rank's own memory, so this measures what the distributed protocol costs (the
count's passes, the level merges, the CAS puts), not NVLink.

    python scripts/bench_dist_edge_index.py [--reads 20000000] [--k 55] [--buckets 80] [--warmup 1] [--iters 3]

The reads come from bench.py's generator (150 bp, 1 % substitutions, seed 42, a genome as long as the read count). They go through
the distributed (k+1)-mer count, the distributed k-mers, both indexes, the distributed extension index and ConstructGraph; the
single-GPU graph build runs over the same sets and indexes. Every iteration
then builds, alternately first and second, the (k+1)-mer DistributedEdgeIndex (num_buckets = --buckets) and the single-GPU
EdgeIndex. The warm-up iteration checks that both serialize to the same SHA-256 and give the same values. One JSON line: medians
over the timed iterations (the distributed build's phases: pack, count, keys, levels with their merges, ranks, fill, values), the
card's name and power limit, and the context's device high-water mark over the whole run.
"""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as BN  # noqa: E402  (the read generator of the graded bench)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000)
    ap.add_argument("--k", type=int, default=55)
    ap.add_argument("--buckets", type=int, default=80)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import torch.distributed as dist
    from spades_b200.distributed import (DistributedEdgeIndex, DistributedExtensionIndexBuilder, DistributedGraphConstructor,
                                         DistributedKMerCounter, DistributedKmersFromKpomers, assemble_edge_index_values)
    import ctypes as C
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.graph import DeBruijnGraph, EdgeIndex
    from spades_b200.kmer_index import Context, KMerIndexBuilder
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29541")
    dist.init_process_group("gloo", rank=0, world_size=1)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    k, B, n = args.k, args.buckets, args.reads
    ctx = Context(0, stream=torch.cuda.current_stream().cuda_stream)
    words, offs, lens, nwr = BN.gen_reads_device(torch, n, max(BN.READ_LEN + 1, n), 42, dev)
    ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
    kp = DistributedKMerCounter(ctx, k + 1).Count(B)
    km = DistributedKmersFromKpomers(ctx, kp).Count(B)
    mkp = KMerIndexBuilder(ctx).BuildIndex(kp)
    mk = KMerIndexBuilder(ctx).BuildIndex(km)
    ext = DistributedExtensionIndexBuilder(ctx, kp, mkp, km, mk).Build()
    dg = DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph()
    # the same graph on one GPU, from the same sets (at world size 1 a rank's sets are the union's); the refills read only the
    # graphs' edges, so the sets and indexes are freed before them
    opts = SgpuGraphOptions(1, 0, 0, 0.8, 10, 200)
    h = C.c_void_p()
    ctx.check(ctx.L.sgpu_graph_build_opts(ctx.h, kp.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h)))
    g = DeBruijnGraph(ctx, h, None, None, None, None)
    ext.free(); mk.free(); mkp.free(); km.free(); kp.free()
    del words, offs, lens
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    def clock(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    def distributed(row, check):
        dei, t = clock(lambda: DistributedEdgeIndex(dg, None, B))
        vals, tv = clock(lambda: assemble_edge_index_values(dei))
        row.update(dist_ms=t, dist_phases_ms=dei.times(), dist_download_ms=tv, levels=dei.levels)
        if check:
            row["_dist"] = (hashlib.sha256(dei.serialize()).hexdigest(), vals)
        dei.free()

    def single(row, check):
        ei, t = clock(lambda: EdgeIndex(g, None, B))
        vals, tv = clock(ei.values)
        row.update(single_gpu_ms=t, single_gpu_download_ms=tv)
        if check:
            row["_single"] = (hashlib.sha256(ei.serialize()).hexdigest(), vals)
        ei.free()

    runs, same_index, same_values, sha = [], None, None, None
    for it in range(args.warmup + args.iters):
        row = {}
        check = it == 0
        if it % 2:
            single(row, check); distributed(row, check)
        else:
            distributed(row, check); single(row, check)
        if check:
            (sha, dv), (sha_s, sv) = row.pop("_dist"), row.pop("_single")
            same_index = sha == sha_s
            same_values = bool(np.array_equal(dv[0], sv[0]) and np.array_equal(dv[1], sv[1]))
        if it >= args.warmup:
            runs.append(row)
    med = lambda xs: float(np.median(xs))     # noqa: E731
    phases = runs[0]["dist_phases_ms"].keys()
    out = {"reads": n, "k": k, "buckets": B, "iters": args.iters, "edges": g.ctx.L.sgpu_graph_num_unitigs(g.h), "slots": None,
           "dist_ms": med([r["dist_ms"] for r in runs]), "dist_phases_ms": {p: med([r["dist_phases_ms"][p] for r in runs]) for p in phases},
           "dist_download_ms": med([r["dist_download_ms"] for r in runs]), "levels": runs[0]["levels"],
           "single_gpu_ms": med([r["single_gpu_ms"] for r in runs]), "single_gpu_download_ms": med([r["single_gpu_download_ms"] for r in runs]),
           "index_sha256": sha, "same_index_as_single_gpu": same_index, "same_values_as_single_gpu": same_values,
           "peak_bytes": ctx.times()["peak_bytes"], "runs": runs}
    ei = EdgeIndex(g, None, B)
    out["slots"] = ei.size()
    ei.free()
    print(json.dumps({"gpu": BN.gpu_facts(0), "result": out}))
    g.free(); dg.free()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
