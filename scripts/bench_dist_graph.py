#!/usr/bin/env python
"""Time the distributed unitigs and perfect loops (DistributedGraphConstructor.ConstructGraph) next to the single-GPU graph
build's unitig and loop phases, at world size 1 on one GPU: every "remote" lookup is then local, so this measures what the
DistView costs over the LocalView, not NVLink.

    python scripts/bench_dist_graph.py [--reads 20000000] [--k 55] [--buckets 80] [--warmup 1] [--iters 3] [--early-tc 95] [--early-at]

The reads come from bench.py's generator (150 bp, 1 % substitutions, seed 42, a genome as long as the read count). They go
through the distributed (k+1)-mer count, the distributed k-mers of the (k+1)-mers, both indexes and the distributed extension
index. Every iteration then runs, alternately first and second, ConstructGraph (its phases as the library records them) and the
single-GPU graph build over the same sets and indexes with SGPU_TRACE on, whose junction, unitig and loop marks are summed. The
warm-up iteration checks that both give a GFA with the same SHA-256. One JSON line: medians over the timed iterations, the card's
name and power limit, and the context's device high-water mark over the whole run.

--early-tc L / --early-at run the early tip clipper with length bound L / the A/T clipper (default parameters) in both builds. The
line then also holds the distributed clipper phases (their sum as clipper_ms) next to the single-GPU build's "early clippers" mark
over the same sets, and both builds' GFA SHA-256s.
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as BN  # noqa: E402  (the read generator of the graded bench)


def traced(f):
    """f() with the library's SGPU_TRACE lines on stderr captured: (result, {mark: ms})"""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as tmp:
        os.dup2(tmp.fileno(), 2)
        try:
            r = f()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read()
    marks = {}
    for m in re.finditer(r"\[sgpu graph\] (.+?)\s+([0-9.]+) ms", text):
        marks[m.group(1).strip()] = marks.get(m.group(1).strip(), 0.0) + float(m.group(2))
    return r, marks


SINGLE_MARKS = ("junction list", "unitig probe + offsets", "unitig write", "download + edge table")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000)
    ap.add_argument("--k", type=int, default=55)
    ap.add_argument("--buckets", type=int, default=80)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--early-tc", type=int, default=0)
    ap.add_argument("--early-at", action="store_true")
    args = ap.parse_args()
    clip = bool(args.early_tc or args.early_at)
    CLIP_PHASES = ("at_edges_probe", "at_edges_apply", "at_tips_probe", "tip_probe", "isolate", "unlink")
    os.environ["SGPU_TRACE"] = "1"              # read once by the library, at its first trace mark
    import ctypes as C
    import hashlib
    import numpy as np
    import torch
    import torch.distributed as dist
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.distributed import (DistributedExtensionIndexBuilder, DistributedGraphConstructor, DistributedKMerCounter,
                                         DistributedKmersFromKpomers, assemble_graph)
    from spades_b200.graph import DeBruijnGraph
    from spades_b200.kmer_index import Context, KMerIndexBuilder
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29537")
    dist.init_process_group("gloo", rank=0, world_size=1)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    k, B, n = args.k, args.buckets, args.reads
    ctx = Context(0, stream=torch.cuda.current_stream().cuda_stream)
    words, offs, lens, nwr = BN.gen_reads_device(torch, n, max(BN.READ_LEN + 1, n), 42, dev)
    ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
    kp = DistributedKMerCounter(ctx, k + 1).Count(B)
    km = DistributedKmersFromKpomers(ctx, kp).Count(B)
    del words, offs, lens
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    mkp = KMerIndexBuilder(ctx).BuildIndex(kp)
    mk = KMerIndexBuilder(ctx).BuildIndex(km)
    ext = DistributedExtensionIndexBuilder(ctx, kp, mkp, km, mk).Build()

    def clock(f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t0) * 1e3

    def distributed(row, check):
        dg, t = clock(lambda: DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph(early_tip_clipper_length=args.early_tc,
                                                                                         early_at_clipper=args.early_at))
        row.update(construct_ms=t, construct_phases_ms=dg.times())
        if clip:
            row["clipper_phases_ms"] = dg.clipper_times()
            row["clipper_ms"] = sum(row["clipper_phases_ms"].values())
        if check:
            ag = assemble_graph(dg)
            row["_dist"] = hashlib.sha256(ag.gfa().encode()).hexdigest()
            ag.free()
        dg.free()

    def single(row, check):
        opts = SgpuGraphOptions(1, args.early_tc, 1 if args.early_at else 0, 0.8, 10, 200)
        h = C.c_void_p()
        _, marks = traced(lambda: ctx.check(ctx.L.sgpu_graph_build_opts(ctx.h, kp.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h))))
        g = DeBruijnGraph(ctx, h, kp, km, mk, mkp)
        # the unitig and loop phases: everything after the early clippers' mark, up to the end of the build
        row.update(single_gpu_unitigs_ms=sum(marks.get(m, 0.0) for m in SINGLE_MARKS), single_gpu_marks_ms=marks)
        if clip:
            row["single_gpu_clipper_ms"] = marks.get("early clippers", 0.0)
        if check:
            row["_single"] = hashlib.sha256(g.gfa().encode()).hexdigest()
        g.free()

    runs, same, sha, sha_single = [], None, None, None
    for it in range(args.warmup + args.iters):
        row = {}
        check = it == 0
        if it % 2:
            single(row, check); distributed(row, check)
        else:
            distributed(row, check); single(row, check)
        if check:
            sha, sha_single = row.pop("_dist"), row.pop("_single")
            same = sha == sha_single
        if it >= args.warmup:
            runs.append(row)
    med = lambda xs: float(np.median(xs))     # noqa: E731
    out = {"reads": n, "k": k, "buckets": B, "iters": args.iters, "kpomers": kp.total_kmers(), "kmers": km.total_kmers(),
           "construct_ms": med([r["construct_ms"] for r in runs]),
           "construct_phases_ms": {p: med([r["construct_phases_ms"][p] for r in runs]) for p in runs[0]["construct_phases_ms"]},
           "single_gpu_unitigs_ms": med([r["single_gpu_unitigs_ms"] for r in runs]),
           "gfa_sha256": sha, "same_gfa_as_single_gpu": same, "peak_bytes": ctx.times()["peak_bytes"], "runs": runs}
    if clip:
        out.update(early_tc=args.early_tc, early_at=args.early_at, clipper_ms=med([r["clipper_ms"] for r in runs]),
                   clipper_phases_ms={p: med([r["clipper_phases_ms"][p] for r in runs]) for p in CLIP_PHASES},
                   single_gpu_clipper_ms=med([r["single_gpu_clipper_ms"] for r in runs]), gfa_sha256_single_gpu=sha_single)
    print(json.dumps({"gpu": BN.gpu_facts(0), "result": out}))
    ext.free(); mk.free(); mkp.free(); km.free(); kp.free()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
