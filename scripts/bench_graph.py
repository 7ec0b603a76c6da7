#!/usr/bin/env python
"""Whole-path measurement, BASELINE config 3 shape: synthetic 150 bp reads -> (k+1)-mers -> k-mers -> both KMerIndexes -> masks ->
coverage -> unitigs (+ perfect loops) -> link records -> GFA file, k = 55, on ONE GPU -- what spades-gbuilder does
(projects/spades_tools/gbuilder.cpp:157-225). Not the bench line (bench.py prints that); this prints the per-phase
milliseconds and the peak HBM of the whole path.

    python scripts/bench_graph.py --reads 20000000 [--edge-index] [--host-result]

--host-result: both counts keep their sets in pinned host memory and the graph comes from sgpu_graph_build_streamed, which reads
the sets chunk by chunk; the line then also reports the bytes uploaded and the junction batches.

The graph phase keeps everything resident: per 100 M reads the (k+1)-mer set with multiplicities (79 GB), the k-mer set (62 GB),
two indexes (5.6 GB), masks, coverage (16 GB) and the partition buffers of the second count, together more than 180 GB. The
default of 20 M reads is sized for the 80 GB of an H100.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402  (the read generator and constants of the graded bench)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000)
    ap.add_argument("--buckets", type=int, default=0)
    ap.add_argument("--edge-index", action="store_true", help="also time the EdgeIndex refill (SURVEY 8f-1)")
    ap.add_argument("--early-tc", type=int, default=0)
    ap.add_argument("--cov-threshold", type=int, default=0, help="run the coverage pre-filter (SURVEY 8f-3) with this threshold first")
    ap.add_argument("--host-result", action="store_true", help="both k-mer sets in host memory, the graph from the streamed build")
    args = ap.parse_args()
    import torch
    from spades_b200.graph import DeBruijnGraph, EdgeIndex
    from spades_b200.kmer_index import (Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder)
    from spades_b200._lib import SgpuGraphOptions
    import ctypes as C
    import hashlib
    host = args.host_result
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    k = B.K_GRAPH
    nb = args.buckets or 10 * B.host_threads()
    n = args.reads
    words, offs, lens, nwr = B.gen_reads_device(torch, n, max(B.READ_LEN + 1, n), 42, dev)
    torch.cuda.synchronize(); torch.cuda.empty_cache()
    stream = torch.cuda.current_stream()
    ctx = Context(0, stream=stream.cuda_stream)
    ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
    phases = {}

    def timed(name, fn):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize(); phases[name] = round((time.perf_counter() - t0) * 1e3, 1)
        return r

    cov_stats = None
    if args.cov_threshold:
        from spades_b200.reads_io import CovFilteringWrap
        _, cov_stats = timed("coverage_prefilter_ms", lambda: CovFilteringWrap(ctx, k + 1, args.cov_threshold, apply=True))
    kpomers = timed("count_kpomers_ms", lambda: KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1), result_on_host=host).Count(nb))
    t_kp = ctx.times()
    kmers = timed("kmers_from_kpomers_ms", lambda: KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kpomers), result_on_host=host).Count(nb))
    t_km = ctx.times()
    kmer_index = timed("kmer_index_ms", lambda: KMerIndexBuilder(ctx).BuildIndex(kmers))
    kpomer_index = timed("kpomer_index_ms", lambda: KMerIndexBuilder(ctx).BuildIndex(kpomers))
    stage_bytes = {"kmers_from_kpomers": t_km.get("stage_h2d_bytes", 0)}

    def build():
        h = C.c_void_p()
        opts = SgpuGraphOptions(1, int(args.early_tc), 0, 0.8, 10, 200)
        build_fn = ctx.L.sgpu_graph_build_streamed if host else ctx.L.sgpu_graph_build_opts
        ctx.check(build_fn(ctx.h, kpomers.h, kmers.h, kmer_index.h, kpomer_index.h, C.byref(opts), C.byref(h)))
        return DeBruijnGraph(ctx, h, kpomers, kmers, kmer_index, kpomer_index)
    g = timed("masks_coverage_unitigs_links_ms", build)
    t_g = ctx.times()
    stage_bytes["graph"] = t_g.get("stage_h2d_bytes", 0)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "graph.gfa")
        timed("gfa_text_and_file_ms", lambda: g.write_gfa(path))
        gfa_bytes = os.path.getsize(path)
        hs = hashlib.sha256()
        with open(path, "rb") as f:
            for blk in iter(lambda: f.read(1 << 24), b""):
                hs.update(blk)
    ei_n = None
    if args.edge_index:
        ei = timed("edge_index_refill_ms", lambda: EdgeIndex(g, None, nb))
        ei_n = ei.size()
        ei.free()
    t = ctx.times()
    total = sum(phases.values())
    windows = n * (B.READ_LEN - (k + 1) + 1)
    line = {"what": "reads -> GFA on one GPU (BASELINE config 3 shape at %.0f %% of its size)" % (100.0 * n / 100_000_000),
            "reads": n, "k": k, "buckets": nb, "phases_ms": phases, "total_ms": round(total, 1),
            "Mk-mers/s_whole_path": round(windows / (total / 1e3) / 1e6, 1),
            "distinct_kpomers": kpomers.total_kmers(), "distinct_kmers": kmers.total_kmers(),
            "unitigs": int(ctx.L.sgpu_graph_num_unitigs(g.h)), "unitig_bases": int(ctx.L.sgpu_graph_unitig_bases(g.h)), "gfa_bytes": gfa_bytes,
            "edge_index_kmers": ei_n, "coverage_prefilter": cov_stats,
            "count_kpomers_detail": {q: t_kp[q] for q in ("extract_count_ms", "extract_scatter_ms", "refine_ms", "local_sort_ms", "compact_ms", "passes")},
            "kmers_from_kpomers_detail": {q: t_km[q] for q in ("extract_count_ms", "extract_scatter_ms", "refine_ms", "local_sort_ms", "compact_ms", "passes")},
            "peak_hbm_gb": round(t["peak_bytes"] / 1e9, 2), "host_result": host, "stage_h2d_bytes": stage_bytes,
            "graph_junction_batches": t_g.get("graph_junction_batches"), "gfa_sha256": hs.hexdigest(),
            "device": torch.cuda.get_device_name(0)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
