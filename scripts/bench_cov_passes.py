#!/usr/bin/env python
"""Time the single-GPU coverage pre-filter with its counting table split into key-range passes (sgpu_reads_cov_filter_ex).

    python scripts/bench_cov_passes.py [--reads 20000000] [--k1 56] [--threshold 2] [--passes 1,2,4,8] [--iters 3] [--big-reads N]

Reads come from bench.py's generator on the GPU (150 bp, 150x coverage, 1 % substitutions) and are adopted by the context.
1. --reads reads filtered with each forced P, alternated (P = 1, 2, 4, 8, then again), medians of --iters rounds after a warm-up
   round. Every run has a context of its own, so its peak_bytes is that run's; a filter over the first thousand reads reserves the
   arena before the timed call. The call is timed with CUDA events on the library's stream. The hll / fill / filter split comes from a
   separate torch.profiler run per P (device time of the kernels, summed by name). The SHA-256 of the verdicts must be equal for every P.
2. A read set above the single-table ceiling: --big-reads, or by default sized from the bound per read of (1) so that the single
   table (12 bytes per key of the bound) exceeds the arena of a context created next to the reads. The planned call (passes = 0) is
   timed, then the planned P + 1 forced, whose verdicts must be the same. If the device cannot hold the reads, that is reported.
One JSON line with the card's name and power limit. apply = 0 throughout (the compaction is not part of what passes change).
"""
import argparse
import hashlib
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402  (the read generator of the graded bench)

PHASES = {"hll": ("cov_hll_k",), "fill": ("cov_fill_k",), "filter": ("cov_filter_k",),
          "distinct": ("cov_distinct_k",)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000)
    ap.add_argument("--k1", type=int, default=56, help="k + 1")
    ap.add_argument("--threshold", type=int, default=2)
    ap.add_argument("--passes", default="1,2,4,8")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--big-reads", type=int, default=0, help="0: sized from the bound per read of the first measurement")
    args = ap.parse_args()
    import numpy as np
    import torch
    from spades_b200.kmer_index import Context
    from spades_b200.reads_io import CovFilteringWrap
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    med = lambda xs: float(np.median(xs))     # noqa: E731

    def run(words, offs, lens, nwr, n, passes, profile=False):
        """one filter in a fresh context -> (ms, keep, stats, times, phase ms or None)"""
        ctx = Context(0, stream=stream.cuda_stream)
        try:
            ctx.adopt_device_reads(words.data_ptr(), min(n, 1000) * nwr, offs.data_ptr(), lens.data_ptr(), min(n, 1000))
            CovFilteringWrap(ctx, args.k1, args.threshold, apply=False, passes=passes)       # reserves the arena
            ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
            stream.synchronize()
            phases = None
            if profile:
                from torch.profiler import ProfilerActivity, profile as prof
                with prof(activities=[ProfilerActivity.CUDA]) as p:
                    keep, st = CovFilteringWrap(ctx, args.k1, args.threshold, apply=False, passes=passes)
                    stream.synchronize()
                phases = {k: 0.0 for k in PHASES}
                for e in p.key_averages():
                    for k, names in PHASES.items():
                        # demangled "...::cov_fill_k<...::WholeTable>(unsigned long const*, ..." or mangled "...10cov_fill_kINS0_10WholeTableEEEvPKm...",
                        # and the same without template arguments ("cov_fill_k(", "10cov_fill_kE")
                        if any(re.search(r"\b%s[(<]|\d%s[EI]" % (nm, nm), e.key) for nm in names):
                            phases[k] += e.device_time_total / 1000.0
                return None, keep, st, ctx.times(), phases
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            keep, st = CovFilteringWrap(ctx, args.k1, args.threshold, apply=False, passes=passes)
            e1.record(stream)
            stream.synchronize()
            return e0.elapsed_time(e1), keep, st, ctx.times(), None
        finally:
            ctx.close()

    sha = lambda keep: hashlib.sha256(keep.tobytes()).hexdigest()     # noqa: E731
    out = {"gpu": B.gpu_facts(0), "k_plus_one": args.k1, "threshold": args.threshold}

    # 1. forced P at --reads
    n = args.reads
    words, offs, lens, nwr = B.gen_reads_device(torch, n, max(B.READ_LEN + 1, n), 42, dev)
    torch.cuda.synchronize()
    plist = [int(x) for x in args.passes.split(",")]
    ms, rows = {p: [] for p in plist}, {}
    for it in range(args.iters + 1):                      # round 0 warms up
        for p in plist:
            t, keep, st, tm, _ = run(words, offs, lens, nwr, n, p)
            assert tm["cov_filter_passes"] == p
            if it:
                ms[p].append(t)
            rows[p] = {"sha256_keep": sha(keep), "stats": st, "table_bytes": tm["cov_filter_table_bytes"], "peak_bytes": tm["peak_bytes"]}
    for p in plist:
        _, keep, _, _, phases = run(words, offs, lens, nwr, n, p, profile=True)
        assert sha(keep) == rows[p]["sha256_keep"]
        rows[p].update({"total_ms": med(ms[p]), "runs_ms": ms[p], "kernel_ms": phases})
    out["forced"] = {"reads": n, "iters": args.iters, "by_passes": {str(p): rows[p] for p in plist},
                     "same_verdicts_and_stats": len({(r["sha256_keep"], json.dumps(r["stats"], sort_keys=True)) for r in rows.values()}) == 1}
    bound_per_read = rows[plist[0]]["stats"]["cardinality_upper_bound"] / n
    del words, offs, lens
    torch.cuda.empty_cache()

    # 2. above the single-table ceiling, planned
    free, total = torch.cuda.mem_get_info(0)
    reads_bytes_per_read = nwr * 8 + 8 + 4
    nb = args.big_reads or int(1.15 * 0.92 * free / (12 * bound_per_read + 0.92 * reads_bytes_per_read)) // 1_000_000 * 1_000_000
    big = {"reads": nb, "device_free_bytes_before_reads": free, "device_total_bytes": total}
    try:
        words, offs, lens, nwr = B.gen_reads_device(torch, nb, max(B.READ_LEN + 1, nb), 43, dev)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    except torch.cuda.OutOfMemoryError as e:
        big["result"] = "the device cannot hold %d reads: %s" % (nb, str(e).splitlines()[0])
        out["planned"] = big
        print(json.dumps(out))
        return
    big["reads_bytes"] = nb * reads_bytes_per_read
    big["device_free_bytes_next_to_reads"] = torch.cuda.mem_get_info(0)[0]
    try:
        t, keep, st, tm, _ = run(words, offs, lens, nwr, nb, 0)
    except Exception as e:                                # e.g. SGPU_ENOMEM: reported, as the result of this measurement
        big["result"] = str(e)
        out["planned"] = big
        print(json.dumps(out))
        return
    P = tm["cov_filter_passes"]
    big.update({"stats": st, "planned_passes": P, "total_ms": t, "table_bytes": tm["cov_filter_table_bytes"],
                "single_table_bytes": 8 * max(1024, st["cardinality_upper_bound"] * 3 // 2), "library_peak_bytes": tm["peak_bytes"],
                "peak_hbm_bytes": tm["peak_bytes"] + nb * reads_bytes_per_read, "sha256_keep": sha(keep)})
    big["arena_bytes_about"] = int(0.92 * big["device_free_bytes_next_to_reads"])
    big["single_table_exceeds_arena"] = big["single_table_bytes"] > big["arena_bytes_about"]
    t2, keep2, st2, tm2, _ = run(words, offs, lens, nwr, nb, P + 1)
    big.update({"check_passes": tm2["cov_filter_passes"], "check_total_ms": t2, "check_same_verdicts_and_stats": sha(keep2) == big["sha256_keep"] and st2 == st})
    out["planned"] = big
    print(json.dumps(out))


if __name__ == "__main__":
    main()
