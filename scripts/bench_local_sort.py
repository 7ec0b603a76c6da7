#!/usr/bin/env python
"""Local-sort timing at the bench's shape: the bench's synthetic reads (same seeded generator, imported from bench.py), counted
as the bench's step counts them, at 10 M reads (one pass) and 40 M reads (four passes). Prints one JSON line per size with
local_sort_ms (median over the timed counts) and the local sort's path counters, so that a before/after table of the kernel
comes from one command:

    python scripts/bench_local_sort.py [--reads 10000000,40000000] [--repeats 3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the generator and the bucket rule of the flagship benchmark)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", default="10000000,40000000", help="comma-separated read counts")
    ap.add_argument("--repeats", type=int, default=3, help="timed counts per size (one untimed count first)")
    ap.add_argument("--buckets", type=int, default=0, help="0 = the bench's rule, 10 x host threads")
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_local_sort.py: no CUDA device; this path has no CPU fallback")
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter
    dev = torch.device("cuda", 0)
    B = args.buckets or 10 * bench.host_threads()
    stream = torch.cuda.current_stream()
    ctx = Context(0, stream=stream.cuda_stream)
    for n_reads in (int(x) for x in args.reads.split(",")):
        words, offs, lens, nwr = bench.gen_reads_device(torch, n_reads, max(bench.READ_LEN + 1, n_reads), 42, dev)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        sort_ms, runs = [], []
        for rep in range(args.repeats + 1):
            ctx.adopt_device_reads(words.data_ptr(), n_reads * nwr, offs.data_ptr(), lens.data_ptr(), n_reads)
            st = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(bench.K)).Count(B)
            t = ctx.times()
            distinct = st.total_kmers()
            st.free()
            if rep:
                sort_ms.append(t["local_sort_ms"])
                runs.append({k: t[k] for k in ("refine_ms", "local_sort_ms", "compact_ms")})
        print(json.dumps({"reads": n_reads, "buckets": B, "passes": int(t["passes"]), "instances": int(t["instances"]), "distinct": int(distinct),
                          "local_sort_ms": statistics.median(sort_ms), "local_sort_ms_all": sort_ms,
                          "sort_lsd_fallbacks": int(t["sort_lsd_fallbacks"]), "sort_oversize_equal": int(t["sort_oversize_equal"]),
                          "phases_ms": runs, "gpu": torch.cuda.get_device_name(0)}), flush=True)
        del words, offs, lens
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
