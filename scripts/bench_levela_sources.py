#!/usr/bin/env python
"""Level-A times of the count's two other sources on one GPU: the all-windows count of the reads (spades-kmercount) and the
k-mers of the (k+1)-mers (the graph path's second count), over synthetic 150 bp reads generated as bench.py does.

    python scripts/bench_levela_sources.py [--reads 10000000] [--k 55 21] [--reps 3]

Prints one JSON line per (source, k): the medians over --reps runs of extract_count_ms (levelA_count_roll_k and the partition
totals) and extract_scatter_ms (levelA_scatter_roll_k, every pass), the path counters, and the set's order-independent
checksum, so that two builds can be compared on the same input. The (k+1)-mer set is counted once per k and is not timed.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402  (the read generator and constants of the bench)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, nargs="+", default=[55, 21])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--buckets", type=int, default=0, help="0 = 10 x host threads, as bench.py")
    args = ap.parse_args()
    import statistics
    import torch
    from spades_b200.kmer_index import (Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter,
                                        ParallelSortingSplitter)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    nb = args.buckets or 10 * B.host_threads()
    n = args.reads
    words, offs, lens, nwr = B.gen_reads_device(torch, n, max(B.READ_LEN + 1, n), 42, dev)
    torch.cuda.synchronize(); torch.cuda.empty_cache()
    ctx = Context(0, stream=torch.cuda.current_stream().cuda_stream)
    ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
    info = card()

    def measure(source, k, count):
        runs, sums = [], set()
        for _ in range(args.reps + 1):                    # the first run warms up
            st = count()
            t = ctx.times()
            sums.add(tuple(int(x) for x in st.checksum()))
            st.free()
            runs.append({q: t[q] for q in ("extract_count_ms", "extract_scatter_ms", "passes", "level_a_scatters")})
        timed = runs[1:]
        line = dict(info, source=source, k=k, reads=n, buckets=nb,
                    extract_count_ms=round(statistics.median(r["extract_count_ms"] for r in timed), 2),
                    extract_scatter_ms=round(statistics.median(r["extract_scatter_ms"] for r in timed), 2),
                    extract_count_ms_all=[round(r["extract_count_ms"], 2) for r in timed],
                    extract_scatter_ms_all=[round(r["extract_scatter_ms"], 2) for r in timed],
                    passes=int(timed[0]["passes"]), level_a_scatters=int(timed[0]["level_a_scatters"]),
                    checksum=[list(s) for s in sorted(sums)])
        print(json.dumps(line), flush=True)

    for k in args.k:
        measure("all_windows", k, lambda: KMerDiskCounter(ctx, ParallelSortingSplitter(k)).Count(nb))
        kp = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1)).Count(nb)
        measure("kmers_from_kpomers", k, lambda: KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kp)).Count(nb))
        kp.free()
    ctx.close()


if __name__ == "__main__":
    main()
