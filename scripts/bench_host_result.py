#!/usr/bin/env python
"""Counts whose result goes to host memory (SGPU_RESULT_ON_HOST), measured on the bench's workload: 150 bp synthetic reads, k = 55
(canonical 56-mers), the bench's bucket count. Prints one JSON line (and writes it to --out when given).

  compare   (a) device-set count + MPHF + serialized index + download of every record and multiplicity into pinned memory (the
                bench's e2e_storage leg plus the multiplicities), against
            (b) host-result count + MPHF + serialized index.
            Reads are uploaded from pinned memory in both. Three runs of each, alternating; median and spread of host-clock seconds
            around work that ends in a device synchronise. Also: result_d2h_wait_ms of (b), the time torch takes to pin as many
            bytes as (b)'s set holds, and whether the two sets' checksums are equal.
  capacity  the largest read count up to --max-reads that free host memory allows with 16 GB to spare (psutil), counted with the
            result on the host: count and MPHF seconds, passes, peak HBM, total of the bucket sizes, and whether the MPHF build's
            rank check (the index is minimal: every bucket's rank total equals its size) passed.

    python scripts/bench_host_result.py [--reads 40000000] [--max-reads 125000000] [--runs 3] [--out file.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HEADROOM = 16 << 30          # host memory left free, as bench.py's e2e_storage leg does


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": float(out[2]), "max_sm_clock_mhz": float(out[3])}
    except Exception as ex:
        return {"error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=40_000_000)
    ap.add_argument("--max-reads", type=int, default=125_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--buckets", type=int, default=0)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import psutil
    import torch
    import bench
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_result.py: no CUDA device; this path has no CPU fallback")
    K, L = bench.K, bench.READ_LEN
    B = args.buckets or 10 * bench.host_threads()
    dev = torch.device("cuda", 0)
    res = {"card_before": card(), "K": K, "read_len": L, "buckets": B}

    # ---- compare (a) / (b) at --reads
    n = args.reads
    w, o, ln, nwr = bench.gen_reads_device(torch, n, max(L + 1, n), 42, dev)
    h_words, h_offs, h_lens = w[: n * nwr].cpu().pin_memory(), o.cpu().pin_memory(), ln.cpu().pin_memory()
    del w, o, ln
    torch.cuda.synchronize(); torch.cuda.empty_cache()
    ctx = Context(0)
    h_index = None

    def upload():
        ctx.upload_reads(h_words.data_ptr(), n * nwr, h_offs.data_ptr(), h_lens.data_ptr(), n)

    def index(st):
        nonlocal h_index
        idx = KMerIndexBuilder(ctx).BuildIndex(st)
        need = idx.serialized_size()
        if h_index is None or h_index.numel() < need:
            h_index = torch.empty(int(need * 1.05) + 4096, dtype=torch.uint8).pin_memory()
        idx.serialize_into(h_index.data_ptr(), h_index.numel())
        idx.free()

    # (a)'s destination buffers are pinned once, outside the timed runs
    upload()
    st = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(K)).Count(B)
    distinct, nw = st.total_kmers(), st.nw
    want_cs = st.checksum()
    st.free()
    result_bytes = distinct * (8 * nw + 4)
    res["compare"] = {"reads": n, "distinct": distinct, "result_gb": result_bytes / 1e9}
    if psutil.virtual_memory().available < 2 * result_bytes + HEADROOM:
        res["compare"]["skipped"] = "host memory: %.1f GB available, (a)'s buffers and (b)'s set need %.1f GB + 16 GB" % (
            psutil.virtual_memory().available / 1e9, 2 * result_bytes / 1e9)
    else:
        h_keys = torch.empty(distinct * nw, dtype=torch.int64, pin_memory=True)
        h_cnt = torch.empty(distinct, dtype=torch.int32, pin_memory=True)

        def step_a():
            upload()
            s = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(K)).Count(B)
            index(s)
            s.download_keys_into(h_keys.data_ptr(), s.total_kmers())
            ctx.check(ctx.L.sgpu_kset_download_counts(s.h, 0, s.total_kmers(), h_cnt.data_ptr()))
            s.free()

        host_cs = []

        def step_b(last):
            upload()
            t0 = time.perf_counter()
            s = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(K), result_on_host=True).Count(B)
            t = dict(ctx.times(), count_s=time.perf_counter() - t0)
            index(s)
            torch.cuda.synchronize()
            if last:
                host_cs.append(s.checksum())
            s.free()
            return t

        ta, tb, tb_count, waits, d2h = [], [], [], [], []
        step_a(); step_b(False)            # warm-up of every shape
        for r in range(args.runs):
            torch.cuda.synchronize(); t0 = time.perf_counter(); step_a(); torch.cuda.synchronize(); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            t = step_b(False)
            tb.append(time.perf_counter() - t0)
            waits.append(t["result_d2h_wait_ms"]); d2h.append(t["result_d2h_bytes"]); tb_count.append(t["count_s"])
        step_b(True)
        del h_keys, h_cnt
        torch._C._host_emptyCache()        # torch's pinned-block cache would hand the freed buffers back without pinning anything
        t0 = time.perf_counter()
        pin = torch.empty(result_bytes, dtype=torch.uint8, pin_memory=True)
        pin_s = time.perf_counter() - t0
        del pin
        torch._C._host_emptyCache()
        res["compare"].update({
            "a_device_set_then_download_s": {"median": statistics.median(ta), "min": min(ta), "max": max(ta), "runs": ta},
            "b_host_result_s": {"median": statistics.median(tb), "min": min(tb), "max": max(tb), "runs": tb},
            "b_count_only_s": tb_count, "b_result_d2h_wait_ms": waits, "b_result_d2h_bytes": d2h[-1],
            "pin_same_bytes_with_torch_s": pin_s,
            "checksums_equal": host_cs[0] == want_cs})
    ctx.close()
    del h_words, h_offs, h_lens
    torch.cuda.empty_cache(); torch._C._host_emptyCache()

    # ---- capacity: the largest read count host memory allows, result on the host
    per_read = result_bytes / n
    avail = psutil.virtual_memory().available
    nc = int(min(args.max_reads, (avail - HEADROOM) / per_read))
    nc -= nc % 1_000_000
    cap = {"max_reads": args.max_reads, "host_available_gb": avail / 1e9, "estimated_result_gb_per_m_reads": per_read * 1e6 / 1e9, "reads": nc}
    if nc < 1_000_000:
        cap["skipped"] = "not enough free host memory"
    else:
        w, o, ln, nwr = bench.gen_reads_device(torch, nc, max(L + 1, nc), 43, dev)
        torch.cuda.synchronize(); torch.cuda.empty_cache()
        ctx = Context(0)
        ctx.adopt_device_reads(w.data_ptr(), nc * nwr, o.data_ptr(), ln.data_ptr(), nc)
        t0 = time.perf_counter()
        st = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(K), result_on_host=True).Count(B)
        count_s = time.perf_counter() - t0
        t = ctx.times()
        bsz_total = int(np.asarray(st.bucket_sizes()).sum())
        t0 = time.perf_counter()
        try:
            idx = KMerIndexBuilder(ctx).BuildIndex(st)
            rank_check = True
            idx.free()
        except Exception as ex:
            rank_check = "failed: %s" % ex
        mphf_s = time.perf_counter() - t0
        cap.update({"distinct": st.total_kmers(), "bucket_sizes_total": bsz_total, "result_gb": st.total_kmers() * (8 * st.nw + 4) / 1e9,
                    "count_s": count_s, "mphf_s": mphf_s, "passes": t["passes"], "peak_hbm_gb": ctx.times()["peak_bytes"] / 1e9,
                    "result_d2h_wait_ms": t["result_d2h_wait_ms"], "mphf_rank_check_passed": rank_check})
        st.free()
        ctx.close()
        del w, o, ln
    res["capacity"] = cap
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
