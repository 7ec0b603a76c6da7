#!/usr/bin/env python
"""FASTG and unitig FASTA formatted on the GPU, with the host GFA writer for context: synthetic 150 bp reads -> graph (k = 55, 80
buckets by default) built once, then write_fastg, write_unitigs_fasta and write_gfa each timed as the median of 3 calls after one
warm-up call. Per format: the call's wall time and what the formatter reports: host milliseconds for the vertex structure and for
the record sizes, device formatting and device-to-host copy milliseconds, host write milliseconds, runs and output bytes. The files go to a temporary directory that is removed afterwards.

    python scripts/bench_fastg.py [--reads 20000000] [--samples 100000]

Checks at that size: the FASTG has 2E - (self-conjugate edges) records and twice the bases of the non-self-conjugate edges plus
those of the self-conjugate ones, the unitig FASTA E records and the unitig bases. A random sample of FASTG records is checked
partially (the graph's raw coverages and vertex lists are not visible from Python): the body, the id and length in the record's
own name, its orientation mark, and successor names that are sorted, distinct, at most four, and start where the record ends. The
coverage text and the completeness of the successor set are not checked here; the test suite checks them against the reference.
Sampled unitig FASTA records are compared whole.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench as B  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def scan_records(path, want_offsets):
    """(records, body bases) of a FASTA text, and the text of the records whose index is in want_offsets"""
    n = bases = 0
    keep, cur = {}, None
    with open(path, "rb") as f:
        for line in f:
            if line[:1] == b">":
                if cur is not None:
                    keep[cur[0]] = b"".join(cur[1]).decode()
                cur = (n, [line]) if n in want_offsets else None
                n += 1
            else:
                bases += len(line) - 1
                if cur is not None:
                    cur[1].append(line)
    if cur is not None:
        keep[cur[0]] = b"".join(cur[1]).decode()
    return n, bases, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000_000)
    ap.add_argument("--buckets", type=int, default=80)
    ap.add_argument("--samples", type=int, default=100_000)
    args = ap.parse_args()
    import numpy as np
    import torch
    import fastg_oracle as F
    from spades_b200.graph import DeBruijnGraph
    from spades_b200.kmer_index import Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    from spades_b200._lib import SgpuGraphOptions
    import ctypes as C
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    k, nb, n = B.K_GRAPH, args.buckets, args.reads
    words, offs, lens, nwr = B.gen_reads_device(torch, n, max(B.READ_LEN + 1, n), 42, dev)
    torch.cuda.synchronize(); torch.cuda.empty_cache()
    ctx = Context(0, stream=torch.cuda.current_stream().cuda_stream)
    ctx.adopt_device_reads(words.data_ptr(), n * nwr, offs.data_ptr(), lens.data_ptr(), n)
    kp = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1)).Count(nb)
    km = KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kp)).Count(nb)
    mk, mkp = KMerIndexBuilder(ctx).BuildIndex(km), KMerIndexBuilder(ctx).BuildIndex(kp)
    h = C.c_void_p()
    ctx.check(ctx.L.sgpu_graph_build_opts(ctx.h, kp.h, km.h, mk.h, mkp.h, C.byref(SgpuGraphOptions(1, 0, 0, 0.8, 10, 200)), C.byref(h)))
    g = DeBruijnGraph(ctx, h, kp, km, mk, mkp)
    del words, offs, lens
    torch.cuda.empty_cache()
    unitigs = g.unitigs()
    E = len(unitigs)
    result = {"reads": n, "k": k, "buckets": nb, "edges": E, "card": card()}
    with tempfile.TemporaryDirectory() as d:
        for what, fn in (("fastg", g.write_fastg), ("unitigs_fasta", g.write_unitigs_fasta), ("gfa", g.write_gfa)):
            path = os.path.join(d, what)
            walls, stats = [], []
            for rep in range(4):
                torch.cuda.synchronize(); t0 = time.perf_counter()
                fn(path)
                walls.append((time.perf_counter() - t0) * 1e3)
                if what != "gfa":
                    stats.append(g.format_stats())
            walls, stats = walls[1:], stats[1:]
            r = {"wall_ms_median": round(statistics.median(walls), 1), "bytes": os.path.getsize(path)}
            if stats:
                for q in ("vertices_ms", "sizes_ms", "format_ms", "d2h_ms", "write_ms"):
                    r[q + "_median"] = round(statistics.median(s[q] for s in stats), 1)
                r["runs"] = stats[-1]["runs"]
            result[what] = r
            if what == "fastg":
                selfc = [s == F.revcomp(s) for s in unitigs]
                R = 2 * E - sum(selfc)
                rng = np.random.default_rng(1)
                sample = set(int(x) for x in rng.choice(R, min(args.samples, R), replace=False))
                nrec, bases, keep = scan_records(path, sample)
                want_bases = sum(len(s) * (1 if c else 2) for s, c in zip(unitigs, selfc))
                sc = np.array(selfc, np.int64)
                first = 2 * np.arange(E, dtype=np.int64) - np.concatenate(([0], np.cumsum(sc)[:-1]))    # each edge's first record
                bad = 0
                for r_i, text in keep.items():
                    i = int(np.searchsorted(first, r_i, "right")) - 1
                    st = r_i - int(first[i])
                    head, body = text.split("\n", 1)
                    seq = unitigs[i] if st == 0 else F.revcomp(unitigs[i])
                    own, _, nxt = head[1:-1].partition(":")
                    names = nxt.split(",") if nxt else []
                    ok = body == F.wrapped(seq) and own.startswith("EDGE_%d_length_%d_cov_" % (3 + 2 * i, len(seq)))
                    ok = ok and own.endswith("'") == (st == 1) and names == sorted(set(names)) and len(names) <= 4
                    for x in names:
                        j = (int(x.split("_")[1]) - 3) // 2
                        s2 = F.revcomp(unitigs[j]) if x.endswith("'") else unitigs[j]
                        ok = ok and s2[:k] == seq[-k:]
                    bad += not ok
                result["fastg_check"] = {"records": nrec, "want_records": R, "bases": bases, "want_bases": want_bases,
                                         "sampled": len(keep), "sample_mismatches": bad}
            elif what == "unitigs_fasta":
                nrec, bases, keep = scan_records(path, set(range(min(args.samples, E))))
                bad = sum(keep[i] != F.unitigs_fasta([unitigs[i]]).replace(">EDGE_1_", ">EDGE_%d_" % (i + 1), 1) for i in keep)
                result["unitigs_check"] = {"records": nrec, "want_records": E, "bases": bases, "want_bases": sum(map(len, unitigs)),
                                           "sampled": len(keep), "sample_mismatches": bad}
    print(json.dumps(result), flush=True)
    g.free()
    ctx.close()


if __name__ == "__main__":
    main()
