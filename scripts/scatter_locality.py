"""Does the level-A radix partition lose its time to page spread? Two measurements, one command, on one GPU.

1. `levelA_scatter` (phase `extract_scatter_ms` of sgpu_times) at bench.py's shape (k = 55, 150 bp synthetic reads, B = 10 x host
   threads) with SGPU_A_SUB = 1, 2 and 4 partition sub-ranges, on a single-pass 10 M-read job and the 40 M-read job (4 passes).
   SGPU_A_SUB is read once per process, so every (setting, round) is a child process; settings alternate within a round.
2. scripts/microbench/scatter_bench.cu in its page-locality mode: 640 streams per CTA, 57 MB per CTA (one pass of the 40 M-read
   job spread over 264 CTAs) written into one region vs in slices of 16, 4 and 2 MB.

    python scripts/scatter_locality.py [--out DIR] [--rounds 3] [--steps 2]
Prints one JSON line per child and a summary; writes DIR/scatter_locality.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(reads_list, steps):
    sys.path.insert(0, ROOT)
    import torch
    import bench
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter
    dev = torch.device("cuda", 0)
    B = 10 * bench.host_threads()
    out = {"a_sub": os.environ.get("SGPU_A_SUB"), "buckets": B, "jobs": []}
    ctx = None
    for n in reads_list:
        w, o, l, nwr = bench.gen_reads_device(torch, n, max(bench.READ_LEN + 1, n), 42, dev)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        if ctx is None:
            ctx = Context(0, stream=torch.cuda.current_stream().cuda_stream)
        ctx.adopt_device_reads(w.data_ptr(), n * nwr, o.data_ptr(), l.data_ptr(), n)
        cnt = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(bench.K))
        cnt.Count(B).free()                                  # warm-up
        sc, tot = [], []
        for _ in range(steps):
            st = cnt.Count(B)
            t = ctx.times()
            sc.append(t["extract_scatter_ms"]); tot.append(t["extract_count_ms"] + t["extract_scatter_ms"] + t["refine_ms"] + t["local_sort_ms"] + t["compact_ms"])
            passes, scatters = t["passes"], t["level_a_scatters"]
            st.free()
        out["jobs"].append({"reads": n, "passes": int(passes), "level_a_scatters": int(scatters), "scatter_ms": sc, "count_ms": tot})
        del w, o, l
        torch.cuda.empty_cache()
    print("CHILD " + json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--reads", default="10000000,40000000")
    ap.add_argument("--subs", default="1,2,4")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-micro", action="store_true")
    a = ap.parse_args()
    reads = [int(x) for x in a.reads.split(",")]
    if a.child:
        child(reads, a.steps)
        return
    sys.path.insert(0, ROOT)
    import bench
    gpu = bench.gpu_facts(0)
    print("gpu", json.dumps(gpu), flush=True)
    results = {"gpu": gpu, "scatter": [], "micro": None}
    for rnd in range(a.rounds):
        for sub in a.subs.split(","):
            env = dict(os.environ, SGPU_A_SUB=sub)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reads", a.reads, "--steps", str(a.steps)], env=env,
                               capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("CHILD ")]
            if p.returncode or not line:
                print(p.stdout[-3000:], p.stderr[-3000:], flush=True)
                raise SystemExit("child SGPU_A_SUB=%s failed" % sub)
            r = json.loads(line[0][6:])
            r["round"] = rnd
            results["scatter"].append(r)
            print(json.dumps(r), flush=True)
    summary = {}
    for r in results["scatter"]:
        for j in r["jobs"]:
            summary.setdefault((j["reads"], r["a_sub"]), []).extend(j["scatter_ms"])
    for (n, sub), v in sorted(summary.items()):
        print("reads %9d  A_SUB %s  scatter ms: median %7.1f  min %7.1f  max %7.1f  (n=%d)" % (n, sub, statistics.median(v), min(v), max(v), len(v)), flush=True)
    if not a.skip_micro:
        with tempfile.TemporaryDirectory() as d:
            exe = os.path.join(d, "scatter_bench")
            subprocess.check_call(["nvcc", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                                   os.path.join(ROOT, "scripts", "microbench", "scatter_bench.cu")])
            p = subprocess.run([exe, "-c", "57", "-S", "640", "-r", "57", "-r", "16", "-r", "4", "-r", "2"], capture_output=True, text=True)
            print(p.stdout, p.stderr, flush=True)
            results["micro"] = p.stdout
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "scatter_locality.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
