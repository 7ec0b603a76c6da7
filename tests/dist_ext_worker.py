"""Worker for tests/test_gpu_dist_ext.py: the extension masks, coverage and histogram of distributed sets, run by W processes.

Every case: the ranks' read shards go through the distributed (k+1)-mer count, the distributed k-mers of the (k+1)-mers, both
indexes and DistributedExtensionIndexBuilder.Build. Rank 0 checks the assembled masks and coverage and the histogram byte for byte
against the single-GPU graph build over the union of the reads (early clippers off) and against the oracle. Two ways to run it, as
dist_worker: run_spawned (W processes on device 0 joined by gloo) and __main__ (torch.distributed.run, one GPU per rank, NCCL).
"""
import os
import sys
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dist_worker import ARENA_BYTES, _blocks, _empty_shards, _random_seq, _selfrc, _strided, _synth  # noqa: E402,F401


def _canonical_buckets(seqs, K, B):
    """kmer_bucket of the minimal form of every length-K string of `seqs` (host arithmetic of the library's self test)"""
    import ctypes as C
    from spades_b200 import _lib
    from spades_b200.packing import pack_reads, revcomp
    L = _lib.load()
    nw = (K + 31) // 32

    def words(ss):
        w, offs, _ = pack_reads(ss)
        return np.stack([w[int(o):int(o) + nw] for o in offs]).astype(np.uint64)
    fw, rc = words(seqs), words([revcomp(s) for s in seqs])
    n = len(seqs)
    is_min = np.zeros(n, np.uint64)
    L.sgpu_selftest(None, 0, 4, K, 0, np.ascontiguousarray(fw).ctypes.data_as(C.c_void_p), n, is_min.ctypes.data_as(C.c_void_p))
    canon = np.ascontiguousarray(np.where(is_min[:, None] == 1, fw, rc))
    b = np.zeros(n, np.uint64)
    L.sgpu_selftest(None, 0, 3, K, B, canon.ctypes.data_as(C.c_void_p), n, b.ctypes.data_as(C.c_void_p))
    return b.astype(np.int64)


def _skew(world, k, B):
    # reads of exactly k + 1 bases whose (k+1)-mer lies in a bucket of rank 0 and whose two k-mers both lie in buckets of the last
    # rank (one pass of the distributed counts splits the buckets into contiguous ranges, distributed.owner_bounds): every
    # contribution rank 0 holds goes to another owner. The reads are split strided over the ranks, as any shard would be.
    from spades_b200.distributed import owner_bounds
    rng = np.random.default_rng(900 + k)
    ob = owner_bounds(0, B, world)
    cand = [_random_seq(rng, k + 1) for _ in range(6000 * world * world)]
    bkp = _canonical_buckets(cand, k + 1, B)
    bpre = _canonical_buckets([s[:k] for s in cand], k, B)
    bsuf = _canonical_buckets([s[1:] for s in cand], k, B)
    lo0, hi0, lo1, hi1 = ob[0], ob[1], ob[world - 1], ob[world]
    keep = (bkp >= lo0) & (bkp < hi0) & (bpre >= lo1) & (bpre < hi1) & (bsuf >= lo1) & (bsuf < hi1)
    reads = [s for s, ok in zip(cand, keep) if ok]
    return _strided(reads * 2, world)


READS = {
    "strided": lambda world, case, seed: _strided(_synth(3000, seed), world),
    "blocks": lambda world, case, seed: _blocks(_synth(3000, seed), world),
    # the last rank reads nothing, the one before it only reads shorter than k + 1 = 56
    "empty": lambda world, case, seed: _empty_shards(world, 0),
    # palindromes x + revcomp(x), |x| = 60: their middle (k+1)-mer for k = 55 is its own reverse complement, so both of its bits
    # land on one k-mer
    "selfrc": lambda world, case, seed: _selfrc(world, 0),
    "skew": lambda world, case, seed: _skew(world, case["k"], case["B"]),
}

# k: the k-mers' k; B: buckets of both counts; budget: fixed budget of every mask pass, as a fraction of the bytes of all
# contributions over the world size (forces that many passes at least); host: both sets in host memory; overlap: every rank's
# (k+1)-mer source is the whole set of the union of the reads (the coverage is refused, the masks are still the union's)
CASES = [
    dict(name="k21", k=21, B=16, reads="strided"),
    dict(name="k31", k=31, B=16, reads="blocks"),
    dict(name="k55", k=55, B=40, reads="blocks"),
    dict(name="k63", k=63, B=11, reads="strided"),
    dict(name="k95", k=95, B=9, reads="strided"),
    dict(name="k127", k=127, B=7, reads="strided"),
    dict(name="k55_B1", k=55, B=1, reads="strided"),
    dict(name="k55_B2", k=55, B=2, reads="blocks"),
    dict(name="k55_B8192", k=55, B=8192, reads="strided"),
    dict(name="k55_passes", k=55, B=64, reads="strided", budget=12, min_passes=8),
    dict(name="k33_host", k=33, B=12, reads="strided", host=True, budget=4, min_passes=2),
    dict(name="k55_empty_short", k=55, B=16, reads="empty"),
    dict(name="k55_skew", k=55, B=8, reads="skew"),
    dict(name="k55_selfrc", k=55, B=7, reads="selfrc"),
    dict(name="k55_overlap", k=55, B=16, reads="strided", overlap=True),
]


def check_case(ctx, case, shards, masks, cov, hist, npass):
    """rank 0: the assembled arrays against the single-GPU graph build and the oracle over the union -> names of failed checks"""
    import oracle as O
    from spades_b200.graph import DeBruijnGraphConstructor
    from spades_b200.packing import pack_reads
    k, B = case["k"], case["B"]
    union = [r for s in shards for r in s]
    bad = []
    ctx.set_reads(*pack_reads(union))
    g = DeBruijnGraphConstructor(ctx, k, B).ConstructGraph()
    if not np.array_equal(masks, g.masks()):
        bad.append("masks_single_gpu")
    if cov is not None:
        if not np.array_equal(cov, g.coverage()):
            bad.append("coverage_single_gpu")
        if not np.array_equal(hist, g.histogram()):
            bad.append("histogram_single_gpu")
    g.free()
    kp = O.count(*pack_reads(union), k + 1, B, 0)
    km = O.kmers_from_kpomers(kp, B)
    if not np.array_equal(masks, O.masks(kp, O.Mphf(km), km.n)):
        bad.append("masks_oracle")
    if cov is not None:
        ocov = O.coverage(kp, O.Mphf(kp))
        if not np.array_equal(cov, ocov):
            bad.append("coverage_oracle")
        if not np.array_equal(hist, O.histogram(ocov)):
            bad.append("histogram_oracle")
    if len(set(npass)) != 1:
        bad.append("passes_differ")
    if case.get("min_passes") and npass[0] < case["min_passes"]:
        bad.append("passes")
    return bad, km.n


def run_cases(rank, world, device, backend, cases):
    """every case over the default process group; the result lines on rank 0 (OK or the checks that failed), [] elsewhere"""
    import torch.distributed as dist
    from spades_b200.distributed import (DistributedExtensionIndexBuilder, DistributedKMerCounter, DistributedKmersFromKpomers, assemble_coverage,
                                         assemble_masks)
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    from spades_b200.packing import pack_reads
    assert dist.get_backend() == backend, (dist.get_backend(), backend)
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    lines = []
    for ci, case in enumerate(cases):
        k, B, host = case["k"], case["B"], case.get("host", False)
        shards = READS[case["reads"]](world, case, 8000 + ci)
        if case.get("overlap"):
            ctx.set_reads(*pack_reads([r for s in shards for r in s]))
            kp = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1), result_on_host=host).Count(B)
        else:
            ctx.set_reads(*pack_reads(shards[rank]))
            kp = DistributedKMerCounter(ctx, k + 1, result_on_host=host).Count(B)
        km = DistributedKmersFromKpomers(ctx, kp, result_on_host=host).Count(B)
        mkp = KMerIndexBuilder(ctx).BuildIndex(kp)
        mk = KMerIndexBuilder(ctx).BuildIndex(km)
        budget = None
        if case.get("budget"):
            n_kp = [0] * world
            dist.all_gather_object(n_kp, kp.total_kmers())
            budget = max(1, 2 * sum(n_kp) * (8 * km.nw + 1) // (case["budget"] * world))
        refused = None
        ext = None
        if case.get("overlap"):
            try:
                ext = DistributedExtensionIndexBuilder(ctx, kp, mkp, km, mk).Build(budget)
            except ValueError as e:
                refused = str(e)
            if ext is not None:
                ext.free()
        if ext is None or case.get("overlap"):
            ext = DistributedExtensionIndexBuilder(ctx, kp, None if case.get("overlap") else mkp, km, mk).Build(budget)
        masks = assemble_masks(ext)
        cov = None if case.get("overlap") else assemble_coverage(ext)
        hist = None if case.get("overlap") else ext.histogram()
        res = dict(npass=ext.npass, on_host=kp.on_host() and km.on_host(), refused=refused)
        if case["reads"] == "skew" and rank == 0 and world > 1:
            # the case is what it claims: rank 0 has contributions, and none of them is to a bucket it owns
            res["skew_ok"] = bool(ext.local_counts.sum() > 0 and ext.local_counts[km.owned_buckets()].sum() == 0)
        ext.free(); mk.free(); mkp.free(); km.free(); kp.free()
        gathered = [None] * world
        dist.all_gather_object(gathered, res)
        if rank == 0:
            bad, n = check_case(ctx, case, shards, masks, cov, hist, [r["npass"] for r in gathered])
            if gathered[0].get("skew_ok") is False:
                bad.append("skew_not_exercised")
            if host and not all(r["on_host"] for r in gathered):
                bad.append("placement")
            if case.get("overlap") and (gathered[0]["refused"] is None) != (world == 1):
                bad.append("coverage_not_refused" if world > 1 else "coverage_refused")
            line = "dist ext W=%d %-16s k=%-3d B=%-4d passes=%-3d kmers=%-7d %s" % (
                world, case["name"], k, B, gathered[0]["npass"], n, "OK" if not bad else "FAIL " + ",".join(bad))
            print(line, flush=True)
            lines.append(line)
        dist.barrier()
    ctx.close()
    return lines


def run_spawned(rank, world, port, out_path, cases):
    """mp.spawn entry: W ranks on device 0 over gloo; rank 0 writes the result lines to out_path"""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world, timeout=timedelta(seconds=600))
    try:
        lines = run_cases(rank, world, 0, "gloo", cases)
    finally:
        dist.destroy_process_group()
    if rank == 0:
        with open(out_path, "w") as f:
            f.write("\n".join(lines) + "\n")


def run_gpu():
    """torch.distributed.run entry: one GPU per rank, NCCL; rank 0 prints the result lines"""
    import torch
    import torch.distributed as dist
    rank, world, lrank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lrank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lrank), timeout=timedelta(seconds=600))
    lines = run_cases(rank, world, lrank, "nccl", CASES)
    dist.destroy_process_group()
    if rank == 0 and any(not ln.endswith(" OK") for ln in lines):
        sys.exit(1)


if __name__ == "__main__":
    try:
        run_gpu()
    except Exception:
        import traceback
        traceback.print_exc()
        sys.stdout.flush(); sys.stderr.flush()
        os._exit(1)
