"""Worker for tests/test_gpu_dist_kmers.py: the k-mers of a distributed (k+1)-mer set, run by W processes.

Every case: the ranks' read shards go through the distributed (k+1)-mer count (DistributedKMerCounter), then through the
distributed k-mers of the (k+1)-mers (DistributedKmersFromKpomers). Rank 0 checks
  - the union of the ranks' k-mer shards (keys, bucket sizes, device checksums) against the oracle's k-mers of the (k+1)-mers of
    the union of the reads;
  - assemble_kmer_index against the oracle's index of those k-mers, and byte for byte against the single-GPU index of the
    single-GPU k-mers of the union;
  - the bucket files every rank wrote into one directory (write_owned_buckets, (k+1)-mers and k-mers) against the single-GPU
    bucket files of the union: the same names, the same bytes.
Two ways to run it, as dist_worker: run_spawned (W processes on device 0 joined by gloo) and __main__ (torch.distributed.run,
one GPU per rank, NCCL).
"""
import os
import shutil
import sys
import tempfile
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dist_worker import ARENA_BYTES, PLANNER_RESERVE, _blocks, _empty_shards, _strided, _synth, oracle_checksum  # noqa: E402

READS = {
    "strided": lambda world, seed: _strided(_synth(3000, seed), world),
    "blocks": lambda world, seed: _blocks(_synth(3000, seed), world),
    # the last rank reads nothing, the one before it only reads shorter than k + 1 = 56: empty (k+1)-mer shards
    "empty": lambda world, seed: _empty_shards(world, 0),
}

# k: the k-mers' k (the source holds (k+1)-mers); B: buckets of the (k+1)-mer count; Bk: buckets of the k-mers (default B);
# budget: fixed per-pass budget of the k-mer count, bytes above the planner's reserve per record of the union (two per (k+1)-mer);
# host: source and result in host memory; overlap: every rank's source is the whole (k+1)-mer set of the union of the reads;
# Bk2: the same DistributedKmersFromKpomers counts again into Bk2 buckets
CASES = [
    dict(name="k21", k=21, B=16, reads="strided"),
    dict(name="k32_words2to1", k=32, B=16, Bk=24, reads="strided"),
    dict(name="k55", k=55, B=40, reads="blocks"),
    dict(name="k64", k=64, B=11, reads="strided"),
    dict(name="k127", k=127, B=7, reads="strided"),
    dict(name="k55_B1", k=55, B=1, reads="strided"),
    dict(name="k55_B2", k=55, B=2, reads="blocks"),
    dict(name="k55_B8192", k=55, B=8192, reads="strided"),
    dict(name="k55_passes", k=55, B=64, reads="strided", budget=2, min_passes=3),
    dict(name="k33_host", k=33, B=12, reads="strided", host=True, budget=2, min_passes=3),
    dict(name="k55_empty", k=55, B=16, reads="empty"),
    dict(name="k55_overlap", k=55, B=16, reads="strided", overlap=True),
    dict(name="k55_reuse", k=55, B=12, Bk=40, Bk2=9, reads="strided"),
]


def _same_files(got_dir, want_dir):
    got, want = sorted(os.listdir(got_dir)), sorted(os.listdir(want_dir))
    if got != want:
        return False
    for f in got:
        with open(os.path.join(got_dir, f), "rb") as a, open(os.path.join(want_dir, f), "rb") as b:
            if a.read() != b.read():
                return False
    return True


def check_count(ctx, case, Bk, shards, gathered, union_index, files_dir):
    """rank 0: one k-mer count of a case -> (names of failed checks, distinct k-mers of the union)"""
    import golden_util
    import oracle as O
    from spades_b200.kmer_index import DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    from spades_b200.packing import pack_reads
    k, B = case["k"], case["B"]
    union = [r for s in shards for r in s]
    okm = O.kmers_from_kpomers(O.count(*pack_reads(union), k + 1, B, 0), Bk)
    bad = []
    if not np.array_equal(sum(g["bsz"] for g in gathered), okm.bsz):
        bad.append("bucket_sizes")
    owned = np.stack([g["owned"] for g in gathered])
    if not (owned.sum(axis=0) == 1).all():
        bad.append("ownership")
    else:
        parts, offs = [], [0] * len(gathered)
        for b in range(Bk):
            r = int(np.flatnonzero(owned[:, b])[0])
            nb = int(gathered[r]["bsz"][b])
            parts.append(gathered[r]["keys"][offs[r]:offs[r] + nb])
            offs[r] += nb
        if not np.array_equal(np.concatenate(parts).ravel(), okm.keys.ravel()):
            bad.append("keys")
    m64 = (1 << 64) - 1
    cs = [g["checksum"] for g in gathered]
    tot = [sum(c[0] for c in cs), sum(c[1] for c in cs) & m64, 0, sum(c[3] for c in cs) & m64]
    for c in cs:
        tot[2] ^= c[2]
    if tot != oracle_checksum(okm):
        bad.append("checksum")
    if not golden_util.index_equal(O.Mphf(okm).serialize(), union_index, Bk):
        bad.append("index_oracle")
    # the single-GPU path over the union: its index bytes and its bucket files
    ctx.set_reads(*pack_reads(union))
    kp_u = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1)).Count(B)
    km_u = KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kp_u)).Count(Bk)
    idx_u = KMerIndexBuilder(ctx).BuildIndex(km_u)
    if idx_u.serialize() != union_index:
        bad.append("index_single_gpu")
    want_dir = files_dir + "_single_gpu"
    os.makedirs(want_dir)
    km_u.write_buckets(os.path.join(want_dir, "kmers"))
    if not case.get("overlap"):
        kp_u.write_buckets(os.path.join(want_dir, "kpomers"))
    if not _same_files(files_dir, want_dir):
        bad.append("bucket_files")
    idx_u.free(); km_u.free(); kp_u.free()
    npass = [g["npass"] for g in gathered]
    if len(set(npass)) != 1:
        bad.append("passes_differ")
    if case.get("budget") is not None and npass[0] < case["min_passes"]:
        bad.append("passes")
    if case.get("host"):
        if not all(g["on_host"] and g["src_on_host"] for g in gathered):
            bad.append("placement")
        if any(g["src_n"] > 0 and g["stage_h2d_bytes"] == 0 for g in gathered):
            bad.append("stage_h2d_bytes")
    return bad, okm.n


def run_cases(rank, world, device, backend, cases):
    """every case of `cases` over the default process group; the result lines on rank 0 (one per k-mer count: OK or the checks
    that failed), [] elsewhere; ["SKIP ..."] when a rank other than 0 cannot create its device context"""
    import re
    import torch
    import torch.distributed as dist
    from spades_b200.distributed import DistributedKMerCounter, DistributedKmersFromKpomers, assemble_kmer_index
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder, SpadesGpuError
    from spades_b200.packing import pack_reads
    assert dist.get_backend() == backend, (dist.get_backend(), backend)
    ctx, err = None, None
    try:
        ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    except SpadesGpuError as e:
        err = str(e)
    errs = [None] * world
    dist.all_gather_object(errs, err)
    failed = [(r, e) for r, e in enumerate(errs) if e is not None]
    if failed:
        r, e = failed[0]
        m = re.search(r"code (\d+)", e)
        if r == 0 or not m or int(m.group(1)) != 3:
            raise RuntimeError("rank %d: %s" % (r, e))
        return ["SKIP rank %d of %d on device %d cannot create a device context (%s)" % (r, world, device, e)] if rank == 0 else []
    top = [tempfile.mkdtemp(prefix="dist_kmers_") if rank == 0 else None]
    dist.broadcast_object_list(top, src=0)
    top = top[0]
    lines = []
    for ci, case in enumerate(cases):
        k, B, host = case["k"], case["B"], case.get("host", False)
        shards = READS[case["reads"]](world, 7000 + ci)
        if case.get("overlap"):
            ctx.set_reads(*pack_reads([r for s in shards for r in s]))
            kp = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1), result_on_host=host).Count(B)
        else:
            ctx.set_reads(*pack_reads(shards[rank]))
            kp = DistributedKMerCounter(ctx, k + 1, result_on_host=host).Count(B)
        budget = None
        if case.get("budget") is not None:
            n_kp = [0] * world
            dist.all_gather_object(n_kp, kp.total_kmers())
            budget = PLANNER_RESERVE + case["budget"] * 2 * sum(n_kp)
        counter = DistributedKmersFromKpomers(ctx, kp, result_on_host=host)
        for Bk in [case.get("Bk", B)] + ([case["Bk2"]] if "Bk2" in case else []):
            km = counter.Count(Bk, budget_bytes=budget)
            stage = ctx.times()["stage_h2d_bytes"]          # the index build below starts its own count
            idx = KMerIndexBuilder(ctx).BuildIndex(km)
            union_index = assemble_kmer_index(ctx, km, idx)
            files_dir = os.path.join(top, "%s_B%d" % (case["name"], Bk))
            os.makedirs(files_dir, exist_ok=True)
            km.write_owned_buckets(os.path.join(files_dir, "kmers"))
            if not case.get("overlap"):
                kp.write_owned_buckets(os.path.join(files_dir, "kpomers"))
            res = dict(keys=km.kmers(), bsz=km.bucket_sizes(), owned=km.owned_buckets(), checksum=km.checksum(), npass=counter.npass,
                       stage_h2d_bytes=stage, src_n=kp.total_kmers(), on_host=km.on_host(), src_on_host=kp.on_host())
            idx.free(); km.free()
            gathered = [None] * world
            dist.all_gather_object(gathered, res)        # also: every rank's bucket files are written
            if rank == 0:
                bad, n = check_count(ctx, case, Bk, shards, gathered, union_index, files_dir)
                line = "dist kmers W=%d %-14s k=%-3d B=%-4d Bk=%-4d passes=%-2d distinct=%-7d %s" % (
                    world, case["name"], k, B, Bk, gathered[0]["npass"], n, "OK" if not bad else "FAIL " + ",".join(bad))
                print(line, flush=True)
                lines.append(line)
            dist.barrier()
        kp.free()
    dist.barrier()
    if rank == 0:
        shutil.rmtree(top, ignore_errors=True)
    ctx.close()
    return lines


def expected_lines(cases):
    return sum(1 + ("Bk2" in c) for c in cases)


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
