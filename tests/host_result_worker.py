"""Worker of test_gpu_host_result.test_distributed_host_result: W processes on device 0 joined by gloo run the distributed count
with each rank's set in host memory (SGPU_RESULT_ON_HOST) and fixed multi-pass budgets. Rank 0 checks every rank's set against
the oracle's count of the union (dist_worker.check_case) and the summed checksums against a single-GPU count of the union, and
writes one line per case."""
from datetime import timedelta

from dist_worker import ALLWIN, ARENA_BYTES, CANON, PLANNER_RESERVE, READS, check_case

CASES = [
    dict(name="k33_nw2", K=33, B=40, mode=CANON, reads="k33", budget=6, min_passes=2),
    dict(name="k56_selfrc", K=56, B=7, mode=CANON, reads="selfrc", budget=6, min_passes=2),
    dict(name="k78_passes", K=78, B=64, mode=CANON, reads="all_ctas", budget=6, min_passes=3),
    dict(name="k128_passes", K=128, B=11, mode=CANON, reads="wide128", budget=6, min_passes=3),
    dict(name="k32_allwin", K=32, B=16, mode=ALLWIN, reads="allwin", budget=6, min_passes=2),
    dict(name="k56_empty", K=56, B=16, mode=CANON, reads="empty_shards", budget=6, min_passes=2),
]


def run_cases(rank, world):
    import torch
    import torch.distributed as dist
    from spades_b200.distributed import DistributedKMerCounter
    from spades_b200.kmer_index import Context, KMerDiskCounter, KMerIndexBuilder, SpadesGpuError
    from spades_b200.packing import pack_reads
    ctx, err = None, None
    try:
        ctx = Context(0, hbm_budget_bytes=ARENA_BYTES)
    except SpadesGpuError as e:
        err = str(e)
    errs = [None] * world
    dist.all_gather_object(errs, err)
    failed = [(r, e) for r, e in enumerate(errs) if e is not None]
    if failed:
        if rank == 0 and failed[0][0] != 0:
            return ["SKIP rank %d of %d cannot create a device context (%s)" % (failed[0][0], world, failed[0][1])]
        if failed[0][0] == 0:
            raise RuntimeError(failed[0][1])
        return []
    G = 2 * torch.cuda.get_device_properties(0).multi_processor_count
    lines = []
    for case in CASES:
        K, B, mode = case["K"], case["B"], case["mode"]
        shards = READS[case["reads"]](world, G)
        ctx.set_reads(*pack_reads(shards[rank]))
        windows = sum(max(0, len(r) - K + 1) for s in shards for r in s)
        cnt = DistributedKMerCounter(ctx, K, mode, result_on_host=True)
        st = cnt.Count(B, budget_bytes=PLANNER_RESERVE + case["budget"] * windows)
        t = ctx.times()
        idx = KMerIndexBuilder(ctx).BuildIndex(st)
        W = 8 * st.nw
        res = dict(keys=st.kmers(), counts=st.counts() if mode == CANON else None, bsz=st.bucket_sizes(), npass=cnt.npass,
                   checksum=st.checksum(), index=idx.serialize(), on_host=st.on_host(),
                   d2h_ok=t["result_d2h_bytes"] == st.total_kmers() * (W + 4 if mode == CANON else W))
        idx.free(); st.free()
        gathered = [None] * world
        dist.all_gather_object(gathered, res)
        if rank == 0:
            bad, ks = check_case(case, world, shards, gathered)
            if not all(g["on_host"] for g in gathered):
                bad.append("on_host")
            if not all(g["d2h_ok"] for g in gathered):
                bad.append("result_d2h_bytes")
            # the union counted by one GPU (a device set): the ranks' checksums add / xor up to its checksum
            ctx.set_reads(*pack_reads([r for s in shards for r in s]))
            one = KMerDiskCounter(ctx, _splitter(K, mode)).Count(B)
            want = one.checksum()
            one.free()
            m64 = (1 << 64) - 1
            cs = [g["checksum"] for g in gathered]
            tot = [sum(c[0] for c in cs), sum(c[1] for c in cs) & m64, 0, sum(c[3] for c in cs) & m64]
            for c in cs:
                tot[2] ^= c[2]
            if tot != want:
                bad.append("checksum_vs_single_gpu")
            line = "host-result dist case W=%d %-12s K=%-3d B=%-3d passes=%-2d distinct=%-7d %s" % (
                world, case["name"], K, B, gathered[0]["npass"], ks.n, "OK" if not bad else "FAIL " + ",".join(bad))
            print(line, flush=True)
            lines.append(line)
        dist.barrier()
    ctx.close()
    return lines


def _splitter(K, mode):
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, ParallelSortingSplitter
    return DeBruijnReadKMerSplitter(K) if mode == CANON else ParallelSortingSplitter(K)


def run_spawned(rank, world, port, out_path):
    """mp.spawn entry: W ranks on device 0 over gloo; rank 0 writes the result lines to out_path"""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world, timeout=timedelta(seconds=600))
    try:
        lines = run_cases(rank, world)
    finally:
        dist.destroy_process_group()
    if rank == 0:
        with open(out_path, "w") as f:
            f.write("\n".join(lines) + "\n")

