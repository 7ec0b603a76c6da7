"""Worker for tests/test_gpu_dist_graph.py: the unitigs and perfect loops of distributed sets, run by W processes.

Every case: the ranks' read shards go through the distributed (k+1)-mer count, the distributed k-mers, both indexes,
DistributedExtensionIndexBuilder.Build, DistributedGraphConstructor.ConstructGraph and assemble_graph. Rank 0 checks the GFA and
the unitigs against the single-GPU graph build over the union of the reads (early clippers off) and against the oracle; every rank
checks that its extension index's masks did not change. Run as dist_ext_worker: run_spawned (W processes on device 0, gloo) and
__main__ (torch.distributed.run, one GPU per rank, NCCL).
"""
import os
import sys
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dist_ext_worker import READS as EXT_READS  # noqa: E402
from dist_worker import ARENA_BYTES, _random_seq, _strided, _synth  # noqa: E402,F401


def _circles(world, case, seed):
    # error-free reads around circular sequences: each circle is a perfect loop whose k-mers lie in buckets of every owner
    rng = np.random.default_rng(seed)
    reads = []
    for n in (300, 451, 1200):
        c = _random_seq(rng, n)
        cc = c + c
        reads += [cc[i:i + 150] for i in range(0, n, 7)]
    return _strided(reads + _synth(500, seed), world)


def _long(world, case, seed):
    # one 6 000 bp sequence tiled by error-free reads: a unitig of several thousand k-mers through the buckets of every rank
    rng = np.random.default_rng(seed)
    g = _random_seq(rng, 6000)
    return _strided([g[i:i + 150] for i in range(0, len(g) - 150 + 1, 9)], world)


READS = dict(EXT_READS, circles=_circles, long=_long, many=lambda world, case, seed: _strided(_synth(48000, seed, genome=20000), world))

# k, B as in dist_ext_worker; loops: keep_perfect_loops; nocov: no (k+1)-mer index; host: both sets in host memory; batches: a
# junction-batch budget of one byte (4 096 junctions a batch) and at least that many batches on every rank
CASES = [
    dict(name="k21", k=21, B=16, reads="strided"),
    dict(name="k31", k=31, B=16, reads="blocks"),
    dict(name="k55", k=55, B=40, reads="blocks"),
    dict(name="k63", k=63, B=11, reads="strided"),
    dict(name="k95", k=95, B=9, reads="strided"),
    dict(name="k127", k=127, B=7, reads="strided"),
    dict(name="k55_B1", k=55, B=1, reads="strided"),
    dict(name="k55_B2", k=55, B=2, reads="blocks"),
    dict(name="k33_host", k=33, B=12, reads="strided", host=True),
    dict(name="k55_empty_short", k=55, B=16, reads="empty"),
    dict(name="k55_skew", k=55, B=8, reads="skew"),
    dict(name="k55_selfrc", k=55, B=7, reads="selfrc"),
    dict(name="k21_loops", k=21, B=10, reads="circles"),
    dict(name="k21_noloops", k=21, B=10, reads="circles", loops=False),
    dict(name="k55_long", k=55, B=24, reads="long"),
    dict(name="k31_nocov", k=31, B=16, reads="strided", nocov=True),
    dict(name="k21_batches", k=21, B=16, reads="many", batches=2),
]


def check_case(ctx, case, shards, gfa, unitigs):
    """rank 0: the assembled graph against the single-GPU graph build and the oracle over the union -> names of failed checks"""
    import oracle as O
    from spades_b200.graph import DeBruijnGraphConstructor
    from spades_b200.packing import pack_reads
    k, B, loops, cov = case["k"], case["B"], case.get("loops", True), not case.get("nocov")
    union = [r for s in shards for r in s]
    bad = []
    ctx.set_reads(*pack_reads(union))
    g = DeBruijnGraphConstructor(ctx, k, B).ConstructGraph(keep_perfect_loops=loops, with_coverage=cov)
    if gfa != g.gfa():
        bad.append("gfa_single_gpu")
    if unitigs != g.unitigs():
        bad.append("unitigs_single_gpu")
    g.free()
    if cov and gfa != O.full_graph(union, k, B, keep_loops=loops)["gfa"]:
        bad.append("gfa_oracle")
    return bad, len(unitigs)


def run_cases(rank, world, device, backend, cases):
    """every case over the default process group; the result lines on rank 0 (OK or the checks that failed), [] elsewhere"""
    import torch.distributed as dist
    from spades_b200.distributed import (DistributedExtensionIndexBuilder, DistributedGraphConstructor, DistributedKMerCounter,
                                         DistributedKmersFromKpomers, assemble_graph)
    from spades_b200.kmer_index import Context, KMerIndexBuilder
    from spades_b200.packing import pack_reads
    assert dist.get_backend() == backend, (dist.get_backend(), backend)
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    lines = []
    for ci, case in enumerate(cases):
        k, B, host = case["k"], case["B"], case.get("host", False)
        shards = READS[case["reads"]](world, case, 9000 + ci)
        ctx.set_reads(*pack_reads(shards[rank]))
        kp = DistributedKMerCounter(ctx, k + 1, result_on_host=host).Count(B)
        km = DistributedKmersFromKpomers(ctx, kp, result_on_host=host).Count(B)
        mkp = None if case.get("nocov") else KMerIndexBuilder(ctx).BuildIndex(kp)
        mk = KMerIndexBuilder(ctx).BuildIndex(km)
        ext = DistributedExtensionIndexBuilder(ctx, kp, mkp, km, mk).Build()
        before = ext.masks()
        dg = DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph(keep_perfect_loops=case.get("loops", True),
                                                                          budget_bytes=1 if case.get("batches") else None)
        ag = assemble_graph(dg)
        res = dict(masks_kept=bool(np.array_equal(before, ext.masks())), batches=dg.stats()[3], on_host=kp.on_host() and km.on_host(),
                   times=dg.times())
        gfa, unitigs = (ag.gfa(), ag.unitigs()) if ag is not None else (None, None)
        if ag is not None:
            ag.free()
        dg.free(); ext.free(); mk.free()
        if mkp is not None:
            mkp.free()
        km.free(); kp.free()
        gathered = [None] * world
        dist.all_gather_object(gathered, res)
        if rank == 0:
            bad, n = check_case(ctx, case, shards, gfa, unitigs)
            if not all(r["masks_kept"] for r in gathered):
                bad.append("masks_changed")
            if host and not all(r["on_host"] for r in gathered):
                bad.append("placement")
            if case.get("batches") and min(r["batches"] for r in gathered) < case["batches"]:
                bad.append("batches")
            line = "dist graph W=%d %-16s k=%-3d B=%-4d edges=%-6d batches=%-3d %s" % (
                world, case["name"], k, B, n, min(r["batches"] for r in gathered), "OK" if not bad else "FAIL " + ",".join(bad))
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
