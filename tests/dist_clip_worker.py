"""Worker for tests/test_gpu_dist_clippers.py: the early tip and A/T clippers of distributed sets, run by W processes.

Every case: the ranks' read shards go through the distributed (k+1)-mer count, the distributed k-mers, both indexes,
DistributedExtensionIndexBuilder.Build, DistributedGraphConstructor.ConstructGraph with the clippers on, assemble_masks and
assemble_graph. Rank 0 checks the union's clipper statistics, the clipped masks, the unitigs and the GFA against the single-GPU
graph build over the union of the reads with the same options and against the oracle; every rank checks that its extension index's
masks did not change. Run as dist_graph_worker: run_spawned (W processes on device 0, gloo) and __main__ (torch.distributed.run,
one GPU per rank, NCCL).
"""
import ctypes as C
import os
import sys
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from dist_graph_worker import READS as GRAPH_READS  # noqa: E402
from dist_worker import ARENA_BYTES, _strided  # noqa: E402,F401
from make_golden import at_arm_reads, at_reads, loops_reads  # noqa: E402

BIG = 2 ** 32 + 3


def _synthetic(n, L, glen, err, seed):
    from spades_b200.packing import synthetic_reads
    return synthetic_reads(n, L, glen, err, seed=seed)


# the shapes of test_gpu_graph_options.py: TC_READS (L, n, glen, err, seed) and AT_READS plus the 350-vertex A-rich arm
def _tc(L, n, glen, err, seed):
    return lambda world, case, s: _strided(_synthetic(n, L, glen, err, seed), world)


def _at(L, n, glen, err, seed):
    return lambda world, case, s: _strided(at_reads(n, L, glen, err, seed) + at_arm_reads(350, L, seed), world)


def _loops_at(world, case, seed):
    return _strided(loops_reads(250, 250) + _synthetic(600, 150, 1500, 0.01, 104) + at_reads(1500, 150, 2000, 0.01, 105), world)


READS = dict(GRAPH_READS, tc21=_tc(100, 3000, 2500, 0.02, 81), tc77=_tc(150, 1500, 2500, 0.01, 82), tc127=_tc(250, 800, 3000, 0.005, 83),
             at21=_at(100, 2000, 2000, 0.01, 91), at97=_at(250, 150, 1000, 0.002, 92), loops_at=_loops_at)

# tc: the tip clipper's length bound (0 = off); at: the A/T clipper with at_params (ratio, min_length, max_length); loops, nocov,
# host, batches as in dist_graph_worker. Every case makes the oracle's clippers remove something.
CASES = [
    dict(name="tc_k21", k=21, B=8, reads="tc21", tc=100 - 21),
    dict(name="tc_k77", k=77, B=5, reads="tc77", tc=150 - 77),
    dict(name="tc_k127", k=127, B=6, reads="tc127", tc=250 - 127),
    dict(name="tc_k21_bound1", k=21, B=8, reads="tc21", tc=1),
    dict(name="tc_k21_bound_big", k=21, B=8, reads="tc21", tc=BIG),
    dict(name="at_tc_k21", k=21, B=8, reads="at21", tc=100 - 21, at=(0.8, 10, 200)),
    dict(name="at_tc_k97", k=97, B=6, reads="at97", tc=250 - 97, at=(0.8, 10, 200)),
    dict(name="at_k97_max1e6", k=97, B=6, reads="at97", tc=250 - 97, at=(0.8, 10, 10 ** 6)),
    dict(name="both_noloops_k55", k=55, B=7, reads="loops_at", tc=150 - 55, at=(0.8, 10, 200), loops=False),
    dict(name="tc_k21_B1", k=21, B=1, reads="tc21", tc=100 - 21),
    dict(name="at_tc_k21_B2", k=21, B=2, reads="at21", tc=100 - 21, at=(0.8, 10, 200)),
    dict(name="tc_k55_empty_short", k=55, B=16, reads="empty", tc=150 - 55),
    dict(name="at_tc_k33_host", k=33, B=12, reads="at21", tc=100 - 33, at=(0.8, 10, 200), host=True),
    dict(name="tc_k31_nocov", k=31, B=16, reads="strided", tc=150 - 31, nocov=True),
    dict(name="tc_k21_batches", k=21, B=16, reads="many", tc=150 - 21, batches=2),
]


def _opts(case):
    at = case.get("at")
    ratio, mn, mx = at if at else (0.8, 10, 200)
    return dict(keep_perfect_loops=case.get("loops", True), early_tip_clipper_length=case.get("tc", 0), early_at_clipper=at is not None,
                at_ratio=ratio, at_min_length=mn, at_max_length=mx)


def _sets(ctx, case, shard):
    """this rank's sets, indexes and extension index of one case"""
    from spades_b200.distributed import DistributedExtensionIndexBuilder, DistributedKMerCounter, DistributedKmersFromKpomers
    from spades_b200.kmer_index import KMerIndexBuilder
    from spades_b200.packing import pack_reads
    k, B, host = case["k"], case["B"], case.get("host", False)
    ctx.set_reads(*pack_reads(shard))
    kp = DistributedKMerCounter(ctx, k + 1, result_on_host=host).Count(B)
    km = DistributedKmersFromKpomers(ctx, kp, result_on_host=host).Count(B)
    mkp = None if case.get("nocov") else KMerIndexBuilder(ctx).BuildIndex(kp)
    mk = KMerIndexBuilder(ctx).BuildIndex(km)
    ext = DistributedExtensionIndexBuilder(ctx, kp, mkp, km, mk).Build()
    return [kp, km, mkp, mk, ext]


def _free(objs):
    for o in reversed(objs):
        if o is not None:
            o.free()


def distributed(ctx, case, shard):
    """the whole distributed chain of one case on this rank: (result dict for every rank, (masks, unitigs, gfa) on rank 0)"""
    from spades_b200.distributed import DistributedGraphConstructor, assemble_graph, assemble_masks
    objs = _sets(ctx, case, shard)
    kp, km, mkp, mk, ext = objs
    before = ext.masks()
    dg = DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph(budget_bytes=1 if case.get("batches") else None, **_opts(case))
    masks = assemble_masks(dg)
    ag = assemble_graph(dg)
    res = dict(masks_kept=bool(np.array_equal(before, ext.masks())), batches=dg.stats()[3], on_host=kp.on_host() and km.on_host(),
               remote=dg.remote_clipper_stores(), owners=len(set(int(o) for o in dg.owners)), times=dg.clipper_times())
    art = None
    if ag is not None:
        art = dict(masks=masks, unitigs=ag.unitigs(), gfa=ag.gfa(), tc=dg.tip_clipper_stats(), at=dg.at_clipper_stats())
        ag.free()
    dg.free()
    _free(objs)
    return res, art


def check_case(ctx, case, shards, art):
    """rank 0: the assembled artefacts against the single-GPU build and the oracle over the union -> names of failed checks"""
    import oracle as O
    from spades_b200.graph import DeBruijnGraphConstructor
    from spades_b200.packing import pack_reads
    k, B, cov = case["k"], case["B"], not case.get("nocov")
    opts = _opts(case)
    union = [r for s in shards for r in s]
    bad = []
    ctx.set_reads(*pack_reads(union))
    g = DeBruijnGraphConstructor(ctx, k, B).ConstructGraph(with_coverage=cov, **opts)
    single = dict(masks=g.masks(), unitigs=g.unitigs(), gfa=g.gfa(), tc=g.tip_clipper_stats(), at=g.at_clipper_stats())
    g.free()
    r = O.full_graph(union, k, B, early_tc=opts["early_tip_clipper_length"], early_at=opts["early_at_clipper"], keep_loops=opts["keep_perfect_loops"],
                     at_params=(opts["at_ratio"], opts["at_min_length"], opts["at_max_length"]))
    oracle = dict(masks=r["masks"], unitigs=r["unitigs"].seqs, gfa=r["gfa"],
                  tc=(r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"]) if r["tc"] else (0, 0, 0), at=r["at"] if r["at"] else [0, 0, 0, 0])
    for name in ("tc", "at", "masks", "unitigs", "gfa"):
        eq = (lambda a, b: np.array_equal(a, b)) if name == "masks" else (lambda a, b: list(a) == list(b) if name != "gfa" else a == b)
        if not eq(art[name], single[name]):
            bad.append(name + "_single_gpu")
        if (cov or name != "gfa") and not eq(art[name], oracle[name]):
            bad.append(name + "_oracle")
    if case.get("tc") and oracle["tc"][0] == 0:
        bad.append("oracle_tc_removes_nothing")
    if case.get("at") and oracle["at"][1] + oracle["at"][2] == 0:
        bad.append("oracle_at_removes_nothing")
    return bad, len(art["unitigs"]), oracle["tc"][0], oracle["at"][1] + oracle["at"][2]


def run_cases(rank, world, device, backend, cases):
    """every case over the default process group; the result lines on rank 0 (OK or the checks that failed), [] elsewhere"""
    import torch.distributed as dist
    from spades_b200.kmer_index import Context
    assert dist.get_backend() == backend, (dist.get_backend(), backend)
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    lines = []
    for ci, case in enumerate(cases):
        shards = READS[case["reads"]](world, case, 9100 + ci)
        res, art = distributed(ctx, case, shards[rank])
        gathered = [None] * world
        dist.all_gather_object(gathered, res)
        if rank == 0:
            bad, n, tc_removed, at_removed = check_case(ctx, case, shards, art)
            if not all(r["masks_kept"] for r in gathered):
                bad.append("masks_changed")
            if case.get("host") and not all(r["on_host"] for r in gathered):
                bad.append("placement")
            if case.get("batches") and min(r["batches"] for r in gathered) < case["batches"]:
                bad.append("batches")
            remote = {key: sum(r["remote"][key] for r in gathered) for key in ("marks", "roots", "clears")}
            if world > 1 and gathered[0]["owners"] > 1:
                if remote["marks"] == 0:
                    bad.append("no_cross_owner_marks")
                if case.get("at") and (remote["roots"] == 0 or remote["clears"] == 0):
                    bad.append("no_cross_owner_roots_or_clears")
            line = "dist clip W=%d %-20s k=%-3d B=%-3d edges=%-6d tc_removed=%-6d at_links_kmers=%-6d remote=%d/%d/%d %s" % (
                world, case["name"], case["k"], case["B"], n, tc_removed, at_removed, remote["marks"], remote["roots"], remote["clears"],
                "OK" if not bad else "FAIL " + ",".join(bad))
            print(line, flush=True)
            lines.append(line)
        dist.barrier()
    ctx.close()
    return lines


def run_fixtures(rank, world, device, names):
    """every reference fixture (*_tcgraph, *_atgraph) through the distributed path, checked with golden_util.check_graph"""
    import torch.distributed as dist
    import golden_util as G
    from spades_b200.kmer_index import Context
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    lines = []
    for name in names:
        g = G.load(name)
        case = dict(k=g["k"], B=g["B"], tc=g.get("tc_bound", 0), at=(0.8, 10, 200) if name.endswith("_atgraph") else None)
        _, art = distributed(ctx, case, _strided(g["reads"], world)[rank])
        if rank == 0:
            want = dict(masks=art["masks"], unitigs=art["unitigs"], gfa=art["gfa"])
            if case["tc"]:
                want["tc_removed"] = art["tc"][0]
            if case["at"]:
                want["at_removed"] = [art["at"][0], art["at"][2]]
            bad = G.check_graph(g, want)
            line = "dist clip fixture W=%d %-24s %s" % (world, name, "OK" if not bad else "FAIL " + ",".join(bad))
            print(line, flush=True)
            lines.append(line)
        dist.barrier()
    ctx.close()
    return lines


def _expect(ok, what, bad):
    if not ok:
        bad.append(what)


def run_refusals(rank, world, device):
    """refusals on every rank, each followed by a use of the same context: bad A/T parameters, options that differ between the
    ranks, phase entries out of order. One result line on rank 0."""
    import torch.distributed as dist
    from spades_b200 import _lib
    from spades_b200.distributed import SGPU_DIST_GRAPH_IPC_BYTES, DistributedGraphConstructor, _check_owned_once, _open_peers, _ownership
    from spades_b200.kmer_index import Context, SpadesGpuError, _p
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    L = ctx.L
    bad = []
    case = dict(name="refusals", k=21, B=8, reads="at21", tc=79, at=(0.8, 10, 200))
    shards = READS["at21"](world, case, 0)
    objs = _sets(ctx, case, shards[rank])
    kp, km, mkp, mk, ext = objs
    con = DistributedGraphConstructor(ctx, ext, mkp, mk)
    # bad A/T parameters: min_length > k, ratio outside (0, 1], max_length 0 -> SGPU_EINVAL on every rank
    for params in ((0.8, 22, 200), (0.0, 10, 200), (1.0000001, 10, 200), (0.8, 10, 0)):
        try:
            con.ConstructGraph(early_at_clipper=True, early_tip_clipper_length=79, at_ratio=params[0], at_min_length=params[1], at_max_length=params[2])
            bad.append("accepted %s" % (params,))
        except SpadesGpuError as e:
            _expect(str(e).startswith("[2] "), "code %s" % e, bad)
        dist.barrier()
    # options that differ between the ranks -> ValueError on every rank, before any phase
    try:
        con.ConstructGraph(early_tip_clipper_length=79 + rank)
        _expect(world == 1, "differing options accepted", bad)
    except ValueError:
        _expect(world > 1, "ValueError at W=1", bad)
    dist.barrier()
    # phase entries out of order, on a handle with both clippers on (begin_opts as ConstructGraph calls it)
    bsz_all, owned_all = _ownership(km, None)
    _check_owned_once(bsz_all, owned_all)
    owners = np.ascontiguousarray(owned_all.argmax(axis=0), np.int32)
    _, powned = _ownership(kp, None)
    powners = np.ascontiguousarray(powned.argmax(axis=0), np.int32)
    ubsz = np.ascontiguousarray(bsz_all.sum(axis=0), np.uint64)
    opts = _lib.SgpuGraphOptions(1, 79, 1, 0.8, 10, 200)
    h = C.c_void_p()
    ctx.check(L.sgpu_dist_graph_begin_opts(ctx.h, ext.h, _p(owners), _p(powners), _p(ubsz), 0, C.byref(opts), C.byref(h)))
    n = km.total_kmers()
    out = np.zeros(max(n, 1), np.uint8)
    at, tc, rm = np.zeros(4, np.uint64), np.zeros(3, np.uint64), np.zeros(3, np.uint64)
    _expect(L.sgpu_dist_graph_at_edges_probe(h) == 2, "probe before open_peers", bad)
    _open_peers(ctx, None, lambda o: L.sgpu_dist_graph_ipc_handle(h, o), lambda d: L.sgpu_dist_graph_open_peers(h, d), SGPU_DIST_GRAPH_IPC_BYTES)

    def step(name, want):
        rc = getattr(L, "sgpu_dist_graph_" + name)(h)
        _expect(rc == want, "%s returned %d, not %d" % (name, rc, want), bad)
        if rc == 0:
            dist.barrier()
    for name in ("unitigs", "isolate", "unlink", "tip_probe", "junctions", "at_edges_apply"):
        step(name, 2)
    _expect(L.sgpu_dist_graph_masks(h, _p(out), n) == 2, "masks before the clippers", bad)
    step("at_edges_probe", 0)
    step("at_edges_probe", 2)
    step("unlink", 2)
    for name in ("at_edges_apply", "at_tips_probe", "isolate"):
        step(name, 0)
    step("isolate", 2)
    step("unlink", 0)
    step("at_edges_probe", 2)
    step("tip_probe", 0)
    step("unlink", 2)
    step("isolate", 0)
    step("unlink", 0)
    step("unitigs", 2)
    step("junctions", 0)
    for name in ("at_edges_probe", "tip_probe", "isolate", "unlink", "junctions"):
        step(name, 2)
    _expect(L.sgpu_dist_graph_masks(h, _p(out), n) == 0, "masks after the junctions", bad)
    _expect(L.sgpu_dist_graph_clipper_stats(h, _p(at), _p(tc), _p(rm)) == 0, "clipper stats", bad)
    step("unitigs", 0)
    for name in ("at_edges_probe", "tip_probe", "junctions"):
        step(name, 2)
    L.sgpu_dist_graph_free(h)
    # the clippers off: no clipper phase, and the junctions are listed by begin
    h = C.c_void_p()
    ctx.check(L.sgpu_dist_graph_begin(ctx.h, ext.h, _p(owners), _p(powners), _p(ubsz), 0, C.byref(h)))
    _open_peers(ctx, None, lambda o: L.sgpu_dist_graph_ipc_handle(h, o), lambda d: L.sgpu_dist_graph_open_peers(h, d), SGPU_DIST_GRAPH_IPC_BYTES)
    for name in ("at_edges_probe", "tip_probe", "isolate", "unlink", "junctions"):
        step(name, 2)
    _expect(L.sgpu_dist_graph_masks(h, _p(out), n) == 0 and np.array_equal(out[:n], ext.masks()), "unclipped masks", bad)
    L.sgpu_dist_graph_free(h)
    dist.barrier()
    _free(objs)
    # the context is still usable: a whole case runs and matches
    res, art = distributed(ctx, case, shards[rank])
    if rank == 0:
        more, _, _, _ = check_case(ctx, case, shards, art)
        bad += more
    gathered = [None] * world
    dist.all_gather_object(gathered, bad)
    ctx.close()
    if rank != 0:
        return []
    allbad = sorted(set(b for bb in gathered for b in bb))
    line = "dist clip refusals W=%d %s" % (world, "OK" if not allbad else "FAIL " + "; ".join(allbad))
    print(line, flush=True)
    return [line]


def run_spawned(rank, world, port, out_path, what):
    """mp.spawn entry: W ranks on device 0 over gloo; `what` is "cases", "refusals" or a list of fixture names; rank 0 writes the
    result lines to out_path"""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world, timeout=timedelta(seconds=600))
    try:
        if what == "cases":
            lines = run_cases(rank, world, 0, "gloo", CASES)
        elif what == "refusals":
            lines = run_refusals(rank, world, 0)
        else:
            lines = run_fixtures(rank, world, 0, what)
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
