"""Worker for tests/test_gpu_dist_edge_index.py: the EdgeIndex refill across ranks (DistributedEdgeIndex), run by W processes.

Every case: the ranks' read shards go through the distributed (k+1)-mer count, the distributed k-mers, both indexes,
DistributedExtensionIndexBuilder.Build, DistributedGraphConstructor.ConstructGraph and DistributedEdgeIndex. Rank 0 builds the
single-GPU graph and EdgeIndex over the union of the reads with the same options. Every rank checks that its serialized index is
byte-identical to one GPU's and that seq_idx gives one GPU's slots for a sample of the union's keys and some absent keys; rank 0
checks the assembled (edge id, offset) of every slot against one GPU's and, for small cases, against the oracle. Run as
dist_graph_worker: run_spawned (W processes on device 0, gloo) and __main__ (torch.distributed.run, one GPU per rank, NCCL).
"""
import hashlib
import os
import sys
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from dist_clip_worker import READS as CLIP_READS, _free, _sets  # noqa: E402
from dist_worker import ARENA_BYTES, PLANNER_RESERVE, _strided  # noqa: E402,F401
from make_golden import isolated_reads, pal_reads  # noqa: E402


def _synthetic(n, L, glen, err, seed):
    from spades_b200.packing import synthetic_reads
    return synthetic_reads(n, L, glen, err, seed=seed)


def _pal(world, case, seed):
    # palindromes of length K (self-RC windows on ordinary edges) and hairpins (self-conjugate edges)
    K = case.get("K") or case["k"] + 1
    return _strided(pal_reads(K // 2, 20, 10, seed, _synthetic(300, 150, 1500, 0.01, seed)), world)


def _repeats(world, case, seed):
    # one 400-bp repeat copied into three random contexts, the copies' reads on different ranks; with K = 7 most K-mers occur on
    # several edges of several ranks and end as tombstones
    rng = np.random.default_rng(seed)
    rep = "".join("ACGT"[i] for i in rng.integers(0, 4, 400))
    shards = [[] for _ in range(world)]
    for c in range(3):
        g = "".join("ACGT"[i] for i in rng.integers(0, 4, 600)) + rep + "".join("ACGT"[i] for i in rng.integers(0, 4, 600))
        shards[c % world] += [g[i:i + 150] for i in range(0, len(g) - 150 + 1, 5)]
    return shards


def _iso(n):
    # n isolated 70-bp edges spread over the ranks: 4 n vertices counting conjugates (the single-index boundary at B = 4 n)
    return lambda world, case, seed: _strided(isolated_reads(n, 7), world)


def _lone(world, case, seed):
    # every read on the last rank: the others own buckets but bring no edge
    shards = [[] for _ in range(world)]
    shards[-1] = _synthetic(400, 150, 1500, 0.01, seed)
    return shards


READS = dict(CLIP_READS, pal=_pal, repeats=_repeats, iso4=_iso(4), iso5=_iso(5), lone=_lone,
             small=lambda world, case, seed: _strided(_synthetic(150, 100, 1500, 0.01, seed), world))

# k, B: the graph's; K: the index's (None = k + 1); eB: num_buckets of the index (chunks for K = k + 1); oracle: also against
# tests/oracle.py (python loops: small cases); tc / at: the clippers as in dist_clip_worker; budget: a count pass budget in bytes
# (the planner's reserve plus a few bytes: passes of one or two buckets)
CASES = [
    dict(name="k21", k=21, B=16, reads="strided", eB=20),
    dict(name="k31", k=31, B=16, reads="blocks", eB=20),
    dict(name="k55", k=55, B=40, reads="blocks", eB=80),
    dict(name="k63", k=63, B=11, reads="strided", eB=20),
    dict(name="k95", k=95, B=9, reads="strided", eB=20),
    dict(name="k127", k=127, B=7, reads="strided", eB=20),
    dict(name="K1_small", k=21, B=8, reads="small", K=1, eB=20, oracle=True),
    dict(name="K2_small", k=21, B=8, reads="small", K=2, eB=20, oracle=True),
    dict(name="K15", k=21, B=16, reads="strided", K=15, eB=20),
    dict(name="K33", k=55, B=16, reads="strided", K=33, eB=40),
    dict(name="K66_pal", k=77, B=12, reads="pal", K=66, eB=20),
    dict(name="K97", k=99, B=9, reads="strided", K=97, eB=7),
    dict(name="single_iso4", k=21, B=4, reads="iso4", eB=16, oracle=True),
    dict(name="multi_iso4", k=21, B=4, reads="iso4", eB=17, oracle=True),
    dict(name="single_iso5", k=21, B=4, reads="iso5", eB=20, oracle=True),
    dict(name="pal_k21", k=21, B=8, reads="pal", eB=20, oracle=True),
    dict(name="repeats_K7", k=21, B=8, reads="repeats", K=7, eB=20, oracle=True),
    dict(name="loops_k21", k=21, B=10, reads="circles", eB=20),
    dict(name="selfrc_k55", k=55, B=7, reads="selfrc", eB=20),
    dict(name="lone_rank", k=21, B=8, reads="lone", eB=20),
    dict(name="no_edges", k=55, B=16, reads="empty", eB=20),
    dict(name="clippers_k21", k=21, B=8, reads="at21", eB=20, tc=100 - 21, at=(0.8, 10, 200)),
    dict(name="budget_K15", k=21, B=16, reads="many", K=15, eB=64, budget=PLANNER_RESERVE + (1 << 16)),
]


def _opts(case):
    at = case.get("at")
    ratio, mn, mx = at if at else (0.8, 10, 200)
    return dict(keep_perfect_loops=True, early_tip_clipper_length=case.get("tc", 0), early_at_clipper=at is not None,
                at_ratio=ratio, at_min_length=mn, at_max_length=mx)


def _index_args(case):
    K = case.get("K")
    return (None, case["eB"]) if K is None or K == case["k"] + 1 else (K, case["eB"])


def single_gpu(ctx, case, union):
    """rank 0: the single-GPU graph and EdgeIndex over the union -> (serialized bytes, ids, offsets, unitigs, key sample, slots)"""
    from spades_b200.graph import DeBruijnGraphConstructor, EdgeIndex
    from spades_b200.packing import pack_reads, revcomp
    ctx.set_reads(*pack_reads(union))
    g = DeBruijnGraphConstructor(ctx, case["k"], case["B"]).ConstructGraph(**_opts(case))
    k, B = _index_args(case)
    ei = EdgeIndex(g, k, B)
    K = ei.K
    unitigs = g.unitigs()
    ids, offs = ei.values()
    # a sample of the union's keys (stored, minimal form) and random K-mers, most of them absent
    rng = np.random.default_rng(11)
    kms = []
    for s in unitigs:
        if len(s) >= K:
            for j in rng.integers(0, len(s) - K + 1, 3):
                x = s[j:j + K]
                kms.append(min(x, revcomp(x)))
    kms = kms[:3000] + ["".join("ACGT"[i] for i in rng.integers(0, 4, K)) for _ in range(200)]
    kms = [min(x, revcomp(x)) for x in kms]
    keys = np.zeros((len(kms), ei.nw), np.uint64)
    for i, x in enumerate(kms):
        w, _, _ = pack_reads([x])
        keys[i] = w[:ei.nw]
    slots = ei.seq_idx(keys) if len(keys) else np.zeros(0, np.uint64)
    ser = ei.serialize()
    ei.free(); g.free()
    return ser, ids, offs, unitigs, keys, slots


def distributed(ctx, case, shard, keys_of):
    """this rank's distributed chain of one case: (serialized sha256, slots of the key sample keys_of(K), assembled values on rank 0)"""
    from spades_b200.distributed import DistributedEdgeIndex, DistributedGraphConstructor, assemble_edge_index_values
    objs = _sets(ctx, case, shard)
    kp, km, mkp, mk, ext = objs
    dg = DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph(**_opts(case))
    k, B = _index_args(case)
    dei = DistributedEdgeIndex(dg, k, B, budget_bytes=case.get("budget"))
    dg.free()
    _free(objs)
    ser = dei.serialize()
    keys = keys_of(dei.K)
    slots = dei.seq_idx(keys) if len(keys) else np.zeros(0, np.uint64)
    vals = assemble_edge_index_values(dei)
    res = dict(sha=hashlib.sha256(ser).hexdigest(), slots=slots, npass=dei.npass, levels=dei.levels, slice=dei.slot_range(), size=dei.size())
    dei.free()
    return res, vals


def _check(case, world, single, gathered, vals):
    """rank 0 -> names of failed checks"""
    import oracle as O
    ser, ids, offs, unitigs, _, slots = single
    bad = []
    sha = hashlib.sha256(ser).hexdigest()
    if any(r["sha"] != sha for r in gathered):
        bad.append("serialize")
    if any(not np.array_equal(r["slots"], slots) for r in gathered):
        bad.append("seq_idx")
    if vals is None or not np.array_equal(vals[0], ids) or not np.array_equal(vals[1], offs):
        bad.append("values_single_gpu")
    if case.get("oracle"):
        K = case.get("K") or case["k"] + 1
        _, _, oids, ooffs = O.edge_index(unitigs, case["k"], K, 1 if K == case["k"] + 1 else case["eB"])
        if not np.array_equal(oids, ids) or not np.array_equal(ooffs, offs):
            bad.append("values_oracle")
    if case.get("budget") and min(r["npass"] for r in gathered) < 2:
        bad.append("one_count_pass")
    n = len(ids)
    if [tuple(r["slice"]) for r in gathered] != [(n * r // world, n * (r + 1) // world) for r in range(world)]:
        bad.append("slot_ranges")
    if case["name"] == "repeats_K7" and not (ids == (1 << 64) - 2).any():
        bad.append("no_tombstone")
    return bad


def run_case(ctx, rank, world, case, shards):
    import torch.distributed as dist
    single = single_gpu(ctx, case, [r for s in shards for r in s]) if rank == 0 else None
    obj = [single[4] if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    res, vals = distributed(ctx, case, shards[rank], lambda K: obj[0])
    gathered = [None] * world
    dist.all_gather_object(gathered, res)
    if rank != 0:
        return None
    bad = _check(case, world, single, gathered, vals)
    return "dist edge index W=%d %-14s k=%-3d K=%-3d slots=%-7d levels=%-2d passes=%-2d %s" % (
        world, case["name"], case["k"], case.get("K") or case["k"] + 1, len(single[1]), gathered[0]["levels"],
        min(r["npass"] for r in gathered), "OK" if not bad else "FAIL " + ",".join(bad))


def run_cases(rank, world, device, backend, cases):
    """every case over the default process group; the result lines on rank 0 (OK or the checks that failed), [] elsewhere"""
    import torch.distributed as dist
    from spades_b200.kmer_index import Context
    assert dist.get_backend() == backend, (dist.get_backend(), backend)
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    lines = []
    for ci, case in enumerate(cases):
        shards = READS[case["reads"]](world, case, 9200 + ci)
        line = run_case(ctx, rank, world, case, shards)
        if line:
            print(line, flush=True)
            lines.append(line)
        dist.barrier()
    ctx.close()
    return lines


def run_fixtures(rank, world, device, names):
    """every reference fixture (*_eigraph) through the distributed path, checked with golden_util.check_edge_index"""
    import torch.distributed as dist
    import golden_util as G
    from spades_b200.distributed import DistributedEdgeIndex, DistributedGraphConstructor, assemble_edge_index_values
    from spades_b200.kmer_index import Context
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    lines = []
    for name in names:
        g = G.load(name)
        k, B, K = g["k"], g["B"], int(g["ei_k"][0])
        objs = _sets(ctx, dict(k=k, B=B), _strided(g["reads"], world)[rank])
        kp, km, mkp, mk, ext = objs
        dg = DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph()
        dei = DistributedEdgeIndex(dg, None if K == k + 1 else K, int(g["ei_chunks"][0]) if K == k + 1 else B)
        dg.free()
        _free(objs)
        ser = dei.serialize()
        vals = assemble_edge_index_values(dei)
        shas = [None] * world
        dist.all_gather_object(shas, hashlib.sha256(ser).hexdigest())
        dei.free()
        if rank == 0:
            bad = G.check_edge_index(g, ser, vals[0], vals[1], 1 if K == k + 1 else B)
            if len(set(shas)) != 1:
                bad.append("serialize_differs_across_ranks")
            line = "dist edge index fixture W=%d %-26s %s" % (world, name, "OK" if not bad else "FAIL " + ",".join(bad))
            print(line, flush=True)
            lines.append(line)
        dist.barrier()
    ctx.close()
    return lines


def run_refusals(rank, world, device):
    """arguments that differ between the ranks -> ValueError on every rank; then a run on the same context that matches one GPU"""
    import torch.distributed as dist
    from spades_b200.distributed import DistributedEdgeIndex, DistributedGraphConstructor
    from spades_b200.kmer_index import Context
    ctx = Context(device, hbm_budget_bytes=ARENA_BYTES)
    bad = []
    case = dict(name="refusals", k=21, B=8, reads="small", eB=20, oracle=True)
    shards = READS["small"](world, case, 3)
    objs = _sets(ctx, case, shards[rank])
    kp, km, mkp, mk, ext = objs
    dg = DistributedGraphConstructor(ctx, ext, mkp, mk).ConstructGraph()
    for args in ((None, 20 + rank), (15 + rank, 20)):
        try:
            DistributedEdgeIndex(dg, *args).free()
            if world > 1:
                bad.append("differing %s accepted" % (args,))
        except ValueError:
            if world == 1:
                bad.append("ValueError at W=1")
        dist.barrier()
    dg.free()
    _free(objs)
    line = run_case(ctx, rank, world, case, shards)
    gathered = [None] * world
    dist.all_gather_object(gathered, bad)
    ctx.close()
    if rank != 0:
        return []
    allbad = sorted(set(b for bb in gathered for b in bb))
    if not line.endswith(" OK"):
        allbad.append(line)
    out = "dist edge index refusals W=%d %s" % (world, "OK" if not allbad else "FAIL " + "; ".join(allbad))
    print(out, flush=True)
    return [out]


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
