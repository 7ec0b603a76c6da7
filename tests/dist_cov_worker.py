"""Worker for the distributed coverage pre-filter tests (launched by mp.spawn): W processes on ONE device joined by a gloo group,
each with its own context and arena. For every case of CASES each rank filters its shard with spades_b200.distributed.
distributed_cov_filter; rank 0 checks the ranks' results against sgpu_reads_cov_filter over the union (shards concatenated in
rank order) in its own context and against the oracle, and writes one line per case."""
import os
import re
import sys
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ARENA_BYTES = 1 << 30              # explicit per-rank device arena: W ranks share one device


def _random_seq(rng, n):
    return "".join("ACGT"[c] for c in rng.integers(0, 4, n))


def _union(K, seed):
    """reads at several coverages (some pass the filter, some do not), ragged and short reads, palindromes whose centred window
    of an even K is its own reverse complement, and low-complexity reads"""
    from spades_b200.packing import revcomp, synthetic_reads
    rng = np.random.default_rng(seed)
    reads = synthetic_reads(1500, 120, 3000, 0.01, seed=seed) + synthetic_reads(400, 100, 40000, 0.02, seed=seed + 100)
    for _ in range(6):
        x = _random_seq(rng, 60)
        reads += [x + revcomp(x)] * 3
    reads += ["A" * 150, "T" * 97, "AC" * 40]
    reads = [r[: int(rng.integers(K - 2, len(r) + 1))] if rng.random() < 0.2 and len(r) > K else r for r in reads]
    return [reads[i] for i in rng.permutation(len(reads))]


def _short(K, seed, n=150):
    rng = np.random.default_rng(seed)
    return [_random_seq(rng, int(m)) for m in rng.integers(1, K, n)]


# shard layouts: a read set -> the shards of all ranks (every rank builds the same list and takes its own)
def strided(reads, world):
    return [reads[r::world] for r in range(world)]


def blocked(reads, world):
    n = len(reads)
    return [reads[n * r // world: n * (r + 1) // world] for r in range(world)]


def skewed(reads, world):
    # rank 0 holds 70 % of the reads, the others share the rest
    if world == 1:
        return [reads]
    cut = len(reads) * 7 // 10
    return [reads[:cut]] + blocked(reads[cut:], world - 1)


def empty_short(reads, world, short):
    # the last rank holds no reads, the one before only reads shorter than K
    if world == 1:
        return [reads + short]
    if world == 2:
        return [reads + short, []]
    return blocked(reads, world - 2) + [short, []]


def owner_skew(world, K=32):
    """one window per read, all distinct; with two or more ranks about 90 % of a slice's capacity is owned by rank 0 (more than the
    even share x 1.5, so the load reaches into the headroom). The reads are spread over the ranks strided, so most inserts are remote."""
    import oracle as O
    from spades_b200.distributed import cov_layout_host
    from spades_b200.packing import pack_reads
    total = 3000                                   # bound ~3 300: key bits 21 (2^11 < bound < 2^12), fixed whatever the split
    _, cap = cov_layout_host(world, int(total * 1.1), np.zeros(0, np.uint64))
    want0 = min(total, int(cap * 0.9))
    rng = np.random.default_rng(4242)
    cand = [_random_seq(rng, K) for _ in range(5 * total)]
    words, offs, _ = pack_reads(cand)
    keys = np.array([O.cyclic_hash(words[int(o):], 0, K) for o in offs], np.uint64) & np.uint64((1 << 21) - 1)
    owners, _ = cov_layout_host(world, 0, keys)
    zero, rest, seen = [], [], set()
    for r, k, o in zip(cand, keys.tolist(), owners.tolist()):
        if k in seen:
            continue
        if o == 0 and len(zero) < want0:
            zero.append(r); seen.add(k)
        elif o != 0 and len(rest) < total - want0:
            rest.append(r); seen.add(k)
    reads = zero + rest
    reads = [reads[i] for i in rng.permutation(len(reads))]
    return strided(reads, world), len(zero)


CASES = [
    # k+1 x threshold, each over one shard layout
    dict(name="k12_t1_strided", K=12, thr=1, layout="strided"),
    dict(name="k12_t2_blocked", K=12, thr=2, layout="blocked"),
    dict(name="k12_t5_skewed", K=12, thr=5, layout="skewed"),
    dict(name="k22_t1_blocked", K=22, thr=1, layout="blocked"),
    dict(name="k22_t2_empty", K=22, thr=2, layout="empty"),
    dict(name="k22_t5_strided", K=22, thr=5, layout="strided", apply=False),
    dict(name="k32_t1_skewed", K=32, thr=1, layout="skewed"),
    dict(name="k32_t2_strided", K=32, thr=2, layout="strided", count_B=16),
    dict(name="k32_t5_empty", K=32, thr=5, layout="empty"),
    dict(name="k56_t1_empty", K=56, thr=1, layout="empty"),
    dict(name="k56_t2_skewed", K=56, thr=2, layout="skewed", count_B=7),
    dict(name="k56_t5_blocked", K=56, thr=5, layout="blocked", apply=False),
    dict(name="k70_t1_strided", K=70, thr=1, layout="strided"),
    dict(name="k70_t2_blocked", K=70, thr=2, layout="blocked", count_B=9),
    dict(name="k70_t5_skewed", K=70, thr=5, layout="skewed"),
    # the unmodified reference's CoverageFilter phase (tests/golden/cov_*_covfilter.npz), split into shards
    dict(name="cov_k20_t3", golden="cov_k20_t3_covfilter", layout="blocked"),
    dict(name="cov_k21_t2", golden="cov_k21_t2_covfilter", layout="strided", count_B=12),
    dict(name="cov_k31_t5", golden="cov_k31_t5_covfilter", layout="skewed"),
    dict(name="cov_k55_t2", golden="cov_k55_t2_covfilter", layout="empty"),
    # rank 0 owns ~90 % of a slice's capacity
    dict(name="owner_skew", K=32, thr=1, layout="owner_skew"),
]


def case_shards(case, world):
    """-> (K, threshold, shards, extra checks)"""
    import golden_util as G
    extra = {}
    if case.get("golden"):
        g = G.load(case["golden"])
        K, thr, reads = g["k"] + 1, int(g["thr"][0]), g["reads"]
        extra = dict(card=int(g["card"][0]), key_bits=int(g["key_bits"][0]), keep=g["keep"])
    else:
        K, thr = case["K"], case["thr"]
        reads = None if case["layout"] == "owner_skew" else _union(K, 1000 + K * 10 + thr)
    lay = case["layout"]
    if lay == "owner_skew":
        shards, extra["owned0"] = owner_skew(world, K)
    elif lay == "empty":
        shards = empty_short(reads, world, _short(K, K))
    else:
        shards = {"strided": strided, "blocked": blocked, "skewed": skewed}[lay](reads, world)
    if extra.get("keep") is not None:
        # the fixture's verdicts follow its read order; the union is the shards in rank order
        pos = {"strided": lambda: np.concatenate([np.arange(len(reads))[r::world] for r in range(world)]),
               "blocked": lambda: np.arange(len(reads)), "skewed": lambda: np.arange(len(reads))}
        if lay == "empty":
            extra["keep"] = np.concatenate([extra["keep"], np.zeros(sum(len(s) for s in shards) - len(reads), np.uint8)])
        else:
            extra["keep"] = extra["keep"][pos[lay]()]
    return K, thr, shards, extra


def check_case(case, world, K, thr, shards, extra, gathered, single):
    import oracle as O
    from spades_b200.packing import pack_reads
    union = [r for s in shards for r in s]
    want_keep, want = O.cov_filter(*pack_reads(union), K, thr)
    bad = []
    keep = np.concatenate([g["keep"] for g in gathered] + [np.zeros(0, np.uint8)])
    if not np.array_equal(keep, single["keep"]):
        bad.append("keep_vs_single_gpu")
    if not np.array_equal(keep, want_keep):
        bad.append("keep_vs_oracle")
    if "keep" in extra and (extra["card"] != gathered[0]["stats"]["cardinality_upper_bound"] or extra["key_bits"] != gathered[0]["stats"]["key_bits"]
                            or not np.array_equal(keep, extra["keep"])):
        bad.append("fixture")
    st = [g["stats"] for g in gathered]
    if any((s["cardinality_upper_bound"], s["key_bits"]) != (single["stats"]["cardinality_upper_bound"], single["stats"]["key_bits"]) for s in st):
        bad.append("bound_or_key_bits")
    if [st[0]["cardinality_upper_bound"], st[0]["key_bits"]] != want[:2]:
        bad.append("bound_vs_oracle")
    distinct = sum(s["distinct_keys_rank"] for s in st)
    if distinct != single["stats"]["distinct_keys"] or distinct != want[2] or any(s["distinct_keys"] != distinct for s in st):
        bad.append("distinct_keys")
    if [s["kept"] for s in st] != [int(g["keep"].sum()) for g in gathered]:
        bad.append("kept")
    apply = case.get("apply", True)
    for r, g in enumerate(gathered):
        survivors = [x for x, f in zip(shards[r], g["keep"]) if f] if apply else shards[r]
        if g["reads_after"] != survivors:
            bad.append("reads_r%d" % r)
    if "owned0" in extra:
        from spades_b200.distributed import cov_layout_host
        _, cap = cov_layout_host(world, st[0]["cardinality_upper_bound"], np.zeros(0, np.uint64))
        share = -(-st[0]["cardinality_upper_bound"] // world)
        if st[0]["distinct_keys_rank"] != extra["owned0"] or \
                (world > 1 and (st[0]["distinct_keys_rank"] < 0.85 * cap or st[0]["distinct_keys_rank"] <= share * 3 // 2)):
            bad.append("owner_load %d of %d" % (st[0]["distinct_keys_rank"], cap))
    return bad


def run_cases(rank, world, device, cases):
    import torch.distributed as dist
    from dist_worker import check_case as check_count
    from spades_b200.distributed import DistributedKMerCounter, distributed_cov_filter
    from spades_b200.kmer_index import Context, KMerIndexBuilder, SpadesGpuError
    from spades_b200.packing import pack_reads, unpack_reads
    from spades_b200.reads_io import CovFilteringWrap, download_reads
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
    lines = []
    for case in cases:
        K, thr, shards, extra = case_shards(case, world)
        apply = case.get("apply", True)
        ctx.set_reads(*pack_reads(shards[rank]))
        keep, stats = distributed_cov_filter(ctx, K, thr, apply=apply)
        res = dict(keep=keep, stats=stats, reads_after=unpack_reads(*download_reads(ctx)))
        cnt = None
        if case.get("count_B"):
            # filter then count: the survivors of every rank are the distributed count's shards
            st = DistributedKMerCounter(ctx, K).Count(case["count_B"])
            idx = KMerIndexBuilder(ctx).BuildIndex(st)
            cnt = dict(keys=st.kmers(), counts=st.counts(), bsz=st.bucket_sizes(), npass=1, checksum=st.checksum(), index=idx.serialize())
            idx.free(); st.free()
        gathered = [None] * world
        dist.all_gather_object(gathered, res)
        counts = [None] * world
        dist.all_gather_object(counts, cnt)
        if rank == 0:
            union = [r for s in shards for r in s]
            ctx.set_reads(*pack_reads(union))
            skeep, sstats = CovFilteringWrap(ctx, K, thr, apply=False)
            bad = check_case(case, world, K, thr, shards, extra, gathered, dict(keep=skeep, stats=sstats))
            if cnt is not None:
                filtered = [g["reads_after"] for g in gathered]
                cbad, _ = check_count(dict(K=K, B=case["count_B"], mode=0), world, filtered, counts)
                bad += ["count_" + b for b in cbad]
            line = "dist cov case W=%d %-16s K=%-3d thr=%d reads=%-5d bound=%-6d kept=%-5d %s" % (
                world, case["name"], K, thr, sum(len(s) for s in shards), gathered[0]["stats"]["cardinality_upper_bound"],
                sum(g["stats"]["kept"] for g in gathered), "OK" if not bad else "FAIL " + ",".join(bad))
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
        lines = run_cases(rank, world, 0, cases)
    finally:
        dist.destroy_process_group()
    if rank == 0:
        with open(out_path, "w") as f:
            f.write("\n".join(lines) + "\n")
