"""Worker for the multi-process tests (launched by mp.spawn or torch.distributed.run).

run_plan (CPU, gloo): every rank fabricates per-partition counts, all_gathers them, runs the planning step of the
    distributed count and checks the tiling invariants of the exchange layout.
run_cases (GPU): the distributed count of a sharded read set for every case of CASES; rank 0 compares each rank's buckets,
    multiplicities, device checksums and per-rank KMerIndex with the oracle's count of the union and returns one line per
    case. Two ways to run it:
      run_spawned   W processes on ONE device joined by a gloo group (peer arenas are cudaIpc mappings between processes on
                    the same GPU, so the whole exchange protocol runs on a single card);
      __main__      one process per GPU under torch.distributed.run, NCCL.
"""
import os
import re
import sys
from datetime import timedelta

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ARENA_BYTES = 1 << 30              # explicit per-rank device arena: W ranks share one device
PLANNER_RESERVE = 192 << 20        # per-pass tables the distributed planner reserves next to the record buffers (kDistFixedBytes)


def run_plan(rank, world, port, out):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from spades_b200.distributed import owner_bounds, plan_host
    B, rA, W = 37, 2, 16
    npart = B << rA
    rng = np.random.default_rng(100 + rank)
    local = rng.integers(0, 5000, size=npart).astype(np.uint64)
    local[rng.integers(0, npart, 10)] = 0
    t = torch.from_numpy(local.view(np.int64))
    g = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(g, t)
    allc = torch.stack(g).numpy().view(np.uint64)
    tot = allc.sum(axis=0)
    budget = int(tot.sum() * W * 2 / 3)          # forces several passes
    npass, bounds, mx = plan_host(world, B, rA, allc, budget, W)
    ok = npass >= 1 and bounds[0] == 0 and bounds[-1] == B and all(bounds[i] < bounds[i + 1] for i in range(npass))
    # exchange layout: for every pass and owner the (source, partition) pieces tile [0, recv) without gaps or overlaps
    worst = 0
    for p in range(npass):
        ob = owner_bounds(int(bounds[p]), int(bounds[p + 1]), world)
        for gidx in range(world):
            qlo, qhi = ob[gidx] << rA, ob[gidx + 1] << rA
            pieces = []
            run = 0
            for q in range(qlo, qhi):
                off = run
                for s in range(world):
                    pieces.append((off, int(allc[s, q])))
                    off += int(allc[s, q])
                run += int(tot[q])
            pos = 0
            for off, n in pieces:
                ok &= off == pos
                pos += n
            ok &= pos == int(tot[qlo:qhi].sum())
            worst = max(worst, pos)
    ok &= worst == mx
    # every rank must have computed the same plan
    sig = torch.tensor([npass, mx] + [int(x) for x in bounds], dtype=torch.int64)
    sigs = [torch.empty_like(sig) for _ in range(world)]
    dist.all_gather(sigs, sig)
    ok &= all(bool((s == sig).all()) for s in sigs)
    out[rank] = bool(ok) and npass > 1
    dist.destroy_process_group()


# ---- read sets: every generator returns the shards of all ranks (each rank builds the same list and takes its own) ------------
def _synth(n, seed, L=150, genome=4000):
    from spades_b200.packing import synthetic_reads
    return synthetic_reads(n, L, genome, 0.01, seed=seed)


def _random_seq(rng, n):
    return "".join("ACGT"[c] for c in rng.integers(0, 4, n))


def _strided(reads, world):
    return [reads[r::world] for r in range(world)]


def _blocks(reads, world):
    n = len(reads)
    return [reads[n * r // world: n * (r + 1) // world] for r in range(world)]


def _selfrc(world, G):
    # palindromic reads x + revcomp(x): the centred window of an even K is its own reverse complement. Copies are adjacent, so
    # the strided split hands one key's copies to different ranks.
    from spades_b200.packing import revcomp
    rng = np.random.default_rng(22)
    pal = []
    for _ in range(10):
        x = _random_seq(rng, 60)
        pal += [x + revcomp(x)] * 5
    return _strided(pal + _synth(4000, 22), world)


def _skew(world, G):
    # rank 0: 5 000 copies of one read and 3 000 poly-A reads (a few keys with huge multiplicities, from every level-A CTA of
    # the source); the other ranks: random reads plus a few copies of the repeated read
    one = _synth(1, 5600)[0]
    heavy = [one] * 5000 + ["A" * 150] * 3000
    rest = _synth(4000, 5601)
    if world == 1:
        return [heavy + rest]
    return [heavy] + [s + [one] * 100 for s in _strided(rest, world - 1)]


def _all_ctas(world, G):
    # rank 0 holds exactly one 32-read tile per level-A CTA (G = 2 x SMs CTAs): every piece of that source is non-empty
    return [_synth(G * 32, 78)] + [_synth(1000, 78 + r) for r in range(1, world)]


def _empty_shards(world, G):
    # the last rank gets no reads at all, the one before it only reads shorter than K = 56
    rng = np.random.default_rng(5616)
    short = [_random_seq(rng, int(n)) for n in rng.integers(20, 56, 200)]
    rest = _synth(3000, 5616)
    if world == 1:
        return [rest + short]
    if world == 2:
        return [rest + short, []]
    return _strided(rest, world - 2) + [short, []]


def _long(world, G):
    # the last rank holds 64 reads of 400 .. 6 000 bp: their tiles do not fit the shared-memory stage of the rolling kernels
    rng = np.random.default_rng(569)
    genome = _random_seq(rng, 8000)
    long_reads = []
    for n in rng.integers(400, 6001, 64):
        s = int(rng.integers(0, 8000 - n + 1))
        long_reads.append(genome[s:s + n])
    rest = _synth(3000, 569)
    if world == 1:
        return [rest + long_reads]
    return _strided(rest, world - 1) + [long_reads]


READS = {
    "selfrc": _selfrc,
    "allwin": lambda world, G: _blocks(_synth(3000, 32), world),
    "k33": lambda world, G: _strided(_synth(5000, 33), world),
    "k56_blocks": lambda world, G: _blocks(_synth(3000, 56), world),
    "skew": _skew,
    "all_ctas": _all_ctas,
    "wide97": lambda world, G: _strided(_synth(4000, 97), world),
    "wide128": lambda world, G: _strided(_synth(4000, 128), world),
    "k5": lambda world, G: _strided(_synth(2000, 5), world),
    "empty_shards": _empty_shards,
    "long": _long,
    "reuse": lambda world, G: _strided(_synth(3000, 40), world),
}

CANON, ALLWIN = 0, 1
# name, K, B, mode, read set, fixed per-pass budget (bytes above the planner's reserve per window of the union; None: free memory),
# passes required, counter shared between cases (None: a new DistributedKMerCounter)
CASES = [
    dict(name="k22_selfrc", K=22, B=7, mode=CANON, reads="selfrc"),
    dict(name="k32_allwin", K=32, B=16, mode=ALLWIN, reads="allwin"),
    dict(name="k33_nw2", K=33, B=40, mode=CANON, reads="k33"),
    dict(name="k56_B1", K=56, B=1, mode=CANON, reads="k56_blocks"),
    dict(name="k56_B2", K=56, B=2, mode=CANON, reads="k56_blocks"),
    dict(name="k56_skew", K=56, B=2, mode=CANON, reads="skew"),
    dict(name="k78_passes", K=78, B=64, mode=CANON, reads="all_ctas", budget=6, min_passes=3),
    dict(name="k97_passes", K=97, B=11, mode=CANON, reads="wide97", budget=6, min_passes=3),
    dict(name="k128_passes", K=128, B=11, mode=CANON, reads="wide128", budget=6, min_passes=3),
    dict(name="k5_sparse", K=5, B=64, mode=CANON, reads="k5"),
    dict(name="k56_B3000", K=56, B=3000, mode=CANON, reads="k56_blocks"),
    dict(name="k56_B8192", K=56, B=8192, mode=CANON, reads="k56_blocks"),
    dict(name="k56_empty", K=56, B=16, mode=CANON, reads="empty_shards"),
    dict(name="k56_long", K=56, B=9, mode=CANON, reads="long"),
    dict(name="reuse_B40", K=56, B=40, mode=CANON, reads="reuse", counter="reuse"),
    dict(name="reuse_B12", K=56, B=12, mode=CANON, reads="reuse", counter="reuse"),
]


def _rotl(w, s):
    return (w << np.uint64(s)) | (w >> np.uint64(64 - s))


def oracle_checksum(ks):
    """kset_checksum_k of the oracle's set: (n, sum of words x (2q+1), xor of words rotated by 7q+1, sum of multiplicities)"""
    if ks.n == 0:
        return [0, 0, 0, 0]
    keys = ks.keys.astype(np.uint64)
    s = int((keys * (2 * np.arange(ks.nw, dtype=np.uint64) + 1)[None, :]).sum(dtype=np.uint64))
    x = 0
    for q in range(ks.nw):
        x ^= int(np.bitwise_xor.reduce(_rotl(keys[:, q], 7 * q + 1)))
    c = int(ks.counts.astype(np.uint64).sum()) if ks.counts is not None else 0
    return [int(ks.n), s, x, c]


def check_case(case, world, shards, gathered):
    """rank 0: the ranks' results of one case against the oracle's count of the union -> (names of failed checks, oracle set)"""
    import golden_util
    import oracle as O
    from spades_b200.packing import pack_reads
    K, B, mode = case["K"], case["B"], case["mode"]
    union = [r for s in shards for r in s]
    ks = O.count(*pack_reads(union), K, B, mode)
    bad = []
    bsz = [g["bsz"] for g in gathered]
    if not np.array_equal(sum(bsz), ks.bsz):
        bad.append("bucket_sizes")
    # every non-empty bucket is non-empty on exactly one rank; reassemble the ranks' records in bucket order
    nonempty = np.stack([b > 0 for b in bsz])
    if not np.array_equal(nonempty.sum(axis=0), (ks.bsz > 0).astype(np.int64)):
        bad.append("ownership")
    parts_k, parts_c = [], []
    offs_r = [0] * world
    for b in range(B):
        for r in np.flatnonzero(nonempty[:, b]):
            nb = int(bsz[r][b])
            parts_k.append(gathered[r]["keys"][offs_r[r]:offs_r[r] + nb])
            if mode == CANON:
                parts_c.append(gathered[r]["counts"][offs_r[r]:offs_r[r] + nb])
            offs_r[r] += nb
    allk = np.concatenate(parts_k) if parts_k else np.zeros((0, ks.nw), np.uint64)
    if not np.array_equal(allk.ravel(), ks.keys.ravel()):
        bad.append("keys")
    if mode == CANON:
        allc = np.concatenate(parts_c) if parts_c else np.zeros(0, np.uint32)
        if not np.array_equal(allc, ks.counts):
            bad.append("multiplicities")
    # the order-independent device checksums (bench.py's multi-GPU self check) add / xor up to the union's
    cs = [g["checksum"] for g in gathered]
    m64 = (1 << 64) - 1
    tot = [sum(c[0] for c in cs), sum(c[1] for c in cs) & m64, 0, sum(c[3] for c in cs) & m64]
    for c in cs:
        tot[2] ^= c[2]
    if tot != oracle_checksum(ks):
        bad.append("checksum")
    # per-rank KMerIndex = the oracle's MPHF over the same buckets: the rank's buckets at full size, every other bucket empty
    start = np.concatenate(([0], np.cumsum(ks.bsz)))
    for r in range(world):
        own = nonempty[r]
        sel = np.concatenate([np.arange(start[b], start[b + 1]) for b in np.flatnonzero(own)] + [np.zeros(0, np.int64)]).astype(np.int64)
        part = O.kset_from_arrays(ks.keys[sel], None if ks.counts is None else ks.counts[sel], np.where(own, ks.bsz, 0), K)
        if not golden_util.index_equal(O.Mphf(part).serialize(), gathered[r]["index"], B):
            bad.append("index_r%d" % r)
    npass = [g["npass"] for g in gathered]
    if len(set(npass)) != 1:
        bad.append("passes_differ")
    if case.get("budget") is not None and npass[0] < max(2, case.get("min_passes", 2)):
        bad.append("passes")
    return bad, ks


def run_cases(rank, world, device, backend, cases):
    """Run every case of `cases` (dicts of CASES) as one distributed count over the default process group. Returns the
    result lines on rank 0 (one per case: OK or the checks that failed), [] elsewhere; ["SKIP ..."] when a rank other than 0
    cannot create its device context."""
    import torch
    import torch.distributed as dist
    from spades_b200.distributed import DistributedKMerCounter
    from spades_b200.kmer_index import Context, KMerIndexBuilder, SpadesGpuError
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
    G = 2 * torch.cuda.get_device_properties(device).multi_processor_count      # level-A CTAs per source (levelA_ctas_per_sm)
    lines = []
    counters = {}
    for case in cases:
        K, B, mode = case["K"], case["B"], case["mode"]
        shards = READS[case["reads"]](world, G)
        mine = shards[rank]
        ctx.set_reads(*pack_reads(mine))
        budget = None
        if case.get("budget") is not None:
            windows = sum(max(0, len(r) - K + 1) for s in shards for r in s)
            budget = PLANNER_RESERVE + case["budget"] * windows
        key = case.get("counter")
        cnt = counters.setdefault(key, DistributedKMerCounter(ctx, K, mode)) if key else DistributedKMerCounter(ctx, K, mode)
        st = cnt.Count(B, budget_bytes=budget)
        idx = KMerIndexBuilder(ctx).BuildIndex(st)
        res = dict(keys=st.kmers(), counts=st.counts() if mode == CANON else None, bsz=st.bucket_sizes(), npass=cnt.npass,
                   checksum=st.checksum(), index=idx.serialize())
        idx.free(); st.free()
        gathered = [None] * world
        dist.all_gather_object(gathered, res)
        if rank == 0:
            bad, ks = check_case(case, world, shards, gathered)
            line = "dist case W=%d %-12s K=%-3d B=%-4d reads=%-5d passes=%-2d distinct=%-7d %s" % (
                world, case["name"], K, B, sum(len(s) for s in shards), gathered[0]["npass"], ks.n, "OK" if not bad else "FAIL " + ",".join(bad))
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
