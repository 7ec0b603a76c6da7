"""Child process of tests/test_gpu_tuning.py: every case of CASES under ONE setting of the count's tuning knobs.

The knobs (SGPU_PA_MAX, SGPU_RMAX, SGPU_A_SUB) are read once per process, so each setting needs a process of its own; the parent
puts them in this process's environment only. The worker runs every case, then writes what each produced (keys, multiplicities,
bucket sizes, device checksum, serialized KMerIndex, the graph artefacts) and the context's counters after each count to one .npz;
the parent compares them with the C oracle.

    python tuning_worker.py OUT.npz WANT_GRAPH.npz

WANT_GRAPH.npz holds the oracle's (k+1)-mers and k-mers of the graph cases: a graph is only built over sets equal to them (a wrong
set would send the index and graph kernels to slots that do not exist).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from spades_b200.packing import pack_reads, revcomp, synthetic_reads  # noqa: E402

CANON, ALL = 0, 1
BUDGET = 64 << 20                 # the arena's minimum: one bucket per pass
HEAVY_COPIES = 4500               # copies of one read: every one of its keys has > 2 x 2048 records (local-sort capacity)
PATH_COUNTERS = ("level_a_key_bits", "level_a_scatters", "refine_rounds_max", "refine_splits_round0", "refine_splits_later",
                 "sort_lsd_fallbacks", "sort_oversize_equal", "passes", "instances", "launches")

# (name, input, K, B, mode or "graph", HBM budget of a context of its own, 0 = the worker's main context)
CASES = [
    ("k22", "mix", 22, 16, CANON, 0), ("k56", "mix", 56, 16, CANON, 0), ("k78", "mix", 78, 12, CANON, 0), ("k128", "mix", 128, 8, CANON, 0),
    ("all21", "mix", 21, 10, ALL, 0), ("all55", "mix", 55, 10, ALL, 0), ("all70", "mix", 70, 10, ALL, 0),
    ("k6", "mix", 6, 4, CANON, 0), ("k11", "mix", 11, 6, CANON, 0),
    ("k56_b2", "mix", 56, 2, CANON, 0),
    ("k56_passes", "mix", 56, 8, CANON, BUDGET), ("k128_passes", "mix", 128, 8, CANON, BUDGET),
] + [("polyA_few%d" % K, "polyA_few%d" % K, K, 2, CANON, 0) for K in (22, 56, 78, 128)] \
  + [("polyA_many%d" % K, "polyA_many%d" % K, K, 2, CANON, 0) for K in (22, 56, 78, 128)] \
  + [("graph21", "graph", 21, 12, "graph", 0), ("graph55", "graph", 55, 12, "graph", 0)]


def _random_seq(rng, n):
    return "".join("ACGT"[c] for c in rng.integers(0, 4, n))


def mix_reads():
    """~3 M windows at K = 22, the same under every setting:
      - 12 000 reads of a 30 kb genome at 1 % error;
      - HEAVY_COPIES copies of one read: equal-key segments longer than the local-sort capacity at every record width;
      - 300 palindromic reads x + revcomp(x): self-reverse-complement keys at even K;
      - 2 000 reads of 100 A followed by a random tail of 50: long shared key prefixes, many keys per bin;
      - 2 500 reads of their own random sequence: keys that are all distinct;
      - ragged reads of K-2 .. K+2 bases around every K of CASES."""
    rng = np.random.default_rng(2610)
    reads = synthetic_reads(12_000, 150, 30_000, 0.01, seed=261)
    reads += [synthetic_reads(1, 150, 400, 0.0, seed=262)[0]] * HEAVY_COPIES
    for _ in range(300):
        x = _random_seq(rng, 75)
        reads.append(x + revcomp(x))
    reads += ["A" * 100 + _random_seq(rng, 50) for _ in range(2000)]
    reads += [_random_seq(rng, 150) for _ in range(2500)]
    for K in sorted({c[2] for c in CASES}):
        for L in range(max(1, K - 2), K + 3):
            reads += synthetic_reads(20, L, 30_000, 0.01, seed=263 + L)
    return reads


def polyA_reads(K, ndistinct, copies):
    """reads of exactly K bases: K-6 A and a random 6-base tail, `ndistinct` different tails. The key order compares the record's
    words from the first, and a word from its last base down, so the tail goes first when the key is one word (K <= 32) and last
    otherwise. Every key is minimal as it stands and all of them share their 2K-12 most significant key bits, so in a bucket they
    fall into ONE local-sort bin. With ~100 keys per bucket
    (copies 1-3 each) the bin has more than 16 distinct keys; with ~800 single keys per bucket the residual records overflow.
    Either sends the segment to the exact LSD fallback, at every record width."""
    rng = np.random.default_rng(2700 + K + ndistinct)
    tails = rng.choice(4 ** 6, size=ndistinct, replace=False)
    reads = []
    for i, t in enumerate(tails):
        tail = "".join("ACGT"[(int(t) >> (2 * j)) & 3] for j in range(6))
        read = tail + "A" * (K - 6) if K <= 32 else "A" * (K - 6) + tail
        reads += [read] * (1 + (i % 3 if copies else 0))
    return reads


def graph_reads():
    """reads of an 8 kb genome, 2 500 copies of one of them, palindromes and ragged reads: for the graph path at k = 21 and 55"""
    rng = np.random.default_rng(2800)
    reads = synthetic_reads(3000, 150, 8000, 0.01, seed=281)
    reads += [synthetic_reads(1, 150, 8000, 0.0, seed=281)[0]] * 2500
    for _ in range(60):
        x = _random_seq(rng, 75)
        reads.append(x + revcomp(x))
    for L in (20, 21, 22, 23, 54, 55, 56, 57):
        reads += synthetic_reads(20, L, 8000, 0.01, seed=282 + L)
    return reads


def reads_of(name):
    if name == "mix":
        return mix_reads()
    if name == "graph":
        return graph_reads()
    if name.startswith("polyA_few"):
        return polyA_reads(int(name[len("polyA_few"):]), 200, True)
    if name.startswith("polyA_many"):
        return polyA_reads(int(name[len("polyA_many"):]), 1600, False)
    raise ValueError(name)


def _counters(c):
    t = c.times()
    return {f: int(t[f]) for f in PATH_COUNTERS}


def strictly_increasing_in_buckets(keys, bsz):
    """records strictly increasing inside every bucket (word 0 most significant): the precondition of the MPHF build"""
    keys = np.asarray(keys)
    if len(keys) != int(np.sum(bsz)):
        return False
    if len(keys) < 2:
        return True
    a, b = keys[:-1], keys[1:]
    lt = np.zeros(len(a), bool)
    eq = np.ones(len(a), bool)
    for q in range(keys.shape[1]):
        lt |= eq & (a[:, q] < b[:, q])
        eq &= a[:, q] == b[:, q]
    first = np.cumsum(bsz)[:-1]
    first = first[(first > 0) & (first < len(keys))]
    lt[first - 1] = True                # a bucket's first record need not exceed the last record of the bucket before
    return bool(lt.all())


def _count(c, reads_packed, K, B, mode, out, name):
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder, ParallelSortingSplitter
    c.set_reads(*reads_packed)
    splitter = DeBruijnReadKMerSplitter(K) if mode == CANON else ParallelSortingSplitter(K)
    st = KMerDiskCounter(c, splitter).Count(B)
    try:
        cnt = _counters(c)
        keys, bsz = st.kmers(), st.bucket_sizes()
        out[name + "/keys"], out[name + "/bsz"] = keys, bsz
        if mode == CANON:
            out[name + "/counts"] = st.counts()
        out[name + "/checksum"] = np.array(st.checksum(), np.uint64)
        if strictly_increasing_in_buckets(keys, bsz):
            idx = KMerIndexBuilder(c).BuildIndex(st)
            out[name + "/index"] = np.frombuffer(idx.serialize(), np.uint8)
            idx.free()
        return cnt
    finally:
        st.free()


def _graph(c, reads_packed, k, B, want, out, name):
    """count(k+1), the k-mers of the (k+1)-mers, both indexes and the graph with coverage, through the C ABI"""
    import ctypes as C
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.graph import DeBruijnGraph
    from spades_b200.kmer_index import DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    c.set_reads(*reads_packed)
    objs = []
    cnt = {}
    try:
        kp = KMerDiskCounter(c, DeBruijnReadKMerSplitter(k + 1)).Count(B)
        objs.append(kp)
        cnt["kp"] = _counters(c)
        out[name + "/kpomers"], out[name + "/kp_counts"], out[name + "/kp_bsz"] = kp.kmers(), kp.counts(), kp.bucket_sizes()
        if not np.array_equal(out[name + "/kpomers"], want[name + "/kpomers"]):
            return cnt
        km = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(k, kp)).Count(B)
        objs.append(km)
        cnt["km"] = _counters(c)
        out[name + "/kmers"] = km.kmers()
        if not np.array_equal(out[name + "/kmers"], want[name + "/kmers"]):
            return cnt
        mk = KMerIndexBuilder(c).BuildIndex(km)
        objs.append(mk)
        mkp = KMerIndexBuilder(c).BuildIndex(kp)
        objs.append(mkp)
        opts = SgpuGraphOptions(1, 0, 0, 0.8, 10, 200)
        h = C.c_void_p()
        c.check(c.L.sgpu_graph_build_opts(c.h, kp.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h)))
        g = DeBruijnGraph(c, h, kp, km, mk, mkp)
        objs.append(g)
        out[name + "/kmer_index"] = np.frombuffer(mk.serialize(), np.uint8)
        out[name + "/kpomer_index"] = np.frombuffer(mkp.serialize(), np.uint8)
        out[name + "/masks"], out[name + "/cov"], out[name + "/hist"] = g.masks(), g.coverage(), g.histogram().astype(np.int64)
        out[name + "/unitigs"] = np.frombuffer("\n".join(g.unitigs()).encode(), np.uint8)
        out[name + "/gfa"] = np.frombuffer(g.gfa().encode(), np.uint8)
        return cnt
    finally:
        for o in reversed(objs):
            o.free()


def main(out_path, want_path):
    from spades_b200.kmer_index import Context
    want = dict(np.load(want_path))
    out, counters, errors = {}, {}, {}
    packed = {}
    main_ctx = Context(0)
    try:
        for name, inp, K, B, mode, budget in CASES:
            if inp not in packed:
                packed[inp] = pack_reads(reads_of(inp))
            c = Context(0, hbm_budget_bytes=budget) if budget else main_ctx
            try:
                if mode == "graph":
                    counters[name] = _graph(c, packed[inp], K, B, want, out, name)
                else:
                    counters[name] = _count(c, packed[inp], K, B, mode, out, name)
            except Exception as e:          # reported by the parent next to the case's name
                errors[name] = "%s: %s" % (type(e).__name__, e)
            finally:
                if budget:
                    c.close()
    finally:
        main_ctx.close()
    out["counters"] = np.frombuffer(json.dumps(counters).encode(), np.uint8)
    out["errors"] = np.frombuffer(json.dumps(errors).encode(), np.uint8)
    np.savez(out_path, **out)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
