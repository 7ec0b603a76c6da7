"""GPU parity of everything that consumes a counted set split into several chunks (run with -m gpu on an H100).

A count keeps one chunk per bucket-group pass. The session context of the other GPU tests has an arena of most of the device, so
every count there is one pass and every consumer sees a single chunk. Here each test opens its own context with a small HBM
budget, so that the same sets come in many chunks:
  - 64 MiB, the arena's minimum: the budget left after what is resident is below the fixed term of a pass's estimate, so every
    pass holds exactly one bucket (passes == B);
  - a budget calibrated so that a pass holds several buckets, but not all of them (2 <= passes < B).
The checker is the C oracle on the same reads. The pass counts are asserted too, so a budget that stops splitting the sets fails
instead of quietly testing the single-chunk path again."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest

import golden_util as G
import gpu_util
import oracle as O
from spades_b200.packing import pack_reads, revcomp, synthetic_reads
from test_gpu_parity import _compare, _oracle_art

pytestmark = pytest.mark.gpu

MIN_BUDGET = 64 << 20            # the arena's minimum (sgpu_internal.h): one bucket per pass
CALIBRATED_BUDGET = 72 << 20     # 4 passes per count for the k = 55 case below (H100 80GB HBM3, 132 SMs; 70-76 MiB all split it)
MAX_CHUNKS = 128                 # chunks one set may hold (kMaxChunks, sgpu_internal.h)


@contextlib.contextmanager
def _budgeted(budget):
    """a context of its own on device 0 with `budget` bytes of HBM; the session's shared context is closed first"""
    from spades_b200.kmer_index import Context
    gpu_util.release()
    c = Context(0, hbm_budget_bytes=budget)
    try:
        yield c
    finally:
        c.close()


def _loop_reads():
    """the perfect loop and the hairpin loop of test_perfect_loops_and_hairpin_loop"""
    rng = np.random.default_rng(5)
    g = "".join("ACGT"[i] for i in rng.integers(0, 4, 700))
    gg = g + g
    reads = [gg[i:i + 120] for i in range(0, 700, 7)]
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 200))
    h = x + revcomp(x)
    hh = h + h
    return reads + [hh[i:i + 150] for i in range(0, 400, 5)]


def _tiny_reads(glen, seed):
    """error-free reads of a short genome, a short perfect loop and a short hairpin loop: few enough distinct k-mers that some
    buckets stay empty, so empty chunks sit between full ones"""
    rng = np.random.default_rng(seed)
    reads = synthetic_reads(3000, 100, glen, 0.0, seed=seed)
    g = "".join("ACGT"[i] for i in rng.integers(0, 4, 60))
    reads += [(g + g)[i:i + 50] for i in range(0, 60, 3)]
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 30))
    h = x + revcomp(x)
    return reads + [(h + h)[i:i + 50] for i in range(0, 60, 3)]


def _at_reads(n, L, glen, err, seed):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden import at_reads
    return at_reads(n, L, glen, err, seed)


def _graph_path(c, reads, k, B, want, early_tc=0, early_at=False, then=None):
    """DeBruijnGraphConstructor.ConstructGraph step by step: count(k+1), k-mers of the (k+1)-mers, both indexes, the graph.
    Returns (artefacts, (passes of the (k+1)-mer count, passes of the k-mer count), tip clipper stats, A/T clipper stats,
    lookups of every key through both GPU indexes, then(graph) or None). The sets are checked against `want` before anything
    indexes them: a wrong set would send the graph kernels to slots that do not exist."""
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.graph import DeBruijnGraph
    from spades_b200.kmer_index import DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    c.set_reads(*pack_reads(reads))
    objs = []
    try:
        kp = KMerDiskCounter(c, DeBruijnReadKMerSplitter(k + 1)).Count(B)
        objs.append(kp)
        kp_passes = int(c.times()["passes"])
        assert np.array_equal(kp.kmers().ravel(), want["kpomers"].ravel()), "(k+1)-mers differ"
        km = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(k, kp)).Count(B)
        objs.append(km)
        km_passes = int(c.times()["passes"])
        assert np.array_equal(km.kmers().ravel(), want["kmers"].ravel()), "k-mers differ"
        mk = KMerIndexBuilder(c).BuildIndex(km)
        objs.append(mk)
        mkp = KMerIndexBuilder(c).BuildIndex(kp)
        objs.append(mkp)
        opts = SgpuGraphOptions(1, int(early_tc), 1 if early_at else 0, 0.8, 10, 200)
        h = C.c_void_p()
        c.check(c.L.sgpu_graph_build_opts(c.h, kp.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h)))
        g = DeBruijnGraph(c, h, kp, km, mk, mkp)
        objs.append(g)
        art = dict(kpomers=kp.kmers(), kp_bsz=kp.bucket_sizes(), kmers=km.kmers(), kmer_index=mk.serialize(), kpomer_index=mkp.serialize(),
                   masks=g.masks(), cov=g.coverage(), hist=g.histogram().astype(np.int64), unitigs=g.unitigs(), gfa=g.gfa(),
                   kp_counts=kp.counts())
        lookups = dict(kpomers=mkp.seq_idx(art["kpomers"]), kmers=mk.seq_idx(art["kmers"]))
        extra = then(g) if then else None
        return art, (kp_passes, km_passes), g.tip_clipper_stats(), g.at_clipper_stats(), lookups, extra
    finally:
        for o in reversed(objs):
            o.free()


def _oracle_slots(mphf, keys):
    return np.array([mphf.lookup(key) for key in keys], np.uint64)


def _check_lookups(lookups, want):
    """KMerIndex.seq_idx of every key equals the oracle's MPHF lookup, and the slots are a permutation of 0..n-1"""
    r = want["oracle"]
    for name, keys, mphf in (("kpomers", want["kpomers"], r["mkp"]), ("kmers", want["kmers"], r["mk"])):
        got = lookups[name]
        assert np.array_equal(got, _oracle_slots(mphf, keys)), name + " lookups differ"
        assert np.array_equal(np.sort(got), np.arange(len(keys), dtype=np.uint64)), name + " lookups are not a permutation"


def _interior_empty(bsz):
    """an empty bucket with records on both sides of it"""
    nz = np.flatnonzero(bsz)
    return len(nz) > 0 and bool((bsz[nz[0]:nz[-1]] == 0).any())


# (k, B, budget, reads): word pairs (1,1) (2,2) (3,3) (4,4) of k-mers / (k+1)-mers
GRAPH_CASES = [
    (21, 24, MIN_BUDGET, "syn"), (55, 16, MIN_BUDGET, "syn"), (77, 32, MIN_BUDGET, "syn"), (127, 40, MIN_BUDGET, "syn"),
    (21, 120, MIN_BUDGET, "tiny"), (55, 16, CALIBRATED_BUDGET, "syn"),
]


def _case_reads(kind, k):
    if kind == "tiny":
        return _tiny_reads(180, 41)
    return synthetic_reads(3000, 150, 3000, 0.004 if k > 100 else 0.01, seed=40 + k) + _loop_reads()


@pytest.mark.parametrize("k,B,budget,kind", GRAPH_CASES)
def test_graph_path_on_pass_split_sets(k, B, budget, kind):
    """every artefact of the whole path (sets, bucket sizes, both serialized indexes, masks, coverage, histogram, unitigs, GFA)
    and every key's slot in both indexes, over sets of one chunk per bucket (64 MiB) or of a few buckets per chunk"""
    reads = _case_reads(kind, k)
    want = _oracle_art(reads, k, B)
    if kind == "tiny":
        assert _interior_empty(want["kp_bsz"]) and _interior_empty(want["oracle"]["km"].bsz)
    with _budgeted(budget) as c:
        art, passes, _, _, lookups, _ = _graph_path(c, reads, k, B, want)
    if budget == MIN_BUDGET:
        assert passes == (B, B)
    else:
        assert all(2 <= p < B for p in passes), passes
    assert _compare(art, want, B) == []
    _check_lookups(lookups, want)


@pytest.mark.parametrize("k,B", [(21, 24), (55, 16)])
def test_early_tip_clipper_on_pass_split_sets(k, B):
    L = 150
    reads = synthetic_reads(3000, L, 3000, 0.02, seed=50 + k) + _loop_reads()
    want = _oracle_art(reads, k, B, early_tc=L - k)
    r = want["oracle"]
    assert r["tc"]["removed"] > 0
    with _budgeted(MIN_BUDGET) as c:
        art, passes, tc, _, lookups, _ = _graph_path(c, reads, k, B, want, early_tc=L - k)
    assert passes == (B, B)
    assert tc == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])
    assert _compare(art, want, B) == []
    _check_lookups(lookups, want)


def test_early_at_clipper_on_pass_split_sets():
    k, B, L = 21, 20, 100
    reads = _at_reads(2500, L, 2500, 0.01, 61)
    want = _oracle_art(reads, k, B, early_tc=L - k, early_at=True)
    r = want["oracle"]
    assert r["at"][0] > 0 and r["at"][2] > 0
    with _budgeted(MIN_BUDGET) as c:
        art, passes, tc, at, lookups, _ = _graph_path(c, reads, k, B, want, early_tc=L - k, early_at=True)
    assert passes == (B, B)
    assert at == r["at"]
    assert tc == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])
    assert _compare(art, want, B) == []
    _check_lookups(lookups, want)


def test_more_buckets_than_the_chunk_table_holds():
    """B = 300 at the 64 MiB budget: one bucket per pass would make 300 chunks, more than the key table of the MPHF build and the
    graph kernels holds. The planner keeps the set within the table; the whole path must still equal the oracle."""
    k, B = 21, 300
    reads = _tiny_reads(400, 43)
    want = _oracle_art(reads, k, B)
    assert (want["kp_bsz"] == 0).any() and (want["oracle"]["km"].bsz == 0).any()
    with _budgeted(MIN_BUDGET) as c:
        art, passes, _, _, lookups, _ = _graph_path(c, reads, k, B, want)
    assert all(2 <= p <= MAX_CHUNKS for p in passes), passes
    assert _compare(art, want, B) == []
    _check_lookups(lookups, want)


@pytest.mark.parametrize("k,B,K", [(33, 6, 25), (21, 6, None), (99, 6, 97)])
def test_edge_index_in_a_budgeted_context(k, B, K):
    """EdgeIndex refill over a graph built at 64 MiB. K != k+1 counts the edges' K-mers into B buckets (one pass each); K = k+1
    counts them into one bucket. ids, offsets, the serialized index and a lookup of every oracle key against the oracle."""
    from spades_b200.graph import EdgeIndex
    reads = synthetic_reads(1000, 150, 1500, 0.01, seed=80 + k)
    want = _oracle_art(reads, k, B)
    ks, m, want_ids, want_offs = O.edge_index(want["unitigs"], k, K, 1 if K is None else B)

    def refill(gr):
        ei = EdgeIndex(gr, K, B)
        try:
            ids, offs = ei.values()
            return int(gr.ctx.times()["passes"]), ids, offs, ei.serialize(), ei.seq_idx(ks.keys)
        finally:
            ei.free()

    with _budgeted(MIN_BUDGET) as c:
        art, passes, _, _, _, (ei_passes, ids, offs, ser, slots) = _graph_path(c, reads, k, B, want, then=refill)
    assert passes == (B, B) and _compare(art, want, B) == []
    assert ei_passes == (1 if K is None else B)
    want_ser = G.edge_index_bytes(m, want["unitigs"], k, K or k + 1, B)
    assert len(ids) == ks.n and np.array_equal(ids, want_ids) and np.array_equal(offs, want_offs)
    assert G.index_equal(want_ser, ser, 1 if K is None else B)
    assert np.array_equal(slots, _oracle_slots(m, ks.keys))
    assert np.array_equal(np.sort(slots), np.arange(ks.n, dtype=np.uint64))


def test_set_accessors_across_chunk_boundaries(tmp_path):
    """a 64 MiB count, one chunk per bucket: ranged downloads of keys and multiplicities that start at, end at and straddle every
    chunk boundary, out-of-range requests, the device checksum, the per-bucket files and the merged final_kmers file"""
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter, SpadesGpuError
    K, B = 33, 12
    words, offs, lens = pack_reads(synthetic_reads(3000, 150, 3000, 0.01, seed=90))
    ks = O.count(words, offs, lens, K, B, 0)
    bstart = np.concatenate([[0], np.cumsum(ks.bsz)]).astype(np.int64)
    n = int(ks.n)
    with _budgeted(MIN_BUDGET) as c:
        c.set_reads(words, offs, lens)
        st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
        try:
            passes = int(c.times()["passes"])
            keys, counts, bsz = st.kmers(), st.counts(), st.bucket_sizes()
            ranges = [(0, n), (n, 0), (0, 0)]
            for e in bstart[1:-1]:
                e = int(e)
                ranges += [(max(0, e - 5), min(e, 5)), (e, min(5, n - e)), (max(0, e - 3), min(7, n - max(0, e - 3))), (e, 0)]
            got = [(f, m, st.kmers(f, m), st.counts(f, m)) for f, m in ranges]
            errors = []
            for f, m in ((n - 1, 2), (n + 1, 0), (0, n + 1)):
                for get in (st.kmers, st.counts):
                    try:
                        get(f, m)
                        errors.append(False)
                    except SpadesGpuError:
                        errors.append(True)
            checksum = st.checksum()
            st.write_buckets(tmp_path / "kmers")
            st.merge(tmp_path / "final_kmers")
        finally:
            st.free()
    assert passes == B
    assert np.array_equal(bsz, ks.bsz) and np.array_equal(keys, ks.keys) and np.array_equal(counts, ks.counts)
    for f, m, gk, gc in got:
        assert gk.shape == (m, ks.nw) and np.array_equal(gk, ks.keys[f:f + m]), (f, m)
        assert np.array_equal(gc, ks.counts[f:f + m]), (f, m)
    assert all(errors), errors
    wsum = int((ks.keys * (2 * np.arange(ks.nw, dtype=np.uint64) + 1)[None, :]).sum(dtype=np.uint64))
    xr = 0
    for q in range(ks.nw):
        col, rot = ks.keys[:, q], np.uint64(7 * q + 1)
        xr ^= int(np.bitwise_xor.reduce((col << rot) | (col >> (np.uint64(64) - rot))))
    assert checksum == [n, wsum, xr, int(ks.counts.astype(np.uint64).sum())]
    for b in range(B):
        assert (tmp_path / ("kmers.%d" % b)).read_bytes() == ks.keys[bstart[b]:bstart[b + 1]].tobytes(), b
    assert (tmp_path / "final_kmers").read_bytes() == ks.keys.tobytes()
