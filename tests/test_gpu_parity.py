"""GPU parity tests (run with -m gpu on an H100). Everything goes through the C ABI (spades_b200/_lib.py);
the checker is the reference's golden output (tests/golden) or the C oracle on the same seeded inputs."""
import numpy as np
import pytest

import golden_util as G
import oracle as O
from spades_b200.packing import pack_reads, revcomp, synthetic_reads

pytestmark = pytest.mark.gpu


def _oracle_art(reads, k, B, **clippers):
    """the oracle's artefacts of the whole path (clippers: early_tc / early_at of O.full_graph); `oracle` keeps its sets and MPHFs"""
    r = O.full_graph(reads, k, B, **clippers)
    return dict(kpomers=r["kp"].keys, kp_bsz=r["kp"].bsz, kmers=r["km"].keys, kmer_index=r["mk"].serialize(),
                kpomer_index=r["mkp"].serialize(), masks=r["masks"], cov=r["cov"], hist=r["hist"].astype(np.int64),
                unitigs=r["unitigs"].seqs, gfa=r["gfa"], kp_counts=r["kp"].counts, oracle=r)


def _compare(a, b, B):
    bad = []
    for key in ("kpomers", "kp_bsz", "kmers", "masks", "cov", "hist", "kp_counts"):
        if not np.array_equal(np.asarray(a[key]).ravel(), np.asarray(b[key]).ravel()):
            bad.append(key)
    for key in ("kmer_index", "kpomer_index"):
        if not G.index_equal(a[key], b[key], B):
            bad.append(key)
    if list(a["unitigs"]) != list(b["unitigs"]):
        bad.append("unitigs")
    if a["gfa"] != b["gfa"]:
        bad.append("gfa")
    return bad


def test_device_arithmetic():
    from gpu_util import ctx
    from test_hostdev_helpers import check_all, check_roll
    check_all(ctx().h, 1)
    check_roll(ctx().h, 1)


@pytest.mark.parametrize("name", G.names("graph"))
def test_graph_matches_reference_golden(name):
    from gpu_util import gpu_graph_artifacts
    g = G.load(name)
    art, _ = gpu_graph_artifacts(g["reads"], g["k"], g["B"])
    assert G.check_graph(g, art) == []


@pytest.mark.parametrize("name", G.names("tcgraph"))
def test_early_tip_clipper_matches_reference_golden(name):
    """sgpu_graph_build_ex with the pipeline's early tip clipper against the unmodified reference's EarlyTipClipperProcessor:
    clipped mask array, removed-k-mer count, and the unitigs / GFA built from the clipped index"""
    from gpu_util import gpu_graph_artifacts
    g = G.load(name)
    art, gr = gpu_graph_artifacts(g["reads"], g["k"], g["B"], early_tc=g["tc_bound"])
    assert G.check_graph(g, art) == []


@pytest.mark.parametrize("name", G.names("atgraph"))
def test_early_at_clipper_matches_reference_golden(name):
    """sgpu_graph_build_opts with the RNA pipeline's early A/T clipper (and the tip clipper after it where the fixture has one)
    against the unmodified reference's EarlyLowComplexityClipperProcessor: clipped masks, both return values, unitigs, GFA"""
    from gpu_util import gpu_graph_artifacts
    g = G.load(name)
    art, gr = gpu_graph_artifacts(g["reads"], g["k"], g["B"], early_tc=g.get("tc_bound", 0), early_at=True)
    assert G.check_graph(g, art) == []


@pytest.mark.parametrize("k,B,n,L,glen,seed", [(21, 8, 2500, 100, 2500, 61), (55, 12, 2500, 150, 4000, 62), (77, 3, 1500, 150, 2500, 63), (13, 2, 1500, 60, 700, 64)])
def test_early_at_clipper_matches_oracle_random(k, B, n, L, glen, seed):
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden import at_reads
    from gpu_util import gpu_graph_artifacts
    reads = at_reads(n, L, glen, 0.01, seed)
    art, gr = gpu_graph_artifacts(reads, k, B, early_tc=L - k, early_at=True)
    r = O.full_graph(reads, k, B, early_tc=L - k, early_at=True)
    assert r["at"][0] > 0 and r["at"][2] > 0
    assert gr.at_clipper_stats() == r["at"]
    assert gr.tip_clipper_stats() == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])
    assert np.array_equal(art["masks"], r["masks"]) and art["unitigs"] == r["unitigs"].seqs and art["gfa"] == r["gfa"]


@pytest.mark.parametrize("name", G.names("eigraph"))
def test_edge_index_refill_matches_reference_golden(name):
    """sgpu_edge_index_build over the GPU's own unitigs against the unmodified reference's EdgeIndex refill (KmerFreeEdgeIndex +
    GraphPositionFillingIndexBuilder + EdgeInfoUpdater): serialized KMerIndex, and (edge id, offset / tombstone) of every slot"""
    from gpu_util import ctx
    from spades_b200.graph import DeBruijnGraphConstructor, EdgeIndex
    from spades_b200.packing import pack_reads
    g = G.load(name)
    c = ctx()
    c.set_reads(*pack_reads(g["reads"]))
    gr = DeBruijnGraphConstructor(c, g["k"], g["B"]).ConstructGraph()
    assert gr.unitigs() == g["unitigs_txt"].tobytes().decode().split()
    K = int(g["ei_k"][0])
    ei = EdgeIndex(gr, None if K == g["k"] + 1 else K, int(g["ei_chunks"][0]) if K == g["k"] + 1 else g["B"])
    ids, offs = ei.values()
    assert G.check_edge_index(g, ei.serialize(), ids, offs, 1 if K == g["k"] + 1 else g["B"]) == []
    ei.free(); gr.free()


def _edge_index_reads(kind, k, K, seed):
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden import isolated_reads, pal_reads
    if kind == "syn":
        return synthetic_reads(800, 150, 1500, 0.01, seed=seed)
    if kind == "pal":              # palindromes of length K (self-RC windows) and hairpins (self-conjugate edges)
        return pal_reads((K or k + 1) // 2, 20, 10, seed, synthetic_reads(300, 150, 1500, 0.01, seed=seed))
    if kind == "small":            # a few hundred edges: the oracle's loop puts every window of K = 1 or 2
        return synthetic_reads(150, 100, 1500, 0.01, seed=seed)
    if kind == "big":              # > 4096 edges: the unitigs are packed on several host threads
        return synthetic_reads(3000, 150, 4000, 0.02, seed=seed)
    if kind.startswith("iso"):
        return isolated_reads(int(kind[3:]), seed)
    assert kind == "empty"
    return ["ACGTACGTAC", "GGGTTTAAACCC"]


def _check_edge_index_refill(k, B, K, kind, seed):
    """sgpu_edge_index_build against the oracle's refill: ids, offsets, the serialized index (with the branch the (k+1)-mer path
    takes for B vertex chunks) and a lookup of every key"""
    from gpu_util import ctx
    from spades_b200.graph import DeBruijnGraphConstructor, EdgeIndex
    c = ctx()
    c.set_reads(*pack_reads(_edge_index_reads(kind, k, K, seed)))
    gr = DeBruijnGraphConstructor(c, k, B).ConstructGraph()
    u = gr.unitigs()
    ei = EdgeIndex(gr, K, B)
    ids, offs = ei.values()
    ks, m, want_ids, want_offs = O.edge_index(u, k, K, 1 if K is None else B)
    # each case holds what it is there for
    if kind == "pal":              # self-conjugate edges; self-RC windows on ordinary edges for K < k+1 (at K = k+1 there are none)
        Kw = K or k + 1
        on_ordinary = [s[j:j + Kw] for s in u if s != revcomp(s) for j in range(len(s) - Kw + 1) if s[j:j + Kw] == revcomp(s[j:j + Kw])]
        assert any(s == revcomp(s) for s in u) and bool(on_ordinary) == (K is not None)
    if kind == "big":
        assert len(u) >= 4096
    if kind.startswith("iso"):
        assert G.edge_index_single(u, k, B) == (kind == "iso5")
    if kind == "empty":
        assert u == [] and ks.n == 0
    assert ei.size() == ks.n and np.array_equal(ids, want_ids) and np.array_equal(offs, want_offs)
    assert G.index_equal(G.edge_index_bytes(m, u, k, K or k + 1, B), ei.serialize(), 1 if K is None else B)
    slots = ei.seq_idx(ks.keys)
    assert np.array_equal(slots, np.array([m.lookup(key) for key in ks.keys], np.uint64))
    assert np.array_equal(np.sort(slots), np.arange(ks.n, dtype=np.uint64))
    # the reads' set is untouched by the refill: counting again gives the same (k+1)-mers
    assert np.array_equal(DeBruijnGraphConstructor(c, k, B).ConstructGraph().kpomers.kmers(), gr.kpomers.kmers())
    ei.free(); gr.free()


def test_edge_index_refill_matches_oracle_random():
    for k, B, K, seed in ((21, 6, None, 71), (33, 4, 25, 72), (55, 12, None, 73), (77, 3, 41, 74)):
        _check_edge_index_refill(k, B, K, "syn", seed)


@pytest.mark.parametrize("k,B,K,kind,seed", [
    (33, 4, 31, "syn", 75), (33, 4, 32, "syn", 76), (41, 5, 33, "syn", 77),              # one key word | two
    (77, 6, 63, "syn", 78), (63, 6, None, "syn", 79), (99, 7, 65, "syn", 80),            # two | three
    (99, 5, 96, "syn", 81), (99, 6, 97, "syn", 82), (127, 6, None, "syn", 83),           # three | four, K = 128
    (55, 6, 40, "pal", 84), (21, 6, None, "pal", 85),
    (21, 6, 1, "small", 86), (21, 6, 2, "small", 87),
    (21, 20, None, "iso4", 14), (21, 20, None, "iso5", 15), (21, 6, None, "empty", 0), (21, 6, 15, "empty", 0),
    (21, 16, None, "big", 1), (21, 16, 15, "big", 1)])
def test_edge_index_refill_matches_oracle_cases(k, B, K, kind, seed):
    """both sides of every key-word boundary, K = 1 and 2, self-RC windows and self-conjugate edges, both sides of the single-index
    branch, the empty graph, and a graph whose unitigs are packed on several host threads"""
    _check_edge_index_refill(k, B, K, kind, seed)


@pytest.mark.parametrize("k,B,n,L,glen,err,seed", [(21, 16, 3000, 100, 4000, 0.02, 51), (55, 20, 3000, 150, 4000, 0.02, 52), (77, 3, 1500, 150, 2000, 0.01, 53),
                                                   (9, 3, 1000, 60, 600, 0.1, 54), (33, 2, 2000, 120, 900, 0.03, 55)])
def test_early_tip_clipper_matches_oracle_random(k, B, n, L, glen, err, seed):
    from gpu_util import gpu_graph_artifacts
    reads = synthetic_reads(n, L, glen, err, seed=seed)
    art, gr = gpu_graph_artifacts(reads, k, B, early_tc=L - k)
    r = O.full_graph(reads, k, B, early_tc=L - k)
    assert r["tc"]["removed"] > 0
    assert gr.tip_clipper_stats() == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])
    assert np.array_equal(art["masks"], r["masks"]) and art["unitigs"] == r["unitigs"].seqs and art["gfa"] == r["gfa"]


@pytest.mark.parametrize("name", G.names("count"))
def test_kmercount_matches_reference_golden(name):
    from gpu_util import gpu_count_artifacts
    g = G.load(name)
    art, _ = gpu_count_artifacts(g["reads"], g["k"], g["B"])
    assert G.check_count(g, art) == []


@pytest.mark.parametrize("k,B,n,L,glen,seed", [
    (21, 16, 3000, 100, 4000, 1), (31, 7, 2000, 150, 3000, 2), (33, 40, 2000, 150, 3000, 3), (55, 80, 3000, 150, 5000, 4),
    (63, 5, 1500, 150, 2000, 5), (65, 9, 1500, 150, 2000, 6), (77, 3, 1500, 150, 2000, 7), (99, 11, 1200, 150, 2000, 8),
    (127, 2, 1000, 150, 1500, 9), (5, 4, 400, 60, 300, 10), (3, 1, 200, 40, 100, 11),
])
def test_graph_matches_oracle_random(k, B, n, L, glen, seed):
    from gpu_util import gpu_graph_artifacts
    reads = synthetic_reads(n, L, glen, 0.01, seed=seed)
    art, _ = gpu_graph_artifacts(reads, k, B)
    assert _compare(art, _oracle_art(reads, k, B), B) == []


def test_ragged_empty_and_short_reads():
    from gpu_util import gpu_graph_artifacts
    rng = np.random.default_rng(3)
    base = synthetic_reads(600, 150, 1500, 0.01, seed=12)
    reads = []
    for i, r in enumerate(base):
        cut = int(rng.integers(1, 150))
        reads.append(r[:cut])                      # lengths 1..149, many shorter than k+1 (skipped, kmer_splitters.hpp:30-31)
    reads += ["A", "ACGT", "ACGTACGTACGTACGTACGTACGT"]
    art, _ = gpu_graph_artifacts(reads, 21, 6)
    assert _compare(art, _oracle_art(reads, 21, 6), 6) == []


def test_long_reads_take_the_unstaged_path():
    """reads of 400..6000 bp: a warp tile's packed reads no longer fit its shared-memory staging slice (kRollStageWords), so the
    level-A kernels read the words from global memory; mixed with short reads so that staged and unstaged tiles alternate"""
    from gpu_util import gpu_graph_artifacts
    rng = np.random.default_rng(8)
    genome = "".join("ACGT"[i] for i in rng.integers(0, 4, 9000))
    reads = []
    for _ in range(700):
        L = int(rng.choice([150, 400, 1000, 2500, 6000]))
        st = int(rng.integers(0, len(genome) - L + 1))
        r = genome[st:st + L]
        reads.append(r if rng.random() < 0.5 else revcomp(r))
    for k, B in ((21, 5), (55, 3), (77, 2)):
        art, _ = gpu_graph_artifacts(reads, k, B)
        assert _compare(art, _oracle_art(reads, k, B), B) == []


def test_no_kmers_at_all():
    from gpu_util import gpu_graph_artifacts
    reads = ["ACGT", "AC", "GGGTTT"]
    art, _ = gpu_graph_artifacts(reads, 21, 4)
    assert art["kpomers"].size == 0 and art["kmers"].size == 0 and art["unitigs"] == []
    assert _compare(art, _oracle_art(reads, 21, 4), 4) == []


def test_heavy_hitters_and_low_complexity():
    """the same read thousands of times (segments of identical keys larger than the local-sort capacity), poly-A,
    tandem repeats (long shared key prefixes -> the 32-bit optimistic sort window must fall back)."""
    from gpu_util import gpu_graph_artifacts
    one = synthetic_reads(1, 150, 400, 0.0, seed=21)[0]
    reads = [one] * 5000 + ["A" * 150] * 3000 + ["AC" * 75] * 100 + ["ACGTTGCA" * 18 + "ACGTTG"] * 50
    reads += synthetic_reads(500, 150, 800, 0.01, seed=22)
    for k, B in ((21, 3), (55, 2)):
        art, _ = gpu_graph_artifacts(reads, k, B)
        assert _compare(art, _oracle_art(reads, k, B), B) == []


def test_perfect_loops_and_hairpin_loop():
    from gpu_util import gpu_graph_artifacts
    rng = np.random.default_rng(5)
    g = "".join("ACGT"[i] for i in rng.integers(0, 4, 700))
    gg = g + g
    reads = [gg[i:i + 120] for i in range(0, 700, 7)]
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 200))
    h = x + revcomp(x)
    hh = h + h
    reads += [hh[i:i + 150] for i in range(0, 400, 5)]
    for k, B in ((21, 4), (33, 2)):
        art, _ = gpu_graph_artifacts(reads, k, B)
        assert _compare(art, _oracle_art(reads, k, B), B) == []


@pytest.mark.parametrize("K,B,seed", [(21, 16, 31), (32, 3, 32), (55, 16, 33), (64, 5, 34), (96, 4, 35), (128, 2, 36)])
def test_kmercount_matches_oracle_random(K, B, seed):
    from gpu_util import gpu_count_artifacts
    reads = synthetic_reads(1500, 150, 2500, 0.01, seed=seed)
    art, _ = gpu_count_artifacts(reads, K, B)
    words, offs, lens = pack_reads(reads)
    ks = O.count(words, offs, lens, K, B, 1)
    assert np.array_equal(art["final_kmers"].ravel(), ks.keys.ravel()) and np.array_equal(art["bsz"], ks.bsz)


def test_medium_size_properties_and_oracle():
    """60 k reads x 150 bp, k=55 (5.7 M windows): exercises level-A fan-out + MSD refinement at non-toy sizes."""
    from gpu_util import ctx
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    from spades_b200.packing import pack_fixed
    codes = synthetic_reads(60000, 150, 60000, 0.01, seed=77, as_codes=True)
    words, offs, lens = pack_fixed(codes)
    c = ctx()
    c.set_reads(words, offs, lens)
    K, B = 56, 80
    st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
    keys, counts, bsz = st.kmers(), st.counts(), st.bucket_sizes()
    # size-independent properties: total multiplicity == number of windows (no self-RC doubling can lose any), strictly
    # increasing inside buckets, bucket function honoured
    assert int(counts.astype(np.uint64).sum()) >= 60000 * (150 - K + 1)
    off = 0
    for b in range(B):
        kb = keys[off:off + bsz[b]]
        if len(kb) > 1:
            lt = (kb[:-1, 0] < kb[1:, 0]) | ((kb[:-1, 0] == kb[1:, 0]) & (kb[:-1, 1] < kb[1:, 1]))
            assert lt.all()
        off += bsz[b]
    ks = O.count(words, offs, lens, K, B, 0)
    assert np.array_equal(keys.ravel(), ks.keys.ravel()) and np.array_equal(counts, ks.counts) and np.array_equal(bsz, ks.bsz)
    # device checksums (bench.py's multi-GPU self check): n, weighted word sum, xor of rotated words, multiplicity sum
    n_, s_, x_, c_ = st.checksum()
    wsum = int((ks.keys * (2 * np.arange(ks.nw, dtype=np.uint64) + 1)[None, :]).sum(dtype=np.uint64))
    rot = [7 * q + 1 for q in range(ks.nw)]
    xr = 0
    for q in range(ks.nw):
        col = ks.keys[:, q]
        xr ^= int(np.bitwise_xor.reduce((col << np.uint64(rot[q])) | (col >> np.uint64(64 - rot[q]))))
    assert (n_, s_, x_, c_) == (ks.n, wsum, xr, int(ks.counts.astype(np.uint64).sum()))
    idx = KMerIndexBuilder(c).BuildIndex(st)
    ids = idx.seq_idx(keys)
    assert len(np.unique(ids)) == len(keys) and ids.max() == len(keys) - 1       # phm_test.cpp:22-79 properties
    assert G.index_equal(O.Mphf(ks).serialize(), idx.serialize(), B)


# ---- parity at scale (VERDICT r01, "Next round" #2) ----------------------------------------------------------------------------
def _count_with_budget(words, offs, lens, K, B, budget):
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    c = Context(0, hbm_budget_bytes=budget)
    try:
        c.set_reads(words, offs, lens)
        st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
        t = c.times()
        keys, counts, bsz = st.kmers(), st.counts(), st.bucket_sizes()
        idx = KMerIndexBuilder(c).BuildIndex(st)
        ser = idx.serialize()
        idx.free(); st.free()
        return keys, counts, bsz, ser, int(t["passes"])
    finally:
        c.close()


@pytest.mark.parametrize("budget_mb,min_passes", [(420, 3), (200, 5)])
def test_forced_bucket_group_passes_match_oracle(budget_mb, min_passes):
    """200 k reads x 150 bp, k=55 (19 M records = 304 MB per buffer) inside a context whose HBM budget only holds a fraction: the
    multi-pass loop the 100 M-read bench runs (5 passes there), with the partition-id array (420 MB) and without it (200 MB: the ids
    no longer fit, every pass re-hashes). Keys, multiplicities, bucket sizes and the serialized KMerIndex must equal the oracle's."""
    from spades_b200.packing import pack_fixed
    codes = synthetic_reads(200_000, 150, 200_000, 0.01, seed=91, as_codes=True)
    words, offs, lens = pack_fixed(codes)
    K, B = 56, 80
    keys, counts, bsz, ser, passes = _count_with_budget(words, offs, lens, K, B, budget_mb << 20)
    assert passes >= min_passes, passes
    ks = O.count(words, offs, lens, K, B, 0)
    assert np.array_equal(bsz, ks.bsz)
    assert np.array_equal(keys.ravel(), ks.keys.ravel()) and np.array_equal(counts, ks.counts)
    assert G.index_equal(O.Mphf(ks).serialize(), ser, B)


def test_histogram_super_ranges_match_oracle():
    """more buckets than one level-A launch can address (B << rA > 8192): the histogram super-range loop"""
    from gpu_util import ctx
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter
    from spades_b200.packing import pack_fixed
    codes = synthetic_reads(20_000, 150, 20_000, 0.01, seed=92, as_codes=True)
    words, offs, lens = pack_fixed(codes)
    c = ctx()
    for K, B in ((56, 20_000), (22, 9_000)):
        c.set_reads(words, offs, lens)
        st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
        keys, counts, bsz = st.kmers(), st.counts(), st.bucket_sizes()
        st.free()
        ks = O.count(words, offs, lens, K, B, 0)
        assert np.array_equal(bsz, ks.bsz) and np.array_equal(keys.ravel(), ks.keys.ravel()) and np.array_equal(counts, ks.counts)


def _uleb(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


@pytest.mark.parametrize("case", ["k21", "k55"])
def test_million_reads_sha256(case):
    """BASELINE.md 3.6: byte identity with the UNMODIFIED reference on a >= 1 M-read synthetic set. tests/golden/syn1M_sha256.json holds
    the SHA-256 of every artefact `ref_probe graph` wrote for these reads (tests/golden/make_golden_1m.py); the same bytes are
    rebuilt here from the GPU path's outputs."""
    import hashlib
    import json
    import os
    from gpu_util import ctx
    from spades_b200.graph import DeBruijnGraphConstructor
    from spades_b200.packing import pack_fixed
    fx = json.load(open(os.path.join(G.GOLDEN_DIR, "syn1M_sha256.json")))
    r, cs = fx["reads"], fx["cases"][case]
    codes = synthetic_reads(r["n"], r["len"], r["genome_len"], r["err"], seed=r["seed"], as_codes=True)
    lut = np.frombuffer(b"ACGT", dtype=np.uint8)
    txt = np.empty((r["n"], r["len"] + 1), np.uint8)
    txt[:, :r["len"]] = lut[codes]; txt[:, r["len"]] = 10
    assert hashlib.sha256(txt.tobytes()).hexdigest() == r["sha256_text"], "the generator no longer reproduces the fixture's reads"
    del txt
    k, B = cs["k"], cs["B"]
    c = ctx()
    c.set_reads(*pack_fixed(codes))
    g = DeBruijnGraphConstructor(c, k, B).ConstructGraph(keep_perfect_loops=True, with_coverage=True)
    mine = {
        "kpomers": g.kpomers.kmers().tobytes(),
        "kpomer_bucket_sizes.txt": "".join("%d\n" % x for x in g.kpomers.bucket_sizes()).encode(),
        "kmers": g.kmers.kmers().tobytes(),
        "kmer_index.bin": _uleb(k) + g.kmer_index.serialize(),
        "kpomer_index.bin": _uleb(k + 1) + g.kpomer_index.serialize(),
        "masks.bin": g.masks().tobytes(),
        "coverage.bin": g.coverage().tobytes(),
        "histogram.txt": "".join("%d\n" % x for x in g.histogram()).encode(),
        "unitigs.txt": "".join(u + "\n" for u in g.unitigs()).encode(),
        "graph.gfa": g.gfa().encode(),
    }
    bad = [f for f, h in cs["sha256"].items() if hashlib.sha256(mine[f]).hexdigest() != h]
    sizes = {f: (len(mine[f]), cs["bytes"][f]) for f in bad}
    g.free()
    assert bad == [], sizes


# ---- coverage pre-filter (SURVEY 8f-3) --------------------------------------------------------------------------------------------
def _kept_reads(c):
    from spades_b200.reads_io import download_reads
    from spades_b200.packing import unpack_reads
    words, offs, lens = download_reads(c)
    return unpack_reads(words, offs, lens)


@pytest.mark.parametrize("name", G.names("covfilter"))
def test_gpu_coverage_prefilter_matches_reference_golden(name):
    """cardinality bound, filter key width and the verdict per read against the unmodified reference's CoverageFilter phase; with apply
    the context's read set becomes the survivors in their original order"""
    from gpu_util import ctx
    from spades_b200.reads_io import CovFilteringWrap
    g = G.load(name)
    K, thr = g["k"] + 1, int(g["thr"][0])
    c = ctx()
    c.set_reads(*pack_reads(g["reads"]))
    keep, st = CovFilteringWrap(c, K, thr, apply=False)
    assert st["cardinality_upper_bound"] == int(g["card"][0]) and st["key_bits"] == int(g["key_bits"][0])
    assert np.array_equal(keep, g["keep"]) and st["kept"] == int(g["keep"].sum())
    keep2, _ = CovFilteringWrap(c, K, thr, apply=True)
    assert np.array_equal(keep2, keep)
    assert _kept_reads(c) == [r for r, f in zip(g["reads"], g["keep"]) if f]


@pytest.mark.parametrize("K,thr,seed", [(22, 2, 1), (56, 3, 2), (33, 1, 3), (64, 2, 4), (70, 2, 5), (12, 4, 6), (21, 0, 7)])
def test_gpu_coverage_prefilter_matches_oracle_random(K, thr, seed):
    """ragged, short, low-complexity and palindromic reads; K odd / even, one word / two words / K >= 64 (rotation by K mod 64)"""
    from gpu_util import ctx
    from spades_b200.reads_io import CovFilteringWrap
    rng = np.random.default_rng(seed)
    reads = synthetic_reads(1500, 120, 3000, 0.01, seed=seed) + synthetic_reads(300, 90, 40000, 0.02, seed=seed + 100)
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 80))
    reads += [x + revcomp(x)] * 3 + ["A" * 150, "T" * 97, "AC" * 40, "ACGT", "", x[:K - 1], x[:K]]
    reads = [r[: int(rng.integers(K - 2, len(r) + 1))] if rng.random() < 0.2 and len(r) > K else r for r in reads]
    reads = [r for r in reads if r]
    words, offs, lens = pack_reads(reads)
    want_keep, want = O.cov_filter(words, offs, lens, K, thr)
    c = ctx()
    c.set_reads(words, offs, lens)
    keep, st = CovFilteringWrap(c, K, thr, apply=True)
    assert [st["cardinality_upper_bound"], st["key_bits"], st["distinct_keys"], st["kept"]] == want
    assert np.array_equal(keep, want_keep)
    assert _kept_reads(c) == [r for r, f in zip(reads, want_keep) if f]


@pytest.mark.parametrize("case", ["k21", "k55"])
def test_million_reads_coverage_prefilter(case):
    """the coverage pre-filter on the 1 M-read synthetic set: cardinality bound, key width, number of survivors and the SHA-256 of the
    verdicts as the unmodified reference produced them (tests/golden/make_golden_1m_cov.py), then the count of the SURVIVORS against a
    count of the same reads handed over directly"""
    import hashlib
    import json
    import os
    from gpu_util import ctx
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter
    from spades_b200.packing import pack_fixed
    from spades_b200.reads_io import CovFilteringWrap
    r = json.load(open(os.path.join(G.GOLDEN_DIR, "syn1M_sha256.json")))["reads"]
    cs = json.load(open(os.path.join(G.GOLDEN_DIR, "syn1M_covfilter.json")))["cases"][case]
    codes = synthetic_reads(r["n"], r["len"], r["genome_len"], r["err"], seed=r["seed"], as_codes=True)
    c = ctx()
    c.set_reads(*pack_fixed(codes))
    keep, st = CovFilteringWrap(c, cs["k"] + 1, cs["threshold"], apply=True)
    assert st["cardinality_upper_bound"] == cs["cardinality_upper_bound"] and st["key_bits"] == cs["key_bits"] and st["kept"] == cs["kept"]
    assert hashlib.sha256(keep.tobytes()).hexdigest() == cs["sha256_keep"]
    a = KMerDiskCounter(c, DeBruijnReadKMerSplitter(cs["k"] + 1)).Count(16)
    ka, ca = a.kmers().copy(), a.counts().copy(); a.free()
    c.set_reads(*pack_fixed(codes[keep.astype(bool)]))
    b = KMerDiskCounter(c, DeBruijnReadKMerSplitter(cs["k"] + 1)).Count(16)
    assert np.array_equal(ka, b.kmers()) and np.array_equal(ca, b.counts()); b.free()
