"""CPU tests: the plain-C oracle (oracle/spades_oracle.c) against
  * golden fixtures produced by the UNMODIFIED reference (tests/golden/make_golden.py -> ref_probe),
  * the known-answer unitig sets of the reference's own gtest (src/test/debruijn/construction_test.cpp:30-64),
  * RtSeq known answers (src/test/include_test/rtseq_test.cpp) for packing / RC / minimality,
  * the independent python-xxhash binding (xxHash 0.8.2) for the XXH3 restatement.
"""
import numpy as np
import pytest

import golden_util as G
import oracle as O
from spades_b200.packing import pack_reads, revcomp, unpack_kmers


def oracle_artifacts(reads, k, B, early_tc=0, early_at=False):
    r = O.full_graph(reads, k, B, early_tc=early_tc, early_at=early_at)
    art = dict(kpomers=r["kp"].keys, kp_bsz=r["kp"].bsz, kmers=r["km"].keys, kmer_index=r["mk"].serialize(),
               kpomer_index=r["mkp"].serialize(), masks=r["masks"], cov=r["cov"], hist=r["hist"],
               unitigs=r["unitigs"].seqs, gfa=r["gfa"])
    if early_tc:
        art.update(tc_removed=r["tc"]["removed"])
        if not early_at:
            art.update(masks_raw=r["masks_raw"])
    if early_at:
        art.update(at_removed=[r["at"][0], r["at"][2]])
    return art, r


@pytest.mark.parametrize("name", G.names("atgraph"))
def test_oracle_early_at_clipper_matches_reference_golden(name):
    """EarlyLowComplexityClipperProcessor (early_simplification.hpp:164-347; the RNA pipeline's EarlyATClipper), alone and followed by
    the tip clipper: clipped masks, both return values, unitigs and GFA against the unmodified reference; and the order independence
    the CUDA version relies on (tip decisions on a snapshot of the masks give the same array as the sequential walk)."""
    g = G.load(name)
    art, r = oracle_artifacts(g["reads"], g["k"], g["B"], early_tc=g.get("tc_bound", 0), early_at=True)
    assert G.check_graph(g, art) == []
    assert r["at"][0] > 0 and r["at"][2] > 0
    snap_m, snap_s = O.early_at_clip(r["km"], r["mk"], r["masks_raw"], snapshot=True)
    seq_m, seq_s = O.early_at_clip(r["km"], r["mk"], r["masks_raw"], snapshot=False)
    assert np.array_equal(snap_m, seq_m) and snap_s == seq_s == r["at"]


@pytest.mark.parametrize("name", G.names("tcgraph"))
def test_oracle_early_tip_clipper_matches_reference_golden(name):
    """EarlyTipClipperProcessor (early_simplification.hpp:38-162) between mask fill and unitig extraction: clipped masks,
    removed-k-mer count, unitigs and GFA against the unmodified reference; and the order independence the CUDA version
    relies on (every walk on a snapshot of the masks gives the same array as the reference's sequential walk)."""
    g = G.load(name)
    art, r = oracle_artifacts(g["reads"], g["k"], g["B"], early_tc=g["tc_bound"])
    assert G.check_graph(g, art) == []
    assert r["tc"]["removed"] > 0
    snap = O.early_tip_clip(r["km"], r["mk"], r["masks_raw"], g["tc_bound"], snapshot=True)
    assert np.array_equal(snap[0], r["masks"]) and snap[1:] == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])


@pytest.mark.parametrize("name", G.names("eigraph"))
def test_oracle_edge_index_matches_reference_golden(name):
    """EdgeIndex refill (KmerFreeEdgeIndex over the constructed graph; alignment/edge_index.hpp, edge_index_builders.hpp:154-307): the
    serialized index and every slot's (edge id, offset / tombstone) against the unmodified reference, for the (k+1)-mer index of the
    pipeline (one segment) and for the counting path with a smaller K (10 x threads buckets)"""
    g = G.load(name)
    r = O.full_graph(g["reads"], g["k"], g["B"])
    assert r["unitigs"].seqs == g["unitigs_txt"].tobytes().decode().split()
    K = int(g["ei_k"][0])
    B = 1 if K == g["k"] + 1 else g["B"]
    ks, m, ids, offs = O.edge_index(r["unitigs"].seqs, g["k"], K, B)
    ser = G.edge_index_bytes(m, r["unitigs"].seqs, g["k"], K, int(g["ei_chunks"][0]))
    assert G.check_edge_index(g, ser, ids, offs, B) == []


@pytest.mark.parametrize("name", G.names("covfilter"))
def test_oracle_coverage_prefilter_matches_reference_golden(name):
    """SURVEY 8f-3: SymmetricCyclicHash of every window of the first 64 reads, the HLL cardinality bound, the CQF key width and the
    verdict per read as the unmodified reference produced them (EstimateCardinalityUpperBound -> qf::cqf -> FillCoverageHistogram ->
    io::CoverageFilter)"""
    g = G.load(name)
    K, thr = g["k"] + 1, int(g["thr"][0])
    words, offs, lens = pack_reads(g["reads"])
    hh = [O.cyclic_hash(words[int(offs[i]):], j, K) for i in range(min(64, len(g["reads"]))) for j in range(max(0, len(g["reads"][i]) - K + 1))]
    assert np.array_equal(np.array(hh, dtype=np.uint64), g["hashes"])
    keep, stats = O.cov_filter(words, offs, lens, K, thr)
    assert stats[0] == int(g["card"][0]) and stats[1] == int(g["key_bits"][0])
    assert (1 << stats[1]) - 1 == int(g["range_mask"][0])
    assert np.array_equal(keep, g["keep"]) and stats[3] == int(g["keep"].sum())
    assert 0 < stats[3] < len(keep)                                    # the fixtures exercise both verdicts


@pytest.mark.parametrize("name", G.names("graph"))
def test_oracle_graph_matches_reference_golden(name):
    g = G.load(name)
    art, r = oracle_artifacts(g["reads"], g["k"], g["B"])
    assert r["mk"].nfinal() == 0 and r["mkp"].nfinal() == 0
    assert G.check_graph(g, art) == []


@pytest.mark.parametrize("name", G.names("count"))
def test_oracle_kmercount_matches_reference_golden(name):
    g = G.load(name)
    words, offs, lens = pack_reads(g["reads"])
    ks = O.count(words, offs, lens, g["k"], g["B"], 1)
    assert G.check_count(g, dict(final_kmers=ks.keys, bsz=ks.bsz)) == []


GTEST = {  # construction_test.cpp:30-64
    "SimpleThread": (["ACAAACCACCA"], ["ACAAACCACCA"]),
    "SimpleThread2": (["ACAAACCACCC", "AAACCACCCAC"], ["ACAAACCACCCAC"]),
    "SplitThread": (["ACAAACCACCA", "ACAAACAACCC"], ["ACAAAC", "CAAACCACCA", "CAAACAACCC"]),
    "SplitThread2": (["ACAAACCACCA", "ACAAACAACCA"], ["AACCACCA", "ACAAAC", "CAAACCA", "CAAACAACCA"]),
    "Buldge": (["ACAAAACACCA", "ACAAACCACCA"], ["ACAAAACACCA", "ACAAACCACCA"]),
    "CondenseSimple": (["CGAAACCAC", "CGAAAACAC", "AACCACACC", "AAACACACC"], ["CGAAAACACAC", "CACACC", "CGAAACCACAC"]),
}


def test_oracle_reference_gtest_coverage_table():
    """construction_test.cpp:97-105 (SimpleTestEarlyPairedInfo, k = 3): edges and their coverage (every edge holds one 4-mer, so the
    average coverage AssertCoverage checks, test_utils.cpp:144-151, is the raw count KC)."""
    reads = ["CCCAC", "CCACG", "ACCAC", "CCACA"]       # both reads of both pairs; the strand of the mates does not matter
    want = {"CCCA": 1, "ACCA": 1, "CCAC": 4, "CACG": 1, "CACA": 1}
    r = O.full_graph(reads, 3, 2)
    got = {}
    for line in r["gfa"].splitlines():
        f = line.split("\t")
        if f[0] == "S":
            kc = int([x for x in f if x.startswith("KC:i:")][0][5:])
            got[f[2]] = kc
    assert len(got) == len(want)
    for seq, kc in got.items():
        key = seq if seq in want else revcomp(seq)
        assert want[key] == kc


@pytest.mark.parametrize("name", sorted(GTEST))
def test_oracle_reference_gtest_known_answers(name):
    reads, etalon = GTEST[name]
    r = O.full_graph(reads, 5, 3)
    got = set()
    for s in r["unitigs"].seqs:
        got.add(s); got.add(revcomp(s))
    want = set()
    for s in etalon:
        want.add(s); want.add(revcomp(s))
    assert got == want          # AssertGraph, src/test/debruijn/test_utils.cpp:109-138


def test_xxh3_matches_python_xxhash():
    xxhash = pytest.importorskip("xxhash")
    rng = np.random.default_rng(0)
    for nw in (1, 2, 3, 4):
        for _ in range(200):
            w = rng.integers(0, 2**63, size=nw, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=nw, dtype=np.uint64)
            b = w.tobytes()
            assert O.xxh3_64(w) == xxhash.xxh3_64_intdigest(b)
            lo, hi = O.xxh3_128(w)
            assert (hi << 64) | lo == xxhash.xxh3_128_intdigest(b)


def test_rtseq_known_answers():
    # rtseq_test.cpp: packing/str round trip and ReverseComplement (:671 `!RtSeq("ACGTTGCA...")`)
    import ctypes as C
    L = O.lib()
    for s in ["ACGT", "ACGTACGTACGTACGTACGTACGTACGTACGTACG", "TTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTTT", "A" * 127, "ACGTTGCAGGACT"]:
        K = len(s)
        w, _, _ = pack_reads([s])
        assert unpack_kmers(w, K) == [s]
        out = np.zeros(len(w), np.uint64)
        L.orc_rc(w.ctypes.data_as(C.c_void_p), K, out.ctypes.data_as(C.c_void_p))
        assert unpack_kmers(out, K) == [revcomp(s)]
        assert bool(L.orc_is_minimal(w.ctypes.data_as(C.c_void_p), K)) == (s <= revcomp(s))


@pytest.mark.parametrize("K,B,mode", [(22, 7, 0), (32, 16, 1), (33, 40, 0), (78, 5, 0), (128, 11, 0)])
def test_kset_from_arrays_round_trip(K, B, mode):
    """A KSet rebuilt from a count's own arrays is the same set: same records, counts and bucket sizes, and an MPHF that
    serializes to the same bytes. With some buckets emptied (what one rank of a distributed count owns) every other bucket
    keeps its keys and its slots."""
    from spades_b200.packing import synthetic_reads
    words, offs, lens = pack_reads(synthetic_reads(300, 150, 2000, 0.01, seed=K))
    ks = O.count(words, offs, lens, K, B, mode)
    assert ks.n > 0 and (ks.counts is None) == (mode == 1)
    rb = O.kset_from_arrays(ks.keys, ks.counts, ks.bsz, K)
    assert rb.n == ks.n and rb.nw == ks.nw and np.array_equal(rb.keys, ks.keys) and np.array_equal(rb.bsz, ks.bsz)
    assert (rb.counts is None and ks.counts is None) or np.array_equal(rb.counts, ks.counts)
    assert O.Mphf(rb).serialize() == O.Mphf(ks).serialize()
    # keep every other bucket
    start = np.concatenate(([0], np.cumsum(ks.bsz)))
    keep = np.arange(B) % 2 == 0
    sel = np.concatenate([np.arange(start[b], start[b + 1]) for b in range(B) if keep[b]] + [np.zeros(0, np.int64)]).astype(np.int64)
    part = O.kset_from_arrays(ks.keys[sel], None if ks.counts is None else ks.counts[sel], np.where(keep, ks.bsz, 0), K)
    assert part.n == len(sel)
    m_all, m_part = O.Mphf(ks), O.Mphf(part)
    pstart = np.concatenate(([0], np.cumsum(part.bsz)))
    for b in np.flatnonzero(keep)[:3]:
        for i in range(start[b], min(start[b + 1], start[b] + 20)):
            assert m_part.lookup(ks.keys[i]) - pstart[b] == m_all.lookup(ks.keys[i]) - start[b]
    with pytest.raises(ValueError):
        O.kset_from_arrays(ks.keys[:-1], None, ks.bsz, K)


def test_empty_and_short_inputs():
    # reads shorter than K are skipped (kmer_splitters.hpp:30-31); empty input gives empty buckets
    words, offs, lens = pack_reads(["ACGT", "AC"])
    ks = O.count(words, offs, lens, 6, 4, 0)
    assert ks.n == 0 and list(ks.bsz) == [0, 0, 0, 0]
    m = O.Mphf(ks)
    assert len(m.serialize()) == 8 + 4 * (28 + 8) + 5 * 8
