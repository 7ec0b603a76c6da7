"""Generates tests/golden/*.npz from the UNMODIFIED reference (oracle/_ref/ref_probe).

Run where the reference sources are available (they are needed to build oracle/_ref):
    make -C oracle ref && python tests/golden/make_golden.py
Each fixture holds the input reads and every artefact ref_probe dumps for them, so the oracle and the
CUDA path can be pinned against reference output on machines without the reference.
"""
import gzip
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from spades_b200.packing import longest_valid, revcomp, synthetic_reads  # noqa: E402

PROBE = os.path.join(ROOT, "oracle", "_ref", "ref_probe")
ECOLI = os.path.join(HERE, "ecoli_1K")       # the reference's test data set (src/projects/spades/test_dataset)


def ecoli_reads():
    reads = []
    for f in ("ecoli_1K_1.fq.gz", "ecoli_1K_2.fq.gz"):
        lines = gzip.open(os.path.join(ECOLI, f), "rt").read().split("\n")
        for i in range(1, len(lines), 4):
            s = longest_valid(lines[i].strip().upper())
            if s:
                reads.append(s)
    return reads


def loops_reads(loop_len=120, hairpin_len=150):
    """windows of a 500-bp circle (a perfect loop) and of a 400-bp hairpin circle x + rc(x); windows longer than k + 1 for every k"""
    rng = np.random.default_rng(5)
    g = "".join("ACGT"[i] for i in rng.integers(0, 4, 500))
    gg = g + g
    reads = [gg[i:i + loop_len] for i in range(0, 500, 7)]
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 200))
    h = x + revcomp(x)
    hh = h + h
    reads += [hh[i:i + hairpin_len] for i in range(0, 400, 5)]
    return reads


# the six literal-read cases of src/test/debruijn/construction_test.cpp:30-64 (k=5) with their etalon edges
GTEST_CASES = {
    "SimpleThread": (["ACAAACCACCA"], ["ACAAACCACCA"]),
    "SimpleThread2": (["ACAAACCACCC", "AAACCACCCAC"], ["ACAAACCACCCAC"]),
    "SplitThread": (["ACAAACCACCA", "ACAAACAACCC"], ["ACAAAC", "CAAACCACCA", "CAAACAACCC"]),
    "SplitThread2": (["ACAAACCACCA", "ACAAACAACCA"], ["AACCACCA", "ACAAAC", "CAAACCA", "CAAACAACCA"]),
    "Buldge": (["ACAAAACACCA", "ACAAACCACCA"], ["ACAAAACACCA", "ACAAACCACCA"]),
    "CondenseSimple": (["CGAAACCAC", "CGAAAACAC", "AACCACACC", "AAACACACC"], ["CGAAAACACAC", "CACACC", "CGAAACCACAC"]),
}


def at_reads(n, L, glen, err, seed):
    """RNA-like reads: poly-A tails, poly-T heads, A-rich noisy tails and pure low-complexity reads on top of the SURVEY 8(d) generator"""
    rng = np.random.default_rng(seed)
    out = []
    for r in synthetic_reads(n, L, glen, err, seed=seed):
        x = rng.random()
        if x < 0.15:
            cut = int(rng.integers(L // 3, L - 5)); r = r[:cut] + "A" * (L - cut)
        elif x < 0.25:
            cut = int(rng.integers(5, L // 2)); r = "T" * cut + r[cut:]
        elif x < 0.30:
            cut = int(rng.integers(L // 3, L - 5)); r = r[:cut] + "".join(rng.choice(list("AAAAAAAT"), L - cut))
        out.append(r)
    return out + ["A" * L] * 5 + ["AT" * (L // 2)] * 3


def at_arm_reads(arm_len, L, seed):
    """error-free windows of a stem that forks into an A-rich arm and a random arm, and one read that leaves the random arm for a
    4-base poly-A tip. The A-rich arm (88% A between C and G, no run longer than 12: it shares no k-mer with at_reads' A/T tails) is a
    low-complexity dead-end chain of arm_len vertices, so RemoveATTips clips it only when max_length >= arm_len. The poly-A tip
    is low-complexity on its own, but not once the root's last nucleotides are counted up to min_length."""
    rng = np.random.default_rng(seed)
    stem = _random_seq(rng, 150)
    rich, run = "A", 1
    while len(rich) < arm_len:
        c = "A" if run < 12 and rng.random() < 0.88 else "CG"[int(rng.integers(0, 2))]
        rich += c
        run = run + 1 if c == "A" else 0
    arms = [rich, "C" + _random_seq(rng, 199)]                          # the fork: A | C
    reads = [s[i:i + L] for s in (stem + a for a in arms) for i in range(0, len(s) - L + 1, 10)]
    s = stem + arms[1]
    j = max(j for j in range(len(s) - L + 4) if s[j + L - 4] != "A")
    return reads + [s[j:j + L - 4] + "AAAA"]


def _random_seq(rng, n):
    return "".join("ACGT"[i] for i in rng.integers(0, 4, n))


def pal_reads(half, n_pal, n_hairpin, seed, base=()):
    """`base` plus palindromes x + rc(x) (|x| = half) planted in random context, and reads along hairpins y + rc(y) (|y| = 120).
    A planted palindrome is a self-reverse-complementary window of length 2 * half on an ordinary edge; a hairpin becomes a
    self-conjugate edge, whose centre (k+1)-mer is its own reverse complement."""
    rng = np.random.default_rng(seed)
    reads = list(base)
    for _ in range(n_pal):
        x = _random_seq(rng, half)
        reads.append(_random_seq(rng, 60) + x + revcomp(x) + _random_seq(rng, 60))
    for _ in range(n_hairpin):
        y = _random_seq(rng, 120)
        h = y + revcomp(y)
        reads += [h[i:i + 150] for i in range(0, len(h) - 150 + 1, 15)]
    return reads


def isolated_reads(n, seed):
    """n random 70-bp reads: n isolated edges, 4 n vertices counting conjugates"""
    rng = np.random.default_rng(seed)
    return [_random_seq(rng, 70) for _ in range(n)]


def run_probe(mode, reads, k, B, T=2, early_tc=0, early_at=False, edge_index=None, no_loops=False):
    with tempfile.TemporaryDirectory() as d:
        rf = os.path.join(d, "reads.txt")
        open(rf, "w").write("\n".join(reads) + "\n")
        out = os.path.join(d, "out")
        env = dict(os.environ)
        if edge_index is not None:
            env["PROBE_EDGE_INDEX"] = str(edge_index)  # EdgeIndex refill over the constructed graph: 0 = (k+1)-mers, else that K (counting path)
        if early_at:
            env["PROBE_EARLY_AT"] = "1"                # EarlyLowComplexityClipperProcessor (RNA pipeline), before the tip clipper
        if early_tc:
            env["PROBE_EARLY_TC"] = str(early_tc)      # EarlyTipClipperProcessor between mask fill and unitig extraction
        if no_loops:
            env["PROBE_NO_LOOPS"] = "1"                # keep_perfect_loops = false: unbranching paths only
        subprocess.check_call([PROBE, mode, rf, str(k), str(B), str(T), out], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=env)
        res = {}
        for f in os.listdir(out):
            p = os.path.join(out, f)
            if os.path.isfile(p):
                res[f.replace(".", "_")] = np.frombuffer(open(p, "rb").read(), dtype=np.uint8)
        return res


def save(name, mode, reads, k, B, early_tc=0, edge_index=None):
    if ONLY and name not in ONLY:
        return
    """mode "tcgraph" = graph mode with the pipeline's early tip clipper (length bound early_tc); masks_bin is the array
    before the clipper, masks_tc_bin after it, everything downstream (unitigs, GFA) comes from the clipped index.
    mode "atgraph" = graph mode with the RNA pipeline's early A/T clipper (masks_at_bin, at_removed_txt), followed by the tip clipper
    when early_tc is given (then masks_tc_bin is the array after both).
    mode "nlgraph" = graph mode with keep_perfect_loops = false."""
    res = run_probe("graph" if mode in ("tcgraph", "atgraph", "eigraph", "nlgraph") else mode, reads, k, B, early_tc=early_tc,
                    early_at=(mode == "atgraph"), edge_index=edge_index, no_loops=(mode == "nlgraph"))
    if edge_index is not None:
        res["ei_k"] = np.array([edge_index if edge_index else k + 1])
        res["ei_chunks"] = np.array([10 * 2])          # run_probe's T = 2: the (k+1)-mer path walks the edges in 10 x T vertex chunks
    if early_tc:
        res["tc_bound"] = np.array([early_tc])
    res["reads"] = np.frombuffer("\n".join(reads).encode(), dtype=np.uint8)
    res["k"] = np.array([k]); res["B"] = np.array([B]); res["mode"] = np.frombuffer(mode.encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **res)
    print(name, {a: len(b) for a, b in res.items() if a not in ("k", "B", "mode")})


def save_covfilter(name, reads, k, thr):
    if ONLY and name not in ONLY:
        return
    """SURVEY 8f-3: ref_probe covfilter = the pipeline's CoverageFilter phase (EstimateCardinalityUpperBound -> qf::cqf ->
    FillCoverageHistogram -> CoverageFilter on every read) over (k+1)-mers; keeps the cardinality bound, the filter's key bits, the
    verdict per read and the SymmetricCyclicHash of every window of the first 64 reads."""
    with tempfile.TemporaryDirectory() as d:
        rf = os.path.join(d, "reads.txt")
        open(rf, "w").write("\n".join(reads) + "\n")
        out = os.path.join(d, "out")
        env = dict(os.environ); env["PROBE_COV_THR"] = str(thr)
        subprocess.check_call([PROBE, "covfilter", rf, str(k), "4", "2", out], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=env)
        card, bits, mask, _ = [int(x) for x in open(os.path.join(out, "covfilter.txt")).read().split()]
        keep = np.array([int(x) for x in open(os.path.join(out, "keep.txt")).read().split()], dtype=np.uint8)
        hashes = np.fromfile(os.path.join(out, "hashes.bin"), dtype=np.uint64)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), reads=np.frombuffer("\n".join(reads).encode(), dtype=np.uint8), k=np.array([k]),
                        thr=np.array([thr]), card=np.array([card], dtype=np.uint64), key_bits=np.array([bits]), range_mask=np.array([mask], dtype=np.uint64),
                        keep=keep, hashes=hashes, mode=np.frombuffer(b"covfilter", dtype=np.uint8))
    print(name, "reads", len(reads), "kept", int(keep.sum()), "card", card, "key bits", bits)


def covfilter_reads(seed):
    """a well-covered genome, a thinly covered one, palindromes (self-RC (k+1)-mers), short and low-complexity reads"""
    rng = np.random.default_rng(seed)
    reads = synthetic_reads(2500, 100, 4000, 0.01, seed=seed) + synthetic_reads(400, 100, 30000, 0.01, seed=seed + 1)
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 60))
    pal = x + revcomp(x)
    reads += [pal] * 4 + [pal[10:110]] * 2 + ["A" * 100] * 3 + ["ACGT" * 10, "ACGTACGTAC", "AC" * 45]
    order = rng.permutation(len(reads))
    return [reads[i] for i in order]


REF_FASTX = os.path.join(ROOT, "oracle", "_ref", "ref_fastx")


def ingest_case_files():
    """small FASTA/FASTQ files that exercise the vendored kseq's corner semantics (see tests/test_ingest.py)"""
    rng = np.random.default_rng(11)
    def rnd(n, pn=0.0, lower=0.0):
        s = rng.choice(list("ACGT"), n)
        s = np.where(rng.random(n) < pn, "N", s)
        s = np.where(rng.random(n) < lower, np.char.lower(s), s)
        return "".join(s)
    seqs = [rnd(int(rng.integers(1, 200)), 0.03, 0.2) for _ in range(120)] + ["", "NNNN", "n", "ACGT ACGTA"]
    fq = "".join("@r%d c\n%s\n+\n%s\n" % (i, s, ("@>+I" * (len(s) // 4 + 1))[:len(s)]) for i, s in enumerate(seqs))
    fa = "junk before the first record\n" + "".join(">s%d\n%s\n%s" % (i, "\n".join(s[j:j + 40] for j in range(0, len(s), 40)), "\n" if i % 4 == 0 else "")
                                                    for i, s in enumerate(seqs)) + ">last\nACGTTGCA"
    mq = "".join("@m%d\n%s\n+m%d\n%s\nnoise without markers\n" % (i, "\n".join((s or "A")[j:j + 30] for j in range(0, len(s or "A"), 30)), i,
                                                                      "\n".join(("I" * len(s or "A"))[j:j + 30] for j in range(0, len(s or "A"), 30)))
                 for i, s in enumerate(seqs[:60]))
    return {"fastq": fq.encode(), "fastq_crlf_gz": gzip.compress(fq.replace("\n", "\r\n").encode()), "fasta_multiline": fa.encode(), "fastq_multiline": mq.encode()}


def save_ingest():
    if ONLY and "ingest_cases" not in ONLY:
        return
    res = {}
    with tempfile.TemporaryDirectory() as d:
        for name, data in ingest_case_files().items():
            f = os.path.join(d, name + (".gz" if name.endswith("_gz") else ".txt"))
            open(f, "wb").write(data)
            out = os.path.join(d, "out.txt")
            subprocess.check_call([REF_FASTX, f, out], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            res["file_" + name] = np.frombuffer(data, np.uint8)
            res["parsed_" + name] = np.frombuffer(open(out, "rb").read(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "ingest_cases.npz"), **res)
    print("ingest_cases", {a: len(b) for a, b in res.items()})


ONLY = set()          # fixture names to (re)write (the command line); empty = all of them


if __name__ == "__main__":
    ONLY.update(sys.argv[1:])
    save_ingest()
    ec = ecoli_reads()
    save("ecoli_k21_B40_graph", "graph", ec, 21, 40)          # BASELINE.json configs[0]
    save("ecoli_k21_B16_count", "count", ec, 21, 16)          # spades-kmercount defaults (kmercount.cpp:220)
    save("ecoli_k55_B16_graph", "graph", ec[:1500], 55, 16)
    save("ecoli_k77_B7_graph", "graph", ec[:800], 77, 7)
    save("ecoli_k99_B3_graph", "graph", ec[:800], 99, 3)
    save("syn_k21_B10_graph", "graph", synthetic_reads(400, 100, 1500, 0.01, seed=1), 21, 10)
    save("syn_k33_B5_count", "count", synthetic_reads(300, 100, 1500, 0.01, seed=2), 33, 5)
    save("loops_k21_B10_graph", "graph", loops_reads(), 21, 10)
    # keep_perfect_loops = false: the circles' edges are left out; synthetic reads add ordinary unitigs
    save("loops_k21_B10_nlgraph", "nlgraph", loops_reads() + synthetic_reads(300, 120, 700, 0.02, seed=3), 21, 10)
    save("loops_k127_B7_nlgraph", "nlgraph", loops_reads(250, 250) + synthetic_reads(200, 250, 1000, 0.0005, seed=17), 127, 7)
    save("dense_k5_B4_graph", "graph", synthetic_reads(200, 60, 200, 0.02, seed=3), 5, 4)
    save("dense_k3_B1_graph", "graph", synthetic_reads(100, 40, 100, 0.02, seed=4), 3, 1)
    # Construction stage with early_tc (stages/construction.cpp:289-302): length bound = read length - k
    save("ecoli_k21_B40_tcgraph", "tcgraph", ec, 21, 40, early_tc=100 - 21)
    save("ecoli_k55_B16_tcgraph", "tcgraph", ec[:1500], 55, 16, early_tc=100 - 55)
    save("syn_k21_B10_tcgraph", "tcgraph", synthetic_reads(2000, 100, 3000, 0.02, seed=6), 21, 10, early_tc=79)
    save("loops_k21_B10_tcgraph", "tcgraph", loops_reads() + synthetic_reads(300, 120, 700, 0.02, seed=3), 21, 10, early_tc=99)
    save("dense_k7_B4_tcgraph", "tcgraph", synthetic_reads(800, 60, 400, 0.03, seed=14), 7, 4, early_tc=10)
    # four-word k-mers: the multi-k pipeline's k = 99 and 127 on 250-bp reads
    save("syn_k99_B9_tcgraph", "tcgraph", synthetic_reads(150, 250, 1000, 0.001, seed=15), 99, 9, early_tc=250 - 99)
    save("syn_k127_B5_tcgraph", "tcgraph", synthetic_reads(150, 250, 1000, 0.001, seed=16), 127, 5, early_tc=250 - 127)
    # RNA pipeline: EarlyATClipper (stages/construction.cpp:317-340), alone and followed by the tip clipper (:447-450)
    save("rna_k21_B8_atgraph", "atgraph", at_reads(3000, 100, 3000, 0.01, 1), 21, 8)
    save("rna_k33_B5_atgraph", "atgraph", at_reads(1000, 150, 1500, 0.02, 2), 33, 5, early_tc=150 - 33)       # fixtures stay below 1 MB
    save("rna_k55_B16_atgraph", "atgraph", at_reads(1000, 150, 2000, 0.01, 3), 55, 16, early_tc=150 - 55)
    save("rna_k11_B3_atgraph", "atgraph", at_reads(1500, 60, 800, 0.05, 4), 11, 3)
    # four-word k-mers (k = 97): 250-bp reads and an A-rich dead-end arm of 350 vertices, past RemoveATTips' max_length of 200
    save("rna_k97_B6_atgraph", "atgraph", at_reads(120, 250, 800, 0.002, 5) + at_arm_reads(350, 250, 6), 97, 6, early_tc=250 - 97)
    # EdgeIndex refill (SURVEY 8f-1): the (k+1)-mer index of the pipeline and the counting path with a smaller K; B = 10 x 2 threads
    save("syn_k21_B20_eigraph", "eigraph", synthetic_reads(600, 100, 1500, 0.01, seed=5), 21, 20, edge_index=0)
    save("syn_k21_B20_K15_eigraph", "eigraph", synthetic_reads(600, 100, 1500, 0.01, seed=5), 21, 20, edge_index=15)
    save("loops_k21_B10_eigraph", "eigraph", loops_reads(), 21, 10, edge_index=0)
    save("ecoli_k55_B20_K33_eigraph", "eigraph", ec[:1200], 55, 20, edge_index=33)
    # every key width (K = 97: four words, K = 66: three), K = 128 through the (k+1)-mer path, K = 1 and 2 (every slot put many times)
    save("syn_k99_B20_K97_eigraph", "eigraph", synthetic_reads(250, 150, 1500, 0.01, seed=5), 99, 20, edge_index=97)
    save("syn_k127_B20_eigraph", "eigraph", synthetic_reads(400, 150, 1200, 0.005, seed=9), 127, 20, edge_index=0)
    save("syn_k21_B20_K1_eigraph", "eigraph", synthetic_reads(100, 100, 1000, 0.01, seed=10), 21, 20, edge_index=1)
    save("syn_k21_B20_K2_eigraph", "eigraph", synthetic_reads(100, 100, 1000, 0.01, seed=10), 21, 20, edge_index=2)
    # self-reverse-complementary K-mers: on ordinary edges (put from both strands: tombstones) and at the centre of self-conjugate
    # edges (visited once: a position)
    save("pal_k77_B20_K66_eigraph", "eigraph", pal_reads(33, 20, 10, 12, synthetic_reads(100, 150, 1500, 0.01, seed=11)), 77, 20, edge_index=66)
    save("pal_k21_B20_eigraph", "eigraph", pal_reads(11, 20, 30, 13), 21, 20, edge_index=0)
    # the (k+1)-mer path's branch rule: 16 vertices against 20 chunks (one segment, segment_starts_[1] = n), 20 (single index, 0)
    save("iso4_k21_B20_eigraph", "eigraph", isolated_reads(4, 14), 21, 20, edge_index=0)
    save("iso5_k21_B20_eigraph", "eigraph", isolated_reads(5, 15), 21, 20, edge_index=0)
    save("empty_k21_B20_eigraph", "eigraph", ["ACGTACGTAC", "GGGTTTAAACCC"], 21, 20, edge_index=0)
    for nm, (rd, _) in GTEST_CASES.items():
        save("gtest_" + nm + "_k5", "graph", rd, 5, 2)
    # construction_test.cpp:97-105 (SimpleTestEarlyPairedInfo, k=3): its coverage table is the known answer in tests/test_oracle_golden.py
    save("gtest_EarlyPairedInfo_k3", "graph", ["CCCAC", "CCACG", "ACCAC", "CCACA"], 3, 2)
    # coverage pre-filter (SURVEY 8f-3), thresholds 2..5, odd and even k+1 (self-RC windows exist only for even k+1)
    save_covfilter("cov_k21_t2_covfilter", covfilter_reads(31), 21, 2)
    save_covfilter("cov_k20_t3_covfilter", covfilter_reads(32), 20, 3)
    save_covfilter("cov_k55_t2_covfilter", covfilter_reads(33), 55, 2)
    save_covfilter("cov_k31_t5_covfilter", ecoli_reads()[:1500] + covfilter_reads(34)[:800], 31, 5)
