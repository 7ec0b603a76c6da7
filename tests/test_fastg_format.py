"""CPU checks of the FASTG / unitig FASTA formatter's pieces: the coverage text compiled for the host against printf's %f, and the
restatement the GPU tests compare with (fastg_oracle) against the reference's graphs in tests/golden."""
import ctypes as C

import numpy as np
import pytest

import fastg_oracle as F
import golden_util as G


def _lib():
    from spades_b200 import _lib
    return _lib.load()


def _host_cov(raw, den):
    raw = np.ascontiguousarray(raw, np.uint32)
    den = np.ascontiguousarray(den, np.uint32)
    out = np.zeros(max(len(raw), 1) * 32, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert _lib().sgpu_format_coverage(None, 0, p(raw), p(den), len(raw), p(out)) == 0
    return [bytes(r).split(b"\0")[0].decode() for r in out.reshape(-1, 32)[:len(raw)]]


def cov_cases(n, seed):
    """random (raw, len - k) pairs over the whole u32 range and near its small end, plus exact ties of the sixth digit"""
    rng = np.random.default_rng(seed)
    raw = np.concatenate([rng.integers(0, 1 << 32, n // 2, dtype=np.uint64), rng.integers(0, 1000, n - n // 2, dtype=np.uint64)])
    den = np.concatenate([rng.integers(1, 1 << 32, n // 4, dtype=np.uint64), rng.integers(1, 300, n - n // 4, dtype=np.uint64)])
    rng.shuffle(den)
    ties_raw = [1, 3, 5, 7, 1, 3, 9, 0xFFFFFFFF, 0xFFFFFFFF, 1, 0, 1, 0x80000000]
    ties_den = [128, 128, 128, 128, 256, 1024, 2048, 1, 0xFFFFFFFF, 0xFFFFFFFF, 7, 3, 1 << 20]
    raw = np.concatenate([raw, np.array(ties_raw, np.uint64)]).astype(np.uint32)
    den = np.concatenate([den, np.array(ties_den, np.uint64)]).astype(np.uint32)
    return raw, den


def test_cov_text_equals_printf():
    raw, den = cov_cases(1_000_000, 11)
    got = _host_cov(raw, den)
    want = [F.cov_text(int(r), int(d)) for r, d in zip(raw, den)]
    bad = [(int(raw[i]), int(den[i]), got[i], want[i]) for i in range(len(got)) if got[i] != want[i]]
    assert not bad, bad[:5]


def test_cov_text_ties():
    # halfway cases of the sixth digit round to even, as glibc's printf does
    assert _host_cov([1, 3, 5, 7], [128] * 4) == ["0.007812", "0.023438", "0.039062", "0.054688"]
    assert _host_cov([0, 10, 0xFFFFFFFF], [5, 4, 1]) == ["0.000000", "2.500000", "4294967295.000000"]


def test_cov_text_refuses_zero_divisor():
    raw = np.ones(1, np.uint32); den = np.zeros(1, np.uint32); out = np.zeros(32, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert _lib().sgpu_format_coverage(None, 0, p(raw), p(den), 1, p(out)) != 0


GRAPHS = [n for n in G.names() if "graph_gfa" in np.load(G.GOLDEN_DIR + "/" + n + ".npz").files]


@pytest.mark.parametrize("name", GRAPHS)
def test_oracle_fastg_structure(name):
    """on the reference's graphs: one record per strand of every edge (one for a self-conjugate edge), the text of the edge or of its
    reverse complement wrapped at 60, at most four distinct successors in byte order, and each successor starts where the record ends"""
    g = G.load(name)
    gfa, k = g["graph_gfa"].tobytes().decode(), g["k"]
    seqs = [l.split("\t")[2] for l in gfa.split("\n") if l.startswith("S\t")]
    text = F.fastg_from_gfa(gfa, k)
    recs = text.split(">")[1:]
    selfc = sum(s == F.revcomp(s) for s in seqs)
    assert len(recs) == 2 * len(seqs) - selfc
    by_name = {}
    for r in recs:
        head, body = r.split("\n", 1)
        assert head.endswith(";")
        own, _, nxt = head[:-1].partition(":")
        seq = body.replace("\n", "")
        assert body == F.wrapped(seq) and all(len(x) <= 60 for x in body.split("\n"))
        by_name[own] = (seq, nxt.split(",") if nxt else [])
    for own, (seq, nxt) in by_name.items():
        assert nxt == sorted(set(nxt)) and len(nxt) <= 4
        for x in nxt:
            assert by_name[x][0][:k] == seq[-k:]
    assert sorted(len(v[0]) for v in by_name.values()) == sorted([len(s) for s in seqs] + [len(s) for s in seqs if s != F.revcomp(s)])


def test_oracle_fastg_small_case():
    """a hand-checked graph: edge 3 is ACGTTT (k = 3), edge 5 its successor TTTGC; no edge is self-conjugate"""
    gfa = "H\tsp:Z:x\nS\t3\tACGTTT\tDP:f:2\tKC:i:6\nS\t5\tTTTGC\tDP:f:1\tKC:i:2\nL\t3\t+\t5\t+\t3M\n"
    want = (">EDGE_3_length_6_cov_2.000000:EDGE_5_length_5_cov_1.000000;\nACGTTT\n"
            ">EDGE_3_length_6_cov_2.000000';\nAAACGT\n"
            ">EDGE_5_length_5_cov_1.000000;\nTTTGC\n"
            ">EDGE_5_length_5_cov_1.000000':EDGE_3_length_6_cov_2.000000';\nGCAAA\n")
    assert F.fastg_from_gfa(gfa, 3) == want
    assert F.fastg_from_gfa(gfa, 3, with_coverage=False) == want.replace("2.000000", "0.000000").replace("1.000000", "0.000000")
    assert F.unitigs_fasta(["A" * 61, "CCGT"]) == ">EDGE_1_length_61\n" + "A" * 60 + "\nA\n>EDGE_2_length_4\nCCGT\n"


FASTG = G.names("fastg")


@pytest.mark.parametrize("name", FASTG)
def test_oracle_equals_reference_fastg(name):
    """the restatement over the oracle's graph of the fixture's reads is the text the reference's FastgWriter and gbuilder's unitig
    loop wrote: with coverage, without it, and the unitig FASTA"""
    import oracle as O
    g = G.load(name)
    r = O.full_graph(g["reads"], g["k"], g["B"], early_tc=g["tc_bound"])
    assert F.fastg_from_gfa(r["gfa"], g["k"]) == g["fastg"].tobytes().decode()
    assert F.fastg_from_gfa(r["gfa"], g["k"], with_coverage=False) == g["fastg_nocov"].tobytes().decode()
    assert F.unitigs_fasta(r["unitigs"].seqs) == g["unitigs_fasta"].tobytes().decode()
