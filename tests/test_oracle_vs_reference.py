"""CPU test: the C oracle against what the UNMODIFIED reference (oracle/_ref/ref_probe) produced on seeded inputs.

The reference's artefacts for every case below were recorded by running the probe on these same inputs
(`python tests/test_oracle_vs_reference.py`, which needs oracle/_ref/ref_probe) and are stored in
tests/golden/oracle_vs_reference.json as SHA-256 digests of the bytes the comparison looks at (the artefacts
themselves are several MB per case). The digests are taken over the same canonical form golden_util compares:
the k-mer arrays as u64 words, bucket sizes as int64, KMerIndex bytes without the ULEB(k) prefix and with the
uninitialised rank field of empty buckets zeroed, and so on."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))

import golden_util as G  # noqa: E402
import oracle as O  # noqa: E402
from spades_b200.packing import synthetic_reads  # noqa: E402
from make_golden import at_reads, loops_reads  # noqa: E402
from test_oracle_golden import oracle_artifacts  # noqa: E402

PROBE = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "ref_probe")
RECORD = os.path.join(G.GOLDEN_DIR, "oracle_vs_reference.json")

GRAPH_CASES = [(21, 16, 11), (31, 5, 12), (55, 30, 13), (63, 9, 14), (77, 4, 15), (127, 6, 16)]
COUNT_CASES = [(21, 16, 21), (55, 16, 22), (100, 3, 23)]
TC_CASES = [(21, 16, 3000, 100, 4000, 0.01, 41, 1), (21, 8, 3000, 100, 2000, 0.03, 42, 8), (55, 30, 3000, 150, 5000, 0.01, 43, 3),
            (77, 4, 1500, 150, 2000, 0.01, 44, 8), (9, 3, 1000, 60, 600, 0.1, 45, 8),
            (99, 7, 600, 250, 3000, 0.005, 46, 1), (127, 5, 600, 250, 3000, 0.005, 47, 8)]      # four-word k-mers, 250-bp reads
# keep_perfect_loops = false: (k, B, seed, T) over the loop and hairpin circles plus synthetic reads
NL_CASES = [(21, 9, 61, 3), (127, 4, 62, 8)]
# the A/T clipper at non-default (ratio, min_length, max_length), then the tip clipper: (k, B, n, L, glen, err, seed, T, at_params)
AT_CASES = [(33, 6, 1200, 150, 1500, 0.01, 71, 8, (0.7, 20, 60))]
COV_CASES = [(21, 2, 51, 1), (20, 3, 52, 8), (55, 2, 53, 3), (63, 4, 54, 8), (69, 2, 55, 2), (127, 3, 56, 8), (11, 6, 57, 8)]


def _sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def run_probe(mode, reads, k, B, T=3, early_tc=0, at_params=None, no_loops=False):
    with tempfile.TemporaryDirectory() as d:
        rf = os.path.join(d, "reads.txt")
        open(rf, "w").write("\n".join(reads) + "\n")
        out = os.path.join(d, "out")
        env = dict(os.environ)
        if early_tc:
            env["PROBE_EARLY_TC"] = str(early_tc)
        if at_params is not None:
            env["PROBE_EARLY_AT"] = "%r,%d,%d" % tuple(at_params)
        if no_loops:
            env["PROBE_NO_LOOPS"] = "1"
        subprocess.check_call([PROBE, mode, rf, str(k), str(B), str(T), out], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=env, timeout=600)
        g = {f.replace(".", "_"): np.frombuffer(open(os.path.join(out, f), "rb").read(), np.uint8)
             for f in os.listdir(out) if os.path.isfile(os.path.join(out, f))}
    g.update(k=k, B=B, reads=reads)
    return g


def graph_digests_of_reference(g, keys):
    """SHA-256 of each artefact of a ref_probe graph run, in the form golden_util.check_graph compares (only `keys`)"""
    k, B = g["k"], g["B"]
    masks = g["masks_tc_bin"] if "masks_tc_bin" in g else (g["masks_at_bin"] if "masks_at_bin" in g else g["masks_bin"])
    canon = {"kpomers": lambda: g["kpomers"].tobytes(), "kp_bsz": lambda: G._txt_ints(g["kpomer_bucket_sizes_txt"]).tobytes(),
             "kmers": lambda: g["kmers"].tobytes(), "kmer_index": lambda: G.index_canonical(G.strip_uleb_k(g["kmer_index_bin"].tobytes(), k), B),
             "kpomer_index": lambda: G.index_canonical(G.strip_uleb_k(g["kpomer_index_bin"].tobytes(), k + 1), B),
             "masks": lambda: masks.tobytes(), "masks_raw": lambda: g["masks_bin"].tobytes(),
             "tc_removed": lambda: str(int(g["tc_removed_txt"].tobytes().decode().split()[0])).encode(),
             "at_removed": lambda: " ".join(g["at_removed_txt"].tobytes().decode().split()).encode(),
             "cov": lambda: g["coverage_bin"].tobytes(), "hist": lambda: G._txt_ints(g["histogram_txt"]).tobytes(),
             "unitigs": lambda: "\n".join(g["unitigs_txt"].tobytes().decode().split()).encode(), "gfa": lambda: g["graph_gfa"].tobytes()}
    return {key: _sha(canon[key]()) for key in keys}


def graph_digests_of(art, B):
    canon = {"kpomers": lambda v: np.asarray(v, np.uint64).ravel().tobytes(), "kp_bsz": lambda v: np.asarray(v, np.int64).tobytes(),
             "kmers": lambda v: np.asarray(v, np.uint64).ravel().tobytes(), "kmer_index": lambda v: G.index_canonical(v, B),
             "kpomer_index": lambda v: G.index_canonical(v, B), "masks": lambda v: np.asarray(v, np.uint8).tobytes(),
             "masks_raw": lambda v: np.asarray(v, np.uint8).tobytes(), "tc_removed": lambda v: str(int(v)).encode(),
             "at_removed": lambda v: " ".join(str(int(x)) for x in v).encode(),
             "cov": lambda v: np.asarray(v, np.uint32).tobytes(), "hist": lambda v: np.asarray(v, np.int64).tobytes(),
             "unitigs": lambda v: "\n".join(v).encode(), "gfa": lambda v: v.encode()}
    return {key: _sha(canon[key](v)) for key, v in art.items()}


def count_digests_of(final_kmers, bsz):
    return {"final_kmers": _sha(np.asarray(final_kmers, np.uint64).ravel().tobytes()), "bucket_sizes": _sha(np.asarray(bsz, np.int64).tobytes())}


def _graph_id(k, B, seed):
    return "graph_k%d_B%d_s%d" % (k, B, seed)


def _tc_id(k, B, n, L, glen, err, seed, T):
    return "tc_k%d_B%d_n%d_L%d_g%d_e%g_s%d_T%d" % (k, B, n, L, glen, err, seed, T)


def _tc_reads(n, L, glen, err, seed):
    return synthetic_reads(n, L, glen, err, seed=seed)


def _nl_id(k, B, seed, T):
    return "nl_k%d_B%d_s%d_T%d" % (k, B, seed, T)


def _nl_reads(seed):
    return loops_reads(250, 250) + synthetic_reads(400, 250, 1500, 0.002, seed=seed)


def _at_id(k, B, n, L, glen, err, seed, T, at_params):
    return "at_k%d_B%d_n%d_L%d_g%d_e%g_s%d_T%d_r%g_min%d_max%d" % ((k, B, n, L, glen, err, seed, T) + tuple(at_params))


def _cov_reads(seed):
    from spades_b200.packing import revcomp
    rng = np.random.default_rng(seed)
    reads = synthetic_reads(2500, 150, 4000, 0.01, seed=seed) + synthetic_reads(400, 150, 40000, 0.02, seed=seed + 1)
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 90))
    reads += [x + revcomp(x)] * 3 + ["A" * 150, "AC" * 70, "ACGTACGT"]
    return reads


def _recorded(case):
    return json.load(open(RECORD))[case]


@pytest.mark.parametrize("k,B,seed", GRAPH_CASES)
def test_oracle_vs_live_reference_graph(k, B, seed):
    reads = synthetic_reads(1500, 150, 3000, 0.01, seed=seed)
    art, _ = oracle_artifacts(reads, k, B)
    want = _recorded(_graph_id(k, B, seed))
    got = graph_digests_of(art, B)
    assert sorted(want) == sorted(got)
    assert [key for key in want if want[key] != got[key]] == []


@pytest.mark.parametrize("k,B,seed", COUNT_CASES)
def test_oracle_vs_live_reference_kmercount(k, B, seed):
    from spades_b200.packing import pack_reads
    reads = synthetic_reads(800, 150, 2000, 0.01, seed=seed)
    words, offs, lens = pack_reads(reads)
    ks = O.count(words, offs, lens, k, B, 1)
    assert count_digests_of(ks.keys, ks.bsz) == _recorded("count_k%d_B%d_s%d" % (k, B, seed))


@pytest.mark.parametrize("k,B,n,L,glen,err,seed,T", TC_CASES)
def test_oracle_vs_live_reference_early_tip_clipper(k, B, n, L, glen, err, seed, T):
    """the reference's clipper runs racily on T threads; its result (and the oracle's) must not depend on T"""
    art, r = oracle_artifacts(_tc_reads(n, L, glen, err, seed), k, B, early_tc=L - k)
    want = _recorded(_tc_id(k, B, n, L, glen, err, seed, T))
    got = graph_digests_of(art, B)
    assert sorted(want) == sorted(got)
    assert [key for key in want if want[key] != got[key]] == []
    assert r["tc"]["removed"] > 0


@pytest.mark.parametrize("k,B,seed,T", NL_CASES)
def test_oracle_vs_live_reference_no_loops(k, B, seed, T):
    """keep_perfect_loops = false: the unbranching paths of the reference's ExtractUnbranchingPaths, without the loops"""
    reads = _nl_reads(seed)
    art, r = oracle_artifacts(reads, k, B, keep_loops=False)
    want = _recorded(_nl_id(k, B, seed, T))
    got = graph_digests_of(art, B)
    assert sorted(want) == sorted(got)
    assert [key for key in want if want[key] != got[key]] == []
    assert len(O.full_graph(reads, k, B)["unitigs"].seqs) > len(r["unitigs"].seqs)


@pytest.mark.parametrize("k,B,n,L,glen,err,seed,T,at_params", AT_CASES)
def test_oracle_vs_live_reference_early_at_clipper_parameters(k, B, n, L, glen, err, seed, T, at_params):
    """EarlyLowComplexityClipperProcessor constructed with non-default ratio, min_length and max_length, then the tip clipper; the
    parameters change the result against the pipeline's (0.8, 10, 200)"""
    reads = at_reads(n, L, glen, err, seed)
    art, r = oracle_artifacts(reads, k, B, early_tc=L - k, early_at=True, at_params=at_params)
    want = _recorded(_at_id(k, B, n, L, glen, err, seed, T, at_params))
    got = graph_digests_of(art, B)
    assert sorted(want) == sorted(got)
    assert [key for key in want if want[key] != got[key]] == []
    assert r["at"][2] > 0 and r["at"] != O.full_graph(reads, k, B, early_tc=L - k, early_at=True)["at"]


@pytest.mark.parametrize("k,thr,seed,T", COV_CASES)
def test_oracle_vs_live_reference_coverage_prefilter(k, thr, seed, T):
    """SURVEY 8f-3: the CoverageFilter phase of the unmodified reference (HLL bound -> qf::cqf -> median filter, filled by T racing
    threads) against the oracle's restatement: the cardinality bound, the key width, the verdict for every read and the rolling hash
    itself, for k+1 below, at and above 64 (rotation by (k+1) mod 64)"""
    from spades_b200.packing import pack_reads
    reads = _cov_reads(seed)
    want = _recorded("cov_k%d_t%d_s%d_T%d" % (k, thr, seed, T))
    words, offs, lens = pack_reads(reads)
    keep, st = O.cov_filter(words, offs, lens, k + 1, thr)
    assert st[0] == want["card"] and st[1] == want["key_bits"] and (1 << st[1]) - 1 == want["range_mask"]
    assert _sha(np.asarray(keep, np.uint8).tobytes()) == want["keep"]
    hh = [O.cyclic_hash(words[int(offs[i]):], j, k + 1) for i in range(64) for j in range(max(0, len(reads[i]) - k))]
    assert _sha(np.array(hh, dtype=np.uint64).tobytes()) == want["hashes"]


def record():
    """runs the reference on every case above and writes RECORD"""
    graph_keys = ["kpomers", "kp_bsz", "kmers", "kmer_index", "kpomer_index", "masks", "cov", "hist", "unitigs", "gfa"]
    out = {}
    for k, B, seed in GRAPH_CASES:
        g = run_probe("graph", synthetic_reads(1500, 150, 3000, 0.01, seed=seed), k, B)
        out[_graph_id(k, B, seed)] = graph_digests_of_reference(g, graph_keys)
    for k, B, seed in COUNT_CASES:
        g = run_probe("count", synthetic_reads(800, 150, 2000, 0.01, seed=seed), k, B)
        out["count_k%d_B%d_s%d" % (k, B, seed)] = {"final_kmers": _sha(g["final_kmers"].tobytes()),
                                                   "bucket_sizes": _sha(G._txt_ints(g["bucket_sizes_txt"]).tobytes())}
    for c in TC_CASES:
        k, B, n, L, glen, err, seed, T = c
        g = run_probe("graph", _tc_reads(n, L, glen, err, seed), k, B, T=T, early_tc=L - k)
        out[_tc_id(*c)] = graph_digests_of_reference(g, graph_keys + ["tc_removed", "masks_raw"])
    for k, B, seed, T in NL_CASES:
        g = run_probe("graph", _nl_reads(seed), k, B, T=T, no_loops=True)
        out[_nl_id(k, B, seed, T)] = graph_digests_of_reference(g, graph_keys)
    for c in AT_CASES:
        k, B, n, L, glen, err, seed, T, at_params = c
        g = run_probe("graph", at_reads(n, L, glen, err, seed), k, B, T=T, early_tc=L - k, at_params=at_params)
        out[_at_id(*c)] = graph_digests_of_reference(g, graph_keys + ["tc_removed", "at_removed"])
    for k, thr, seed, T in COV_CASES:
        with tempfile.TemporaryDirectory() as d:
            rf = os.path.join(d, "reads.txt")
            open(rf, "w").write("\n".join(_cov_reads(seed)) + "\n")
            env = dict(os.environ); env["PROBE_COV_THR"] = str(thr)
            subprocess.check_call([PROBE, "covfilter", rf, str(k), "4", str(T), os.path.join(d, "out")], stdout=subprocess.DEVNULL,
                                  stderr=subprocess.DEVNULL, env=env, timeout=600)
            card, bits, mask, _ = [int(v) for v in open(os.path.join(d, "out", "covfilter.txt")).read().split()]
            keep = np.array([int(v) for v in open(os.path.join(d, "out", "keep.txt")).read().split()], dtype=np.uint8)
            hashes = np.fromfile(os.path.join(d, "out", "hashes.bin"), dtype=np.uint64)
        out["cov_k%d_t%d_s%d_T%d" % (k, thr, seed, T)] = {"card": card, "key_bits": bits, "range_mask": mask, "keep": _sha(keep.tobytes()),
                                                          "hashes": _sha(hashes.tobytes())}
    json.dump(out, open(RECORD, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    record()
