"""Load tests/golden/*.npz (reference outputs) and compare an implementation's artefacts against them."""
import glob
import os
import struct

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def names(mode=None):
    out = []
    for p in sorted(glob.glob(os.path.join(GOLDEN_DIR, "*.npz"))):
        n = os.path.basename(p)[:-4]
        if mode is None or n.endswith("_" + mode) or (mode == "graph" and n.startswith("gtest_")):
            out.append(n)
    return out


def load(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    g = {k: z[k] for k in z.files}
    g["reads"] = g["reads"].tobytes().decode().split("\n")
    g["k"] = int(g["k"][0]); g["B"] = int(g["B"][0]) if "B" in g else 0; g["mode"] = g["mode"].tobytes().decode()
    if "tc_bound" in g:
        g["tc_bound"] = int(g["tc_bound"][0])
    for f in ("ei_k", "ei_chunks"):
        if f in g:
            g[f] = np.asarray(g[f])
    return g


def _txt_ints(a):
    s = a.tobytes().decode().split()
    return np.array([int(x) for x in s], dtype=np.int64)


def strip_uleb_k(ref_bytes, k):
    """IndexWrapper::BinWrite prefixes KMerIndex::serialize with ULEB128(k) (io/binary/binary.hpp:109-146)."""
    v, shift, i = 0, 0, 0
    while True:
        b = ref_bytes[i]; i += 1
        v |= (b & 0x7F) << shift; shift += 7
        if not (b & 0x80):
            break
    assert v == k
    return bytes(ref_bytes[i:])


def _empty_bucket_rank_fields(layout: bytes, nbuckets: int):
    """offsets of the 8-byte _lastbitsetrank field of every empty bucket in a KMerIndex::serialize output"""
    out = []
    p = 8
    for _ in range(nbuckets):
        n = struct.unpack_from("<Q", layout, p + 20)[0]
        if n == 0:
            out.append(p + 12)
        p += 28
        if n:
            for _l in range(25):
                _size, nchar = struct.unpack_from("<QQ", layout, p); p += 16 + 8 * nchar
                nr = struct.unpack_from("<Q", layout, p)[0]; p += 8 + 8 * nr
        p += 8
    return out


def index_equal(ref: bytes, mine: bytes, nbuckets: int):
    """Byte compare of KMerIndex::serialize output; the reference writes an UNINITIALISED _lastbitsetrank for
    empty buckets (BooPHF.h:514-517 with build() returning early at :426), so those 8 bytes are masked."""
    if len(ref) != len(mine):
        return False
    ref = bytearray(ref); mine = bytearray(mine)
    for q in _empty_bucket_rank_fields(mine, nbuckets):
        ref[q:q + 8] = b"\0" * 8
        mine[q:q + 8] = b"\0" * 8
    return ref == mine


def index_canonical(b: bytes, nbuckets: int):
    """KMerIndex::serialize output with the rank field of empty buckets zeroed (see index_equal): equal canonical forms
    <=> index_equal"""
    b = bytearray(b)
    for q in _empty_bucket_rank_fields(b, nbuckets):
        b[q:q + 8] = b"\0" * 8
    return bytes(b)


def check_graph(g, art):
    """art: dict with kpomers,kp_bsz,kmers,kmer_index,kpomer_index,masks,cov,hist,unitigs,gfa (any subset)."""
    k, B = g["k"], g["B"]
    bad = []
    def chk(name, ok):
        if not ok:
            bad.append(name)
    if "kpomers" in art:
        chk("kpomers", np.array_equal(np.frombuffer(g["kpomers"].tobytes(), np.uint64), np.asarray(art["kpomers"], np.uint64).ravel()))
    if "kp_bsz" in art:
        chk("kp_bsz", np.array_equal(_txt_ints(g["kpomer_bucket_sizes_txt"]), np.asarray(art["kp_bsz"], np.int64)))
    if "kp_counts_sorted" in art:
        pass
    if "kmers" in art:
        chk("kmers", np.array_equal(np.frombuffer(g["kmers"].tobytes(), np.uint64), np.asarray(art["kmers"], np.uint64).ravel()))
    if "kmer_index" in art:
        chk("kmer_index", index_equal(strip_uleb_k(g["kmer_index_bin"].tobytes(), k), art["kmer_index"], B))
    if "kpomer_index" in art:
        chk("kpomer_index", index_equal(strip_uleb_k(g["kpomer_index_bin"].tobytes(), k + 1), art["kpomer_index"], B))
    if "masks" in art:     # clipper fixtures: `masks` is the array after the last clipper that ran (masks_tc.bin, else masks_at.bin)
        want = g["masks_tc_bin"] if "masks_tc_bin" in g else (g["masks_at_bin"] if "masks_at_bin" in g else g["masks_bin"])
        chk("masks", np.array_equal(want, np.asarray(art["masks"], np.uint8)))
    if "at_removed" in art:    # (RemoveATEdges' return value, RemoveATTips' return value)
        chk("at_removed", [int(x) for x in g["at_removed_txt"].tobytes().decode().split()] == [int(x) for x in art["at_removed"]])
    if "masks_raw" in art and "masks_tc_bin" in g:
        chk("masks_raw", np.array_equal(g["masks_bin"], np.asarray(art["masks_raw"], np.uint8)))
    if "tc_removed" in art:
        chk("tc_removed", int(g["tc_removed_txt"].tobytes().decode().split()[0]) == int(art["tc_removed"]))
    if "cov" in art:
        chk("cov", np.array_equal(np.frombuffer(g["coverage_bin"].tobytes(), np.uint32), np.asarray(art["cov"], np.uint32)))
    if "hist" in art:
        chk("hist", np.array_equal(_txt_ints(g["histogram_txt"]), np.asarray(art["hist"], np.int64)))
    if "unitigs" in art:
        chk("unitigs", g["unitigs_txt"].tobytes().decode().split() == list(art["unitigs"]))
    if "gfa" in art:
        chk("gfa", g["graph_gfa"].tobytes().decode() == art["gfa"])
    return bad


def check_edge_index(g, ei_bytes, ids, offs, nbuckets):
    """EdgeIndex fixtures: edge_index.bin = ULEB(K) + KMerIndex::serialize, edge_index_values.bin = per slot {u64 edge id, u32 offset}"""
    bad = []
    K = int(g["ei_k"][0])
    if not index_equal(strip_uleb_k(g["edge_index_bin"].tobytes(), K), ei_bytes, nbuckets):
        bad.append("edge_index")
    v = g["edge_index_values_bin"].reshape(-1, 12)
    want_ids = v[:, :8].copy().view(np.uint64).ravel(); want_off = v[:, 8:].copy().view(np.uint32).ravel()
    if not np.array_equal(want_ids, np.asarray(ids, np.uint64)):
        bad.append("edge_ids")
    if not np.array_equal(want_off, np.asarray(offs, np.uint32)):
        bad.append("edge_offsets")
    return bad


def edge_index_single(unitigs, k, chunks):
    """the (k+1)-mer path's branch: with more than one vertex chunk and at least as many vertices as chunks KMerIndexBuilder takes its
    single-index branch, which never fills segment_starts_[1] (kmer_index_builder.hpp:481-493); with fewer vertices the graph is one
    chunk and the segmented branch stores n there. Vertices = the distinct canonical ends of the edges, each with its conjugate."""
    from spades_b200.packing import revcomp
    ends = set()
    for s in unitigs:
        for v in (s[:k], s[-k:]):
            ends.add(min(v, revcomp(v)))
    return chunks > 1 and 2 * len(ends) >= chunks


def edge_index_bytes(mphf, unitigs, k, K, chunks):
    """the oracle MPHF's KMerIndex::serialize as the EdgeIndex refill writes it: K = k+1 over `chunks` vertex chunks leaves
    segment_starts_[1] = 0 in the single-index branch (edge_index_single); the oracle's one segment stores n there"""
    ser = mphf.serialize()
    if K == k + 1 and edge_index_single(unitigs, k, chunks):
        ser = ser[:-8] + b"\0" * 8
    return ser


def check_count(g, art):
    bad = []
    if not np.array_equal(np.frombuffer(g["final_kmers"].tobytes(), np.uint64), np.asarray(art["final_kmers"], np.uint64).ravel()):
        bad.append("final_kmers")
    if not np.array_equal(_txt_ints(g["bucket_sizes_txt"]), np.asarray(art["bsz"], np.int64)):
        bad.append("bucket_sizes")
    return bad
