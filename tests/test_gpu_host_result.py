"""GPU: counts whose result goes to pinned host memory (SGPU_RESULT_ON_HOST), run with -m gpu on an H100.

A host set must answer every accessor and the MPHF build exactly as a device set of the same reads does, and both must equal the
C oracle. The budgeted contexts of test_gpu_multipass split every count into several passes, so the copy of one pass's chunk runs
behind the next pass and the index is built from many chunks."""
import ctypes as C
import gc
import os
import socket
import subprocess
import tempfile

import numpy as np
import pytest

import golden_util as G
import oracle as O
from spades_b200.packing import pack_reads, revcomp, synthetic_reads
from test_gpu_multipass import MAX_CHUNKS, MIN_BUDGET, _budgeted, _graph_path, _tiny_reads
from test_gpu_parity import _compare, _oracle_art

pytestmark = pytest.mark.gpu

CANON, ALLWIN = 0, 1
SGPU_EUNSUPPORTED = 7
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _splitter(K, mode):
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, ParallelSortingSplitter
    return DeBruijnReadKMerSplitter(K) if mode == CANON else ParallelSortingSplitter(K)


def _count(c, K, B, mode, on_host):
    from spades_b200.kmer_index import KMerDiskCounter
    st = KMerDiskCounter(c, _splitter(K, mode), result_on_host=on_host).Count(B)
    return st, c.times()


def _artefacts(c, st, mode, tmp, tag):
    """everything a client can read from a set: records, multiplicities, bucket sizes, checksum, bucket files, final_kmers, the
    serialized index and the slot of every key"""
    from spades_b200.kmer_index import KMerIndexBuilder
    keys = st.kmers()
    art = dict(keys=keys, bsz=st.bucket_sizes(), checksum=st.checksum(), on_host=st.on_host())
    art["counts"] = st.counts() if mode == CANON else None
    st.write_buckets(os.path.join(tmp, tag + "_kmers"))
    st.merge(os.path.join(tmp, tag + "_final"))
    art["buckets"] = [open(os.path.join(tmp, "%s_kmers.%d" % (tag, b)), "rb").read() for b in range(st.num_buckets())]
    art["final"] = open(os.path.join(tmp, tag + "_final"), "rb").read()
    idx = KMerIndexBuilder(c).BuildIndex(st)
    try:
        art["index"] = idx.serialize()
        art["slots"] = idx.seq_idx(keys)
    finally:
        idx.free()
    return art


def _host_and_device(reads, K, B, mode, budget=MIN_BUDGET):
    """one budgeted context: the device-set count and the host-set count of the same reads, with their artefacts and times"""
    with tempfile.TemporaryDirectory() as tmp, _budgeted(budget) as c:
        c.set_reads(*pack_reads(reads))
        out = {}
        for on_host in (False, True):
            st, t = _count(c, K, B, mode, on_host)
            try:
                out[on_host] = (_artefacts(c, st, mode, tmp, "h" if on_host else "d"), t, st.total_kmers())
            finally:
                st.free()
    return out


def _check_pair(got, reads, K, B, mode, want_passes_above=1):
    words, offs, lens = pack_reads(reads)
    ks = O.count(words, offs, lens, K, B, mode)
    (dev, tdev, ndev), (host, thost, nhost) = got[False], got[True]
    assert not dev["on_host"] and host["on_host"]
    assert nhost == ndev == ks.n
    assert tdev["passes"] > want_passes_above and thost["passes"] > want_passes_above, (tdev["passes"], thost["passes"])
    assert tdev["result_d2h_bytes"] == 0
    W = 8 * ks.nw
    assert thost["result_d2h_bytes"] == ks.n * (W + 4 if mode == CANON else W)
    # the oracle
    assert np.array_equal(host["keys"].ravel(), ks.keys.ravel()) and np.array_equal(host["bsz"], ks.bsz)
    if mode == CANON:
        assert np.array_equal(host["counts"], ks.counts)
    assert G.index_equal(O.Mphf(ks).serialize(), host["index"], B)
    # the device set, byte for byte
    for key in ("keys", "bsz", "counts", "slots"):
        a, b = host[key], dev[key]
        assert (a is None and b is None) or np.array_equal(a, b), key
    assert host["checksum"] == dev["checksum"]
    assert host["buckets"] == dev["buckets"] and host["final"] == dev["final"]
    assert host["index"] == dev["index"]
    if ks.n:
        assert np.array_equal(np.sort(host["slots"]), np.arange(ks.n, dtype=np.uint64))


# K = 21, 55, 56, 78, 128: 1 to 4 words per record; canonical and all-windows
PARITY = [(21, 12, CANON), (55, 16, CANON), (56, 10, CANON), (78, 12, CANON), (128, 11, CANON),
          (21, 12, ALLWIN), (56, 10, ALLWIN), (97, 9, ALLWIN)]


@pytest.mark.parametrize("K,B,mode", PARITY)
def test_host_set_equals_oracle_and_device_set(K, B, mode):
    reads = synthetic_reads(3000, 150, 3000, 0.004 if K > 100 else 0.01, seed=300 + K)
    _check_pair(_host_and_device(reads, K, B, mode), reads, K, B, mode)


def test_capacity_result_three_times_the_budget():
    """one read set and one 1 GiB budget, with a result of 3.2 GB (3x the budget) in 128 buckets, each of which fits the budget alone:
    the device-set count keeps every chunk and peaks above the budget through driver allocations; the host-result count keeps
    its peak within the budget and copies exactly n x (W + 4) bytes to the host"""
    budget = 1 << 30
    K, B, W = 21, 128, 8
    # 2.6 M random 128 bp reads, each listed twice (the copy shares the words): every canonical 21-mer occurs twice, so
    # distinct / instances = 1/2, within the planner's assumption of at most 0.6
    rng = np.random.default_rng(700)
    nu = 2_600_000
    words = rng.integers(0, np.iinfo(np.uint64).max, size=nu * 4, dtype=np.uint64, endpoint=True)
    offs = np.tile(np.arange(nu, dtype=np.uint64) * np.uint64(4), 2)
    lens = np.full(2 * nu, 128, np.uint32)
    res = {}
    for on_host in (True, False):          # host first: peak_bytes is the peak of the context's lifetime
        with _budgeted(budget) as c:
            c.set_reads(words, offs, lens)
            st, t = _count(c, K, B, CANON, on_host)
            try:
                res[on_host] = dict(n=st.total_kmers(), bsz=st.bucket_sizes(), checksum=st.checksum(), peak=t["peak_bytes"],
                                    passes=t["passes"], d2h=t["result_d2h_bytes"], wait=t["result_d2h_wait_ms"], host=st.on_host())
            finally:
                st.free()
        gc.collect()
    h, d = res[True], res[False]
    n = h["n"]
    assert n == d["n"] and n * (W + 4) >= 3 * budget
    assert int(h["bsz"].max()) * (3 * W + 4) < budget // 2                 # a bucket's pass fits the budget alone
    assert h["host"] and not d["host"]
    assert d["peak"] > budget, d
    assert h["peak"] <= budget, h
    assert h["d2h"] == n * (W + 4) and h["passes"] > 1 and h["passes"] <= MAX_CHUNKS
    assert np.array_equal(h["bsz"], d["bsz"]) and h["checksum"] == d["checksum"]
    print("capacity: n=%d result=%.2f GB budget=%.2f GB host peak=%.3f GB (%d passes, %.0f ms waiting on copies) device peak=%.2f GB (%d passes)"
          % (n, n * (W + 4) / 1e9, budget / 1e9, h["peak"] / 1e9, h["passes"], h["wait"], d["peak"] / 1e9, d["passes"]))


def test_empty_read_set():
    reads = ["ACGTACG", "TTG"]             # shorter than K: no k-mer at all
    got = _host_and_device(reads, 21, 8, CANON)
    host, dev = got[True][0], got[False][0]
    assert got[True][2] == 0 and host["on_host"]
    assert host["checksum"] == dev["checksum"] == [0, 0, 0, 0]
    assert host["index"] == dev["index"] and host["final"] == dev["final"] == b""
    assert got[True][1]["result_d2h_bytes"] == 0


def test_one_bucket():
    reads = synthetic_reads(3000, 150, 3000, 0.01, seed=301)
    _check_pair(_host_and_device(reads, 55, 1, CANON), reads, 55, 1, CANON, want_passes_above=0)


def test_full_chunk_table():
    """300 buckets at the 64 MiB budget: the planner fills the chunk table (at most 128 passes, so at most 128 chunks)"""
    reads = _tiny_reads(400, 43)
    got = _host_and_device(reads, 22, 300, CANON)
    assert got[True][1]["passes"] <= MAX_CHUNKS
    _check_pair(got, reads, 22, 300, CANON)


def test_self_reverse_complement_heavy_even_k():
    """palindromic reads x + revcomp(x): at K = 56 the centred window is its own reverse complement (counted twice per read)"""
    rng = np.random.default_rng(302)
    pal = []
    for _ in range(200):
        x = "".join("ACGT"[i] for i in rng.integers(0, 4, 60))
        pal += [x + revcomp(x)] * 3
    reads = pal + synthetic_reads(1000, 150, 2000, 0.01, seed=302)
    _check_pair(_host_and_device(reads, 56, 8, CANON), reads, 56, 8, CANON)


def test_ranged_downloads_across_every_chunk_boundary():
    from spades_b200.kmer_index import SpadesGpuError
    K, B = 33, 12
    words, offs, lens = pack_reads(synthetic_reads(3000, 150, 3000, 0.01, seed=303))
    ks = O.count(words, offs, lens, K, B, CANON)
    bstart = np.concatenate([[0], np.cumsum(ks.bsz)]).astype(np.int64)
    n = int(ks.n)
    with _budgeted(MIN_BUDGET) as c:
        c.set_reads(words, offs, lens)
        st, t = _count(c, K, B, CANON, True)
        try:
            assert st.on_host() and t["passes"] == B
            ranges = [(0, n), (n, 0), (0, 0)]
            for e in bstart[1:-1]:
                e = int(e)
                ranges += [(max(0, e - 5), min(e, 5)), (e, min(5, n - e)), (max(0, e - 3), min(7, n - max(0, e - 3))), (e, 0),
                           (max(0, e - 1000), min(n, e + 1000) - max(0, e - 1000))]
            got = [(f, m, st.kmers(f, m), st.counts(f, m)) for f, m in ranges]
            errors = []
            for f, m in ((n - 1, 2), (n + 1, 0), (0, n + 1), (-1, 1)):
                for get in (st.kmers, st.counts):
                    try:
                        get(f, m)
                        errors.append(False)
                    except SpadesGpuError:
                        errors.append(True)
        finally:
            st.free()
    for f, m, gk, gc_ in got:
        assert gk.shape == (m, ks.nw) and np.array_equal(gk, ks.keys[f:f + m]), (f, m)
        assert np.array_equal(gc_, ks.counts[f:f + m]), (f, m)
    assert all(errors), errors


@pytest.mark.parametrize("order", ["context_first", "set_first"])
def test_free_order(order):
    """the context torn down before its host set (deferred teardown: the set stays readable), or the set freed first"""
    from spades_b200.kmer_index import Context, KMerIndexBuilder
    import gpu_util
    K, B = 55, 8
    words, offs, lens = pack_reads(synthetic_reads(2000, 150, 2000, 0.01, seed=304))
    ks = O.count(words, offs, lens, K, B, CANON)
    gpu_util.release()
    c = Context(0, hbm_budget_bytes=MIN_BUDGET)
    c.set_reads(words, offs, lens)
    st, _ = _count(c, K, B, CANON, True)
    idx = KMerIndexBuilder(c).BuildIndex(st)
    if order == "context_first":
        c.close()
        keys, counts, cs, ser = st.kmers(), st.counts(), st.checksum(), idx.serialize()
        idx.free()
        st.free()
    else:
        keys, counts, cs, ser = st.kmers(), st.counts(), st.checksum(), idx.serialize()
        st.free()
        idx.free()
        c.close()
    assert np.array_equal(keys, ks.keys) and np.array_equal(counts, ks.counts)
    assert G.index_equal(O.Mphf(ks).serialize(), ser, B)
    assert cs[0] == ks.n and cs[3] == int(ks.counts.astype(np.uint64).sum())


def test_graph_calls_refuse_host_sets():
    """a host (k+1)-mer set: the k-mers of the (k+1)-mers and every graph build return SGPU_EUNSUPPORTED, leave nothing behind,
    and a device-set graph build in the same context still equals the oracle"""
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.kmer_index import DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    k, B = 21, 12
    reads = synthetic_reads(2000, 150, 2000, 0.01, seed=305)
    want = _oracle_art(reads, k, B)
    with _budgeted(MIN_BUDGET) as c:
        c.set_reads(*pack_reads(reads))
        kp_dev = KMerDiskCounter(c, DeBruijnReadKMerSplitter(k + 1)).Count(B)
        kp_host = KMerDiskCounter(c, DeBruijnReadKMerSplitter(k + 1), result_on_host=True).Count(B)
        km = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(k, kp_dev)).Count(B)
        mk = KMerIndexBuilder(c).BuildIndex(km)
        mkp = KMerIndexBuilder(c).BuildIndex(kp_host)
        allocated_before = c.times()["cached_bytes"]
        h = C.c_void_p()
        rcs = [c.L.sgpu_kmers_from_kpomers(c.h, kp_host.h, B, C.byref(h))]
        assert not h.value
        msg = c.L.sgpu_last_error(c.h).decode()
        opts = SgpuGraphOptions(1, 0, 0, 0.8, 10, 200)
        rcs.append(c.L.sgpu_graph_build_opts(c.h, kp_host.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h)))
        assert not h.value
        rcs.append(c.L.sgpu_graph_build(c.h, kp_host.h, km.h, mk.h, mkp.h, 1, C.byref(h)))
        assert not h.value
        rcs.append(c.L.sgpu_graph_build_ex(c.h, kp_host.h, km.h, mk.h, None, 1, 0, C.byref(h)))
        assert not h.value
        graph_msg = c.L.sgpu_last_error(c.h).decode()
        assert c.times()["cached_bytes"] == allocated_before
        for o in (mkp, mk, km, kp_host, kp_dev):
            o.free()
        art, passes, _, _, _, _ = _graph_path(c, reads, k, B, want)
    assert rcs == [SGPU_EUNSUPPORTED] * 4, rcs
    assert "host memory" in msg and "host memory" in graph_msg
    assert passes == (B, B)
    assert _compare(art, want, B) == []


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_distributed_host_result(world, tmp_path):
    """W ranks on device 0 over gloo, each rank's set in host memory, forced multi-pass budgets: every rank's set against the
    oracle's count of the union, and the summed checksums against a single-GPU count of the union"""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_worker import ARENA_BYTES
    from host_result_worker import CASES, run_spawned
    gpu_util.release()
    gc.collect()
    free, _ = torch.cuda.mem_get_info(0)
    need = world * (ARENA_BYTES + (3 << 29))
    if free < need:
        pytest.skip("device 0 has %.2f GiB free; %d ranks need %.2f GiB" % (free / 2**30, world, need / 2**30))
    out = tmp_path / "lines.txt"
    mp.spawn(run_spawned, args=(world, _free_port(), str(out)), nprocs=world, join=True)
    lines = out.read_text().splitlines()
    if lines and lines[0].startswith("SKIP"):
        pytest.skip(lines[0][5:])
    assert len(lines) == len(CASES), lines
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


TOOL = os.path.join(ROOT, "integration", "_build", "spades_kmercount_gpu")


@pytest.mark.skipif(not os.path.exists(TOOL), reason="integration/_build/spades_kmercount_gpu not built (needs the reference sources)")
@pytest.mark.parametrize("name", G.names("count"))
def test_kmercount_tool_host_result(name):
    g = G.load(name)
    with tempfile.TemporaryDirectory() as d:
        rf = os.path.join(d, "reads.txt")
        open(rf, "w").write("\n".join(g["reads"]) + "\n")
        w = os.path.join(d, "w")
        p = subprocess.run([TOOL, rf, str(g["k"]), w, str(g["B"]), "--host-result"], capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
        fk = np.fromfile(os.path.join(w, "final_kmers"), np.uint8)
    assert np.array_equal(fk, g["final_kmers"])
    assert "reference-built and GPU-built KMerIndex agree" in p.stdout
