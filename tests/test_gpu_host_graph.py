"""GPU parity of the graph path over k-mer sets in host memory (run with -m gpu on an H100).

sgpu_kmers_from_kpomers_ex counts the k-mers of a (k+1)-mer set that may live in host memory, and sgpu_graph_build_streamed
builds the graph from sets in either place, reading them chunk by chunk. Every test checks against the C oracle and against the
device-set build (the old entries) in the same context. The path counters stage_h2d_bytes and graph_junction_batches are
asserted, so a case that stops reaching its path fails."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import golden_util as G
import oracle as O
from spades_b200.packing import pack_reads, synthetic_reads
from test_gpu_multipass import (GRAPH_CASES, MAX_CHUNKS, MIN_BUDGET, _at_reads, _budgeted, _case_reads, _check_lookups, _graph_path,
                                _loop_reads, _tiny_reads)
from test_gpu_parity import _compare, _oracle_art

pytestmark = pytest.mark.gpu


def _wbytes(K):
    return 8 * ((K + 31) // 32)


def _host_path(c, reads, k, B, kp_host=True, km_host=True, early_tc=0, early_at=False, then=None, artefacts=True):
    """the whole path with the (k+1)-mers and the k-mers placed as asked, the graph from sgpu_graph_build_streamed. Returns
    (artefacts, counters, tip clipper stats, A/T clipper stats, lookups, then(graph))"""
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.graph import DeBruijnGraph
    from spades_b200.kmer_index import DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    c.set_reads(*pack_reads(reads))
    objs = []
    try:
        kp = KMerDiskCounter(c, DeBruijnReadKMerSplitter(k + 1), result_on_host=kp_host).Count(B)
        objs.append(kp)
        kp_passes = int(c.times()["passes"])
        km = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(k, kp), result_on_host=km_host).Count(B)
        objs.append(km)
        t = c.times()
        cnt = dict(kp_passes=kp_passes, km_passes=int(t["passes"]), ex_stage=int(t["stage_h2d_bytes"]), n_kp=kp.total_kmers())
        assert kp.on_host() == kp_host and km.on_host() == km_host
        mk = KMerIndexBuilder(c).BuildIndex(km)
        objs.append(mk)
        mkp = KMerIndexBuilder(c).BuildIndex(kp)
        objs.append(mkp)
        opts = SgpuGraphOptions(1, int(early_tc), 1 if early_at else 0, 0.8, 10, 200)
        h = C.c_void_p()
        c.check(c.L.sgpu_graph_build_streamed(c.h, kp.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h)))
        g = DeBruijnGraph(c, h, kp, km, mk, mkp)
        objs.append(g)
        t = c.times()
        cnt.update(graph_stage=int(t["stage_h2d_bytes"]), batches=int(t["graph_junction_batches"]), n_km=km.total_kmers())
        art = lookups = None
        if artefacts:
            art = dict(kpomers=kp.kmers(), kp_bsz=kp.bucket_sizes(), kmers=km.kmers(), kmer_index=mk.serialize(), kpomer_index=mkp.serialize(),
                       masks=g.masks(), cov=g.coverage(), hist=g.histogram().astype(np.int64), unitigs=g.unitigs(), gfa=g.gfa(),
                       kp_counts=kp.counts())
            lookups = dict(kpomers=mkp.seq_idx(art["kpomers"]), kmers=mk.seq_idx(art["kmers"]))
        extra = then(g) if then else None
        return art, cnt, g.tip_clipper_stats(), g.at_clipper_stats(), lookups, extra
    finally:
        for o in reversed(objs):
            o.free()


def _check_counters(cnt, k, kp_host, km_host, early_tc=0, early_at=False):
    """_ex uploads the host (k+1)-mers once for the histogram (one super-range at these B) and once per pass. The graph build
    uploads the host (k+1)-mers with their multiplicities once, and the host k-mers once per sweep: the junction sweep, four for the
    A/T clipper, two for the tip clipper, and two for the loops when k-mers remain after the unitigs. Returns the loop sweeps."""
    want_ex = (1 + cnt["km_passes"]) * cnt["n_kp"] * _wbytes(k + 1) if kp_host else 0
    assert cnt["ex_stage"] == want_ex, cnt
    kp_bytes = cnt["n_kp"] * (_wbytes(k + 1) + 4) if kp_host else 0
    sweep = cnt["n_km"] * _wbytes(k) if km_host else 0
    sweeps = (1 + (4 if early_at else 0) + (2 if early_tc else 0)) if cnt["n_km"] else 0
    extra = cnt["graph_stage"] - kp_bytes - sweeps * sweep
    if sweep:
        assert extra in (0, 2 * sweep), cnt
    else:
        assert extra == 0, cnt
    return extra // sweep if sweep else None


@pytest.mark.parametrize("k,B,budget,kind", GRAPH_CASES)
def test_graph_path_on_host_sets(k, B, budget, kind):
    """both sets in host memory, split into passes: every artefact and every key's slot against the oracle and against the
    device-set build"""
    reads = _case_reads(kind, k)
    want = _oracle_art(reads, k, B)
    with _budgeted(budget) as c:
        art, cnt, _, _, lookups, _ = _host_path(c, reads, k, B)
        dev, dev_passes, _, _, _, _ = _graph_path(c, reads, k, B, want)
    passes = (cnt["kp_passes"], cnt["km_passes"])
    if budget == MIN_BUDGET:
        assert passes == (B, B)
    else:
        assert all(2 <= p < B for p in passes), passes
    _check_counters(cnt, k, True, True)
    assert _compare(art, want, B) == []
    assert _compare(art, dev, B) == []
    _check_lookups(lookups, want)


@pytest.mark.parametrize("kp_host,km_host", [(True, False), (False, True), (False, False)])
def test_mixed_placement(kp_host, km_host):
    """(k+1)-mers on host with k-mers on device, the reverse, and device sets through the streamed entry"""
    k, B = 55, 16
    reads = _case_reads("syn", k)
    want = _oracle_art(reads, k, B)
    with _budgeted(MIN_BUDGET) as c:
        art, cnt, _, _, lookups, _ = _host_path(c, reads, k, B, kp_host=kp_host, km_host=km_host)
        dev, _, _, _, _, _ = _graph_path(c, reads, k, B, want)
    _check_counters(cnt, k, kp_host, km_host)
    assert _compare(art, want, B) == [] and _compare(art, dev, B) == []
    _check_lookups(lookups, want)


@pytest.mark.parametrize("k,B", [(21, 24), (55, 16), (127, 40)])
def test_early_tip_clipper_on_host_sets(k, B):
    L = 150
    reads = synthetic_reads(3000, L, 3000, 0.02, seed=50 + k) + _loop_reads()
    want = _oracle_art(reads, k, B, early_tc=L - k)
    r = want["oracle"]
    assert r["tc"]["removed"] > 0
    with _budgeted(MIN_BUDGET) as c:
        art, cnt, tc, _, lookups, _ = _host_path(c, reads, k, B, early_tc=L - k)
        dev, _, dev_tc, _, _, _ = _graph_path(c, reads, k, B, want, early_tc=L - k)
    assert (cnt["kp_passes"], cnt["km_passes"]) == (B, B)
    _check_counters(cnt, k, True, True, early_tc=L - k)
    assert tc == dev_tc == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])
    assert _compare(art, want, B) == [] and _compare(art, dev, B) == []
    _check_lookups(lookups, want)


def test_early_at_clipper_on_host_sets():
    k, B, L = 21, 20, 100
    reads = _at_reads(2500, L, 2500, 0.01, 61)
    want = _oracle_art(reads, k, B, early_tc=L - k, early_at=True)
    r = want["oracle"]
    assert r["at"][0] > 0 and r["at"][2] > 0
    with _budgeted(MIN_BUDGET) as c:
        art, cnt, tc, at, lookups, _ = _host_path(c, reads, k, B, early_tc=L - k, early_at=True)
        dev, _, dev_tc, dev_at, _, _ = _graph_path(c, reads, k, B, want, early_tc=L - k, early_at=True)
    _check_counters(cnt, k, True, True, early_tc=L - k, early_at=True)
    assert at == dev_at == r["at"]
    assert tc == dev_tc == (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"])
    assert _compare(art, want, B) == [] and _compare(art, dev, B) == []
    _check_lookups(lookups, want)


def test_host_sets_beyond_the_chunk_table():
    """B = 300 at 64 MiB: the planner keeps both host sets within the chunk table"""
    k, B = 21, 300
    reads = _tiny_reads(400, 43)
    want = _oracle_art(reads, k, B)
    with _budgeted(MIN_BUDGET) as c:
        art, cnt, _, _, lookups, _ = _host_path(c, reads, k, B)
        dev, _, _, _, _, _ = _graph_path(c, reads, k, B, want)
    assert all(2 <= p <= MAX_CHUNKS for p in (cnt["kp_passes"], cnt["km_passes"])), cnt
    _check_counters(cnt, k, True, True)
    assert _compare(art, want, B) == [] and _compare(art, dev, B) == []
    _check_lookups(lookups, want)


def test_empty_host_sets():
    """reads shorter than k + 1: both host sets are empty, and so is the graph"""
    k, B = 21, 8
    reads = ["ACGTACGTAC", "GGGTTTAAACCC"]
    want = _oracle_art(reads, k, B)
    with _budgeted(MIN_BUDGET) as c:
        art, cnt, _, _, _, _ = _host_path(c, reads, k, B)
    assert cnt["n_kp"] == 0 and cnt["n_km"] == 0 and cnt["ex_stage"] == 0 and cnt["batches"] == 0
    assert _compare(art, want, B) == []
    assert art["unitigs"] == [] and len(art["masks"]) == 0


@pytest.mark.parametrize("k,B,K", [(33, 6, 25), (21, 6, None), (99, 6, 97)])
def test_edge_index_over_a_graph_from_host_sets(k, B, K):
    from spades_b200.graph import EdgeIndex
    reads = synthetic_reads(1000, 150, 1500, 0.01, seed=80 + k)
    want = _oracle_art(reads, k, B)
    ks, m, want_ids, want_offs = O.edge_index(want["unitigs"], k, K, 1 if K is None else B)

    def refill(gr):
        ei = EdgeIndex(gr, K, B)
        try:
            ids, offs = ei.values()
            return ids, offs, ei.serialize(), ei.seq_idx(ks.keys)
        finally:
            ei.free()

    with _budgeted(MIN_BUDGET) as c:
        art, cnt, _, _, _, (ids, offs, ser, slots) = _host_path(c, reads, k, B, then=refill)
    _check_counters(cnt, k, True, True)
    assert _compare(art, want, B) == []
    want_ser = G.edge_index_bytes(m, want["unitigs"], k, K or k + 1, B)
    assert np.array_equal(ids, want_ids) and np.array_equal(offs, want_offs)
    assert G.index_equal(want_ser, ser, 1 if K is None else B)
    assert np.array_equal(slots, np.array([m.lookup(key) for key in ks.keys], np.uint64))


CAPACITY_BUDGET = 224 << 20


def _digest(art):
    return dict(masks=hashlib.sha256(art["masks"].tobytes()).hexdigest(), cov=hashlib.sha256(art["cov"].tobytes()).hexdigest(),
                hist=art["hist"].tolist(), unitigs=hashlib.sha256("\n".join(art["unitigs"]).encode()).hexdigest(),
                gfa=hashlib.sha256(art["gfa"].encode() if isinstance(art["gfa"], str) else art["gfa"]).hexdigest())


def test_capacity_host_sets_beyond_the_budget():
    """k = 55, 300 k reads of a 1.5 Mb genome at 1 % errors plus a perfect loop and a hairpin loop, 224 MiB of HBM, the early tip
    clipper on: the two host sets hold more than twice the budget, the junction list takes several batches and the loop sweeps
    run. The host path peaks within the budget; the device path with the old entries does not. Both give the same tip clipper
    statistics, masks, coverage, histogram, unitigs and GFA. This size is checked against the device path only, not the oracle:
    the device path under the same budget extracts its unitigs in batches of another size, so agreeing outputs also show that
    the batch boundaries do not change the edges, their order or their links."""
    from spades_b200._lib import SgpuGraphOptions
    from spades_b200.graph import DeBruijnGraph
    from spades_b200.kmer_index import DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder
    k, B, L = 55, 32, 150
    reads = synthetic_reads(300000, L, 1500000, 0.01, seed=501) + _loop_reads()

    def collect(g):
        return dict(masks=g.masks(), cov=g.coverage(), hist=g.histogram().astype(np.int64), unitigs=g.unitigs(), gfa=g.gfa())

    with _budgeted(CAPACITY_BUDGET) as c:
        host, cnt, tc, _, _, hart = _host_path(c, reads, k, B, early_tc=L - k, artefacts=False, then=collect)
        host_peak = int(c.times()["peak_bytes"])
        set_bytes = cnt["n_kp"] * (_wbytes(k + 1) + 4) + cnt["n_km"] * _wbytes(k)
        objs = []
        try:
            kp = KMerDiskCounter(c, DeBruijnReadKMerSplitter(k + 1)).Count(B)
            objs.append(kp)
            km = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(k, kp)).Count(B)
            objs.append(km)
            mk = KMerIndexBuilder(c).BuildIndex(km)
            objs.append(mk)
            mkp = KMerIndexBuilder(c).BuildIndex(kp)
            objs.append(mkp)
            h = C.c_void_p()
            opts = SgpuGraphOptions(1, L - k, 0, 0.8, 10, 200)
            c.check(c.L.sgpu_graph_build_opts(c.h, kp.h, km.h, mk.h, mkp.h, C.byref(opts), C.byref(h)))
            g = DeBruijnGraph(c, h, kp, km, mk, mkp)
            objs.append(g)
            dart = collect(g)
            dev_tc = g.tip_clipper_stats()
            dev_peak = int(c.times()["peak_bytes"])
        finally:
            for o in reversed(objs):
                o.free()
    print("capacity: sets %.1f MB, host peak %.1f MB, device peak %.1f MB, junction batches %d"
          % (set_bytes / 1e6, host_peak / 1e6, dev_peak / 1e6, cnt["batches"]))
    assert set_bytes >= 2 * CAPACITY_BUDGET, set_bytes
    assert cnt["batches"] >= 2, cnt
    assert _check_counters(cnt, k, True, True, early_tc=L - k) == 2, cnt
    assert tc == dev_tc and tc[0] > 0, (tc, dev_tc)
    assert host_peak <= CAPACITY_BUDGET, host_peak
    assert dev_peak > CAPACITY_BUDGET, dev_peak
    assert _digest(hart) == _digest(dart)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GBUILDER = os.path.join(ROOT, "integration", "_build", "spades_gbuilder_gpu")


@pytest.mark.skipif(not os.path.exists(GBUILDER), reason="integration/_build/spades_gbuilder_gpu not built")
@pytest.mark.parametrize("name,early_tc", [("ecoli_k21_B40_graph", 0), ("loops_k21_B10_graph", 0), ("ecoli_k55_B16_graph", 0), ("syn_k21_B10_tcgraph", 79)])
def test_gbuilder_tool_with_host_result(name, early_tc):
    """spades_gbuilder_gpu --host-result: both counts in host memory, the graph from the streamed build; the unmodified reference
    over the GPU's arrays reproduces the GPU's unitigs and GFA, and the GFA is the golden one"""
    g = G.load(name)
    with tempfile.TemporaryDirectory() as d:
        rf = os.path.join(d, "reads.txt")
        open(rf, "w").write("\n".join(g["reads"]) + "\n")
        w = os.path.join(d, "w")
        p = subprocess.run([GBUILDER, rf, str(g["k"]), w, str(g["B"]), str(early_tc), "--host-result"], capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]
        gfa = open(os.path.join(w, "graph.gfa")).read()
    assert gfa == g["graph_gfa"].tobytes().decode()
