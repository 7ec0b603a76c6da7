"""FASTG and unitig FASTA formatted on the GPU (fastg.cu) against the restatement in fastg_oracle: over the reference's graphs in
tests/golden, over oracle graphs at k = 21 .. 127 with and without coverage, loops and clippers, over host-resident sets, in many
formatting runs under a small HBM budget, with an edge longer than 100 kb, through a host-only graph, and the device's %f against
the host compilation."""
import ctypes as C
import os
import socket
import subprocess
import tempfile

import numpy as np
import pytest

import fastg_oracle as F
import golden_util as G
import gpu_util
import oracle as O
from spades_b200.packing import pack_reads, revcomp, synthetic_reads

pytestmark = pytest.mark.gpu


def _build(reads, k, B, **kw):
    from spades_b200.graph import DeBruijnGraphConstructor
    c = gpu_util.ctx()
    c.set_reads(*pack_reads(reads))
    return DeBruijnGraphConstructor(c, k, B).ConstructGraph(**kw)


def _check(g, gfa, k, unitigs, with_coverage=True):
    assert g.fastg() == F.fastg_from_gfa(gfa, k, with_coverage)
    assert g.unitigs_fasta() == F.unitigs_fasta(unitigs)


def _fixture_options(name, g):
    if name.endswith("_nlgraph"):
        return dict(keep_perfect_loops=False)
    if name.endswith("_tcgraph"):
        return dict(early_tip_clipper_length=g["tc_bound"])
    if name.endswith("_atgraph"):
        return dict(early_tip_clipper_length=g.get("tc_bound", 0), early_at_clipper=True)
    return {}


FIXTURES = [n for n in G.names() if n.endswith(("_graph", "_nlgraph", "_tcgraph", "_atgraph", "_eigraph")) or n.startswith("gtest_")]


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture(name):
    """the device's FASTG equals the one restated from the reference's GFA of the same reads, its unitig FASTA gbuilder's over the
    reference's unitigs"""
    g = G.load(name)
    gr = _build(g["reads"], g["k"], g["B"], **_fixture_options(name, g))
    try:
        ref_unitigs = g["unitigs_txt"].tobytes().decode().split()
        assert gr.unitigs() == ref_unitigs
        _check(gr, g["graph_gfa"].tobytes().decode(), g["k"], ref_unitigs)
        st = gr.format_stats()
        assert st["runs"] == (1 if ref_unitigs else 0) and st["bytes"] == len(gr.unitigs_fasta())
    finally:
        gr.free()


@pytest.mark.parametrize("name", G.names("fastg"))
def test_reference_fastg_fixture(name):
    """byte for byte what the reference's FastgWriter wrote over its graph of the same reads, with and without coverage, and what
    gbuilder's unitig loop wrote"""
    g = G.load(name)
    opts = dict(early_tip_clipper_length=g["tc_bound"])
    gr = _build(g["reads"], g["k"], g["B"], **opts)
    try:
        assert gr.fastg() == g["fastg"].tobytes().decode()
        assert gr.unitigs_fasta() == g["unitigs_fasta"].tobytes().decode()
    finally:
        gr.free()
    gr = _build(g["reads"], g["k"], g["B"], with_coverage=False, **opts)
    try:
        assert gr.fastg() == g["fastg_nocov"].tobytes().decode()
    finally:
        gr.free()


TOOL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "integration", "_build", "spades_gbuilder_gpu")


@pytest.mark.skipif(not os.path.exists(TOOL), reason="integration tool not built (needs the reference sources at build time)")
@pytest.mark.parametrize("args", [("21", "16", "0"), ("55", "8", "95"), ("33", "12", "0", "--host-result")])
def test_integration_tool_fastg(args):
    """spades_gbuilder_gpu --fastg: the GPU's graph.fastg and unitigs.fasta equal the reference's FastgWriter output over the
    reference's graph and gbuilder's unitig loop (exit code 0)"""
    reads = synthetic_reads(3000, 150, 4000, 0.01, seed=int(args[0])) + _loop_reads(int(args[0]))
    with tempfile.TemporaryDirectory() as d:
        rf = os.path.join(d, "reads.txt")
        with open(rf, "w") as f:
            f.write("\n".join(reads) + "\n")
        w = os.path.join(d, "w")
        p = subprocess.run([TOOL, rf, args[0], w] + list(args[1:]) + ["--fastg"], capture_output=True, text=True)
        assert p.returncode == 0, (p.stdout + p.stderr)[-3000:]
        assert "FASTG agrees" in p.stdout + p.stderr and "Unitig FASTA agrees" in p.stdout + p.stderr
        assert os.path.getsize(os.path.join(w, "graph.fastg")) > 0


def _loop_reads(seed):
    rng = np.random.default_rng(seed)
    g = "".join("ACGT"[i] for i in rng.integers(0, 4, 600))
    gg = g + g
    reads = [gg[i:i + 140] for i in range(0, 600, 7)]
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 200))
    h = x + revcomp(x)
    hh = h + h
    return reads + [hh[i:i + 150] for i in range(0, 400, 5)]


CASES = [(k, opts) for k in (21, 33, 55, 77, 99, 127) for opts in ({}, {"with_coverage": False})]
CASES += [(21, {"keep_perfect_loops": False}), (55, {"early_tip_clipper_length": 95}), (33, {"early_tip_clipper_length": 117, "early_at_clipper": True}),
          (127, {"keep_perfect_loops": False, "with_coverage": False})]


@pytest.mark.parametrize("k,opts", CASES)
def test_random_graph(k, opts):
    reads = synthetic_reads(1500, 150, 2500, 0.004 if k > 100 else 0.01, seed=700 + k) + _loop_reads(k)
    B = 16
    gr = _build(reads, k, B, **opts)
    try:
        r = O.full_graph(reads, k, B, early_tc=opts.get("early_tip_clipper_length", 0), early_at=opts.get("early_at_clipper", False),
                         keep_loops=opts.get("keep_perfect_loops", True))
        assert gr.unitigs() == r["unitigs"].seqs
        cov = opts.get("with_coverage", True)
        _check(gr, r["gfa"], k, r["unitigs"].seqs, cov)
        if not cov:
            assert "_cov_0.000000" in gr.fastg() and "_cov_0.000000" not in F.fastg_from_gfa(r["gfa"], k)
    finally:
        gr.free()


def test_host_sets():
    reads = synthetic_reads(2000, 150, 3000, 0.01, seed=91) + _loop_reads(3)
    a = _build(reads, 55, 12)
    b = _build(reads, 55, 12, result_on_host=True)
    try:
        assert a.fastg() == b.fastg() and a.unitigs_fasta() == b.unitigs_fasta()
    finally:
        a.free(); b.free()


def test_long_edge_wraps():
    """one edge of 150 kb: its body spreads over many tiles of the body kernel, both strands wrap at 60"""
    rng = np.random.default_rng(17)
    genome = "".join("ACGT"[i] for i in rng.integers(0, 4, 150_000))
    reads = [genome[i:i + 150] for i in range(0, len(genome) - 150 + 1, 50)] + [genome[-150:]]
    gr = _build(reads, 55, 8)
    try:
        assert max(len(s) for s in gr.unitigs()) == len(genome)
        r = O.full_graph(reads, 55, 8)
        _check(gr, r["gfa"], 55, r["unitigs"].seqs)
        assert F.wrapped(revcomp(genome)) in gr.fastg() and F.wrapped(genome) in gr.unitigs_fasta()
    finally:
        gr.free()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _single_gpu_edges(reads, k, B):
    """the edges and link records of one GPU's graph, from the distributed path at world size 1 (its edges are one GPU's, in order)"""
    import torch.distributed as dist
    from spades_b200.distributed import (DistributedExtensionIndexBuilder, DistributedGraphConstructor, DistributedKMerCounter,
                                         DistributedKmersFromKpomers)
    from spades_b200.kmer_index import KMerIndexBuilder
    c = gpu_util.ctx()
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1)
    try:
        c.set_reads(*pack_reads(reads))
        kp = DistributedKMerCounter(c, k + 1).Count(B)
        km = DistributedKmersFromKpomers(c, kp).Count(B)
        mkp, mk = KMerIndexBuilder(c).BuildIndex(kp), KMerIndexBuilder(c).BuildIndex(km)
        ext = DistributedExtensionIndexBuilder(c, kp, mkp, km, mk).Build()
        dg = DistributedGraphConstructor(c, ext, mkp, mk).ConstructGraph()
        e = dg.edges()
        dg.free(); ext.free(); mk.free(); mkp.free(); km.free(); kp.free()
        return e
    finally:
        dist.destroy_process_group()


def _assembled(reads, k, B):
    from spades_b200.distributed import graph_from_edges
    e = _single_gpu_edges(reads, k, B)
    return graph_from_edges(k, e["text"], e["lens"], e["link_start"], e["link_end"], e["raw_cov"])


def test_assembled_graph_same_bytes():
    reads = synthetic_reads(2000, 150, 3000, 0.01, seed=93) + _loop_reads(5)
    ag = _assembled(reads, 33, 10)
    gr = _build(reads, 33, 10)
    try:
        c = gpu_util.ctx()
        assert ag.unitigs() == gr.unitigs()
        assert ag.fastg(c) == gr.fastg() and ag.unitigs_fasta(c) == gr.unitigs_fasta()
    finally:
        ag.free(); gr.free()


def test_many_runs_under_small_budget(tmp_path):
    """a host-only graph written through a context of 64 MiB: the run buffers take a third of what the per-record tables leave, so the
    FASTG goes out in many runs, byte for byte the text of one run (the unitig FASTA, a quarter of its size, may fit one)"""
    from spades_b200.kmer_index import Context
    reads = synthetic_reads(60_000, 150, 200_000, 0.005, seed=95)
    ag = _assembled(reads, 21, 32)
    c0 = gpu_util.ctx()
    want_fastg, want_fa = ag.fastg(c0), ag.unitigs_fasta(c0)
    assert ag.format_stats()["runs"] == 1
    gpu_util.release()
    small = Context(0, hbm_budget_bytes=64 << 20)
    try:
        assert ag.fastg(small) == want_fastg
        st = ag.format_stats()
        assert st["runs"] > 1, st
        ag.write_fastg(small, tmp_path / "g.fastg")
        assert (tmp_path / "g.fastg").read_text() == want_fastg and ag.format_stats()["runs"] > 1
        ag.write_unitigs_fasta(small, tmp_path / "u.fasta")
        assert (tmp_path / "u.fasta").read_text() == want_fa
    finally:
        ag.free()
        small.close()


def test_device_cov_text_equals_host():
    from test_fastg_format import _host_cov, cov_cases
    raw, den = cov_cases(1_000_000, 12)
    c = gpu_util.ctx()
    out = np.zeros(len(raw) * 32, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    c.check(c.L.sgpu_format_coverage(c.h, 1, p(raw), p(den), len(raw), p(out)))
    dev = [bytes(r).split(b"\0")[0].decode() for r in out.reshape(-1, 32)]
    assert dev == _host_cov(raw, den)


def test_device_graph_refuses_other_context():
    from spades_b200.kmer_index import Context, SpadesGpuError
    from spades_b200.graph import graph_text
    gr = _build(synthetic_reads(500, 150, 1000, 0.0, seed=1), 21, 4)
    other = Context(0, hbm_budget_bytes=64 << 20)
    try:
        with pytest.raises(SpadesGpuError):
            graph_text(other, gr.h, True)
    finally:
        gr.free()
        other.close()
