"""Host-side mirror of the reference's graph-construction interface over the C ABI.

  DeBruijnExtensionIndexBuilder.BuildExtensionIndexFromStream / FromKPOMers
        src/common/kmer_index/extension_index/kmer_extension_index_builder.hpp:63-107
  UnbranchingPathExtractor.ExtractUnbranchingPathsAndLoops, FastGraphFromSequencesConstructor.ConstructGraph
        src/common/assembly_graph/construction/debruijn_graph_constructor.hpp:399-406,506-567
  CoverageHashMapBuilder / PHMCoverageFiller histogram   ph_map/coverage_hash_map_builder.hpp:42-56, stages/construction.cpp:404-418
  gfa::GFAWriter                                            io/graph/gfa_writer.cpp:36-116
  io::FastgWriter, spades-gbuilder's unitig FASTA           io/graph/fastg_writer.cpp:21-46, projects/spades_tools/gbuilder.cpp:191-200
"""
import ctypes as C

import numpy as np

from .kmer_index import (Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter, KMerIndexBuilder, SpadesGpuError, _p)


def graph_text(ctx, h, fastg):
    """the FASTG (fastg=True) or unitig FASTA of graph handle h, formatted on ctx's device"""
    f = ctx.L.sgpu_graph_fastg if fastg else ctx.L.sgpu_graph_unitigs_fasta
    n = f(ctx.h, h, None, 0)
    if n >= 0:
        buf = np.zeros(max(n, 1), np.uint8)
        n = f(ctx.h, h, _p(buf), n)
    if n < 0:
        raise SpadesGpuError(ctx.L.sgpu_last_error(ctx.h).decode())
    return buf[:n].tobytes().decode()


def write_graph_text(ctx, h, fastg, path):
    f = ctx.L.sgpu_graph_write_fastg if fastg else ctx.L.sgpu_graph_write_unitigs_fasta
    ctx.check(f(ctx.h, h, str(path).encode()))


def format_stats(L, h):
    """what the last FASTG or unitig FASTA call on graph handle h did: runs (formatting runs of whole records), records, bytes,
    format_ms and d2h_ms (device), write_ms (host)"""
    from ._lib import SgpuFormatStats
    st = SgpuFormatStats()
    if L.sgpu_graph_format_stats(h, C.byref(st)):
        raise SpadesGpuError("no graph")
    return {name: getattr(st, name) for name, _ in SgpuFormatStats._fields_}


class DeBruijnGraph:
    """masks + coverage + unitigs + links of the condensed graph."""

    def __init__(self, ctx, h, kpomers, kmers, kmer_index, kpomer_index):
        self.ctx, self.h = ctx, h
        self.kpomers, self.kmers, self.kmer_index, self.kpomer_index = kpomers, kmers, kmer_index, kpomer_index

    def masks(self):
        n = self.kmers.total_kmers()
        out = np.zeros(max(n, 1), np.uint8)
        self.ctx.check(self.ctx.L.sgpu_graph_masks(self.h, _p(out), n))
        return out[:n]

    def tip_clipper_stats(self):
        """(removed k-mers, tipped junctions, clipped links) of the early tip clipper; zeros when it was off."""
        out = np.zeros(3, np.uint64)
        self.ctx.check(self.ctx.L.sgpu_graph_tip_clipper_stats(self.h, _p(out)))
        return tuple(int(x) for x in out)

    def at_clipper_stats(self):
        """(edges collected, links removed, k-mers removed, clipped tips) of the early A/T clipper; zeros when it was off."""
        out = np.zeros(4, np.uint64)
        self.ctx.check(self.ctx.L.sgpu_graph_at_clipper_stats(self.h, _p(out)))
        return [int(x) for x in out]

    def coverage(self):
        n = self.kpomers.total_kmers()
        out = np.zeros(max(n, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_graph_coverage(self.h, _p(out), n))
        return out[:n]

    def histogram(self):
        n = self.ctx.L.sgpu_graph_histogram(self.h, None, 0)
        if n < 0:
            raise SpadesGpuError(self.ctx.L.sgpu_last_error(self.ctx.h).decode())
        out = np.zeros(max(n, 1), np.uint64)
        self.ctx.L.sgpu_graph_histogram(self.h, _p(out), n)
        return out[:n]

    def unitigs(self):
        ne = self.ctx.L.sgpu_graph_num_unitigs(self.h)
        nb = self.ctx.L.sgpu_graph_unitig_bases(self.h)
        buf = np.zeros(max(nb, 1), np.uint8); lens = np.zeros(max(ne, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_graph_unitigs(self.h, _p(buf), _p(lens)))
        s = buf[:nb].tobytes().decode()
        out, o = [], 0
        for l in lens[:ne]:
            out.append(s[o:o + int(l)]); o += int(l)
        return out

    def gfa(self, version="SPAdes-4.3.0-dev"):
        n = self.ctx.L.sgpu_graph_gfa(self.h, version.encode(), None, 0)
        if n < 0:
            raise SpadesGpuError(self.ctx.L.sgpu_last_error(self.ctx.h).decode())
        buf = np.zeros(max(n, 1), np.uint8)
        self.ctx.L.sgpu_graph_gfa(self.h, version.encode(), _p(buf), n)
        return buf[:n].tobytes().decode()

    def write_gfa(self, path, version="SPAdes-4.3.0-dev"):
        self.ctx.check(self.ctx.L.sgpu_graph_write_gfa(self.h, version.encode(), str(path).encode()))

    def fastg(self):
        """the graph as io::FastgWriter writes it, built on the GPU"""
        return graph_text(self.ctx, self.h, True)

    def write_fastg(self, path):
        write_graph_text(self.ctx, self.h, True, path)

    def unitigs_fasta(self):
        """the unitigs as spades-gbuilder's default mode writes them (>EDGE_<n>_length_<bases>, 60 bases per line), built on the GPU"""
        return graph_text(self.ctx, self.h, False)

    def write_unitigs_fasta(self, path):
        write_graph_text(self.ctx, self.h, False, path)

    def format_stats(self):
        return format_stats(self.ctx.L, self.h)

    def free(self):
        if self.h:
            self.ctx.L.sgpu_graph_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeBruijnGraphConstructor:
    """spades-gbuilder's sequence: (k+1)-mers -> k-mers -> MPHFs -> masks -> unitigs (+loops) -> graph (+coverage)."""

    def __init__(self, ctx: Context, k: int, num_buckets: int):
        if k % 2 == 0:
            raise ValueError("k-mer size must be odd")   # projects/spades_tools/gbuilder.cpp:125
        self.ctx, self.k, self.B = ctx, k, num_buckets

    def ConstructGraph(self, keep_perfect_loops=True, with_coverage=True, early_tip_clipper_length=0, early_at_clipper=False,
                       at_ratio=0.8, at_min_length=10, at_max_length=200, result_on_host=False) -> DeBruijnGraph:
        """early_tip_clipper_length > 0: run the Construction stage's EarlyTipClipper (stages/construction.cpp:289-302) with that
        length bound (the pipeline uses read length - k) before the unitigs are extracted; 0 = spades-gbuilder's behaviour.
        early_at_clipper: the RNA pipeline's EarlyATClipper (stages/construction.cpp:317-340) before it.
        result_on_host: both k-mer sets go to pinned host memory and the graph is built from them chunk by chunk, so the sets may
        exceed HBM; the graph is the same."""
        ctx, k, B = self.ctx, self.k, self.B
        kpomers = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(k + 1), result_on_host=result_on_host).Count(B)
        kmers = KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(k, kpomers), result_on_host=result_on_host).Count(B)
        kmer_index = KMerIndexBuilder(ctx).BuildIndex(kmers)
        kpomer_index = KMerIndexBuilder(ctx).BuildIndex(kpomers) if with_coverage else None
        h = C.c_void_p()
        from ._lib import SgpuGraphOptions
        opts = SgpuGraphOptions(1 if keep_perfect_loops else 0, int(early_tip_clipper_length), 1 if early_at_clipper else 0, float(at_ratio),
                                int(at_min_length), int(at_max_length))
        build = ctx.L.sgpu_graph_build_streamed if result_on_host else ctx.L.sgpu_graph_build_opts
        ctx.check(build(ctx.h, kpomers.h, kmers.h, kmer_index.h, kpomer_index.h if kpomer_index else None, C.byref(opts), C.byref(h)))
        return DeBruijnGraph(ctx, h, kpomers, kmers, kmer_index, kpomer_index)


class EdgeIndex:
    """debruijn_graph::EdgeIndex<Graph> after Refill() (alignment/edge_index.hpp:88-110): the K-mers of all edges (both strands) ->
    (EdgeId, offset). num_buckets = 10 x the reference's threads. k=None indexes the (k+1)-mers like the pipeline (one index segment
    built over that many vertex chunks); any other k goes through the counting path of the reference (edge_index_builders.hpp:274-307)
    with `num_buckets` buckets."""
    REMOVED, TOMBSTONE = (1 << 64) - 2, 0x7FFFFFFE

    def __init__(self, graph: DeBruijnGraph, k=None, num_buckets=None):
        self.ctx = graph.ctx
        K = 0 if k is None else int(k)
        B = 1 if num_buckets is None else int(num_buckets)
        h = C.c_void_p()
        self.ctx.check(self.ctx.L.sgpu_edge_index_build(self.ctx.h, graph.h, K, B, C.byref(h)))
        self.h = h
        self.K = self.ctx.L.sgpu_edge_index_k(h)
        self.nw = (self.K + 31) // 32

    def size(self):
        return int(self.ctx.L.sgpu_edge_index_size(self.h))

    def serialize(self) -> bytes:
        n = self.ctx.L.sgpu_edge_index_serialized_size(self.h)
        buf = np.zeros(max(n, 1), np.uint8)
        self.ctx.check(self.ctx.L.sgpu_edge_index_serialize(self.h, _p(buf), n))
        return buf[:n].tobytes()

    def values(self):
        """(edge ids u64[n], offsets u32[n]) in slot (MPHF) order"""
        n = self.size()
        ids = np.zeros(max(n, 1), np.uint64); offs = np.zeros(max(n, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_edge_index_values(self.h, _p(ids), _p(offs), n))
        return ids[:n], offs[:n]

    def seq_idx(self, keys):
        keys = np.ascontiguousarray(keys, np.uint64).reshape(-1, self.nw)
        out = np.zeros(max(len(keys), 1), np.uint64)
        self.ctx.check(self.ctx.L.sgpu_edge_index_lookup(self.h, _p(keys), len(keys), _p(out)))
        return out[: len(keys)]

    def free(self):
        if self.h:
            self.ctx.L.sgpu_edge_index_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
