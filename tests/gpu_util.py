"""Run the CUDA path through the C ABI and collect the artefacts golden_util / the oracle comparisons expect."""
import numpy as np

from spades_b200.graph import DeBruijnGraphConstructor
from spades_b200.kmer_index import Context, KMerDiskCounter, ParallelSortingSplitter
from spades_b200.packing import pack_reads

_CTX = None


def ctx():
    """the session's shared context on device 0 (default arena: most of the free device memory), created on first use"""
    global _CTX
    if _CTX is None:
        _CTX = Context(0)
    return _CTX


def release():
    """close the shared context and give its arena back to the device; the next ctx() creates a new one"""
    global _CTX
    if _CTX is not None:
        _CTX.close()
        _CTX = None


def gpu_graph_artifacts(reads, k, B, keep_loops=True, early_tc=0, early_at=False, at_params=(0.8, 10, 200)):
    """at_params: (ratio, min_length, max_length) of the A/T clipper"""
    c = ctx()
    c.set_reads(*pack_reads(reads))
    ratio, min_len, max_len = at_params
    g = DeBruijnGraphConstructor(c, k, B).ConstructGraph(keep_perfect_loops=keep_loops, with_coverage=True, early_tip_clipper_length=early_tc,
                                                       early_at_clipper=early_at, at_ratio=ratio, at_min_length=min_len, at_max_length=max_len)
    art = dict(kpomers=g.kpomers.kmers(), kp_bsz=g.kpomers.bucket_sizes(), kmers=g.kmers.kmers(),
               kmer_index=g.kmer_index.serialize(), kpomer_index=g.kpomer_index.serialize(), masks=g.masks(),
               cov=g.coverage(), hist=g.histogram().astype(np.int64), unitigs=g.unitigs(), gfa=g.gfa())
    art["kp_counts"] = g.kpomers.counts()
    if early_tc:
        art["tc_removed"] = g.tip_clipper_stats()[0]
    if early_at:
        st = g.at_clipper_stats()
        art["at_removed"] = [st[0], st[2]]
    return art, g


def gpu_count_artifacts(reads, K, B):
    c = ctx()
    c.set_reads(*pack_reads(reads))
    st = KMerDiskCounter(c, ParallelSortingSplitter(K)).Count(B)
    return dict(final_kmers=st.kmers(), bsz=st.bucket_sizes()), st
