"""The local sort's segment pipeline against the C oracle, at every record width (run with -m gpu on an H100).

Each CTA of the local sort is persistent and copies the next segment into shared memory while it sorts the current one. These
counts put the pipeline's boundaries in one launch at K = 22, 56, 78 and 128 (one to four words per record):
  - fewer segments than CTAs (a handful of reads);
  - empty segments (refinement children no key fell into) next to segments of exactly the local-sort capacity (one key copied
    CAP times, which the refinement isolates with every key bit fixed);
  - an oversize equal-key segment (one key copied CAP + 1 times) between normal ones;
  - segments that take the exact LSD fallback (poly-A keys sharing one bin) among the normal segments that follow them;
  - segments starting on an 8-byte boundary (1- and 3-word records, any segment after one of odd length)."""
import numpy as np
import pytest

import gpu_util
import oracle as O
from spades_b200.packing import pack_reads, revcomp, synthetic_reads
from tuning_worker import polyA_reads

pytestmark = pytest.mark.gpu

CANON = 0
WIDTHS = [22, 56, 78, 128]


def _cap(K):
    return 2048 if (K + 31) // 32 <= 2 else 1024      # SortCfg<NW>::CAP


def _key_read(rng, K):
    """a read of exactly K bases that is not its own reverse complement: one canonical key"""
    while True:
        x = "".join("ACGT"[c] for c in rng.integers(0, 4, K))
        if x != revcomp(x):
            return x


def _count(reads, K, B):
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter
    c = gpu_util.ctx()
    words, offs, lens = pack_reads(reads)
    c.set_reads(words, offs, lens)
    st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
    try:
        got = dict(keys=st.kmers(), counts=st.counts(), bsz=st.bucket_sizes())
    finally:
        st.free()
    want = O.count(words, offs, lens, K, B, CANON)
    return got, want, c.times()


def _assert_same(got, want):
    assert np.array_equal(np.asarray(got["bsz"]).ravel(), np.asarray(want.bsz).ravel()), "bucket sizes differ"
    assert np.array_equal(np.asarray(got["keys"]).ravel(), np.asarray(want.keys).ravel()), "keys differ"
    assert np.array_equal(np.asarray(got["counts"]).ravel(), np.asarray(want.counts).ravel()), "multiplicities differ"


@pytest.mark.parametrize("K", WIDTHS)
def test_fewer_segments_than_ctas(K):
    reads = synthetic_reads(6, 150, 2000, 0.01, seed=31 + K)
    got, want, _ = _count(reads, K, 2)
    _assert_same(got, want)


@pytest.mark.parametrize("K", WIDTHS)
def test_segment_pipeline_boundaries(K):
    rng = np.random.default_rng(4100 + K)
    cap = _cap(K)
    reads = synthetic_reads(4000, 150, 20_000, 0.01, seed=41 + K)
    reads += [_key_read(rng, K)] * cap                    # a segment of exactly CAP records
    reads += [_key_read(rng, K)] * (cap + 1)              # an oversize equal-key segment
    reads += polyA_reads(K, 200, True)                    # bins with many distinct keys: the LSD fallback
    reads += ["".join("ACGT"[c] for c in rng.integers(0, 4, int(n))) for n in rng.integers(K, K + 40, 500)]
    got, want, t = _count(reads, K, 3)
    _assert_same(got, want)
    assert t["sort_lsd_fallbacks"] > 0, "no segment took the LSD fallback"
    assert t["sort_oversize_equal"] > 0, "no oversize equal-key segment"
