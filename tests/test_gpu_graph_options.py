"""GPU tests of the Construction stage's graph options against the oracle: the early tip clipper's length bound at its edges, the early
A/T clipper's (ratio, min_length, max_length) and their refusals, and keep_perfect_loops = false. Every case compares the clipper
statistics, the masks, the unitigs and the GFA; each option value is also checked to change the oracle's own result, so that a kernel
ignoring it would fail."""
import functools
import os
import sys

import numpy as np
import pytest

import golden_util as G
import oracle as O
from spades_b200.kmer_index import SpadesGpuError
from spades_b200.packing import synthetic_reads

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden import at_arm_reads, at_reads, loops_reads  # noqa: E402

pytestmark = pytest.mark.gpu

AT_DEFAULT = (0.8, 10, 200)


def _gpu_vs_oracle(reads, k, B, early_tc=0, early_at=False, at_params=AT_DEFAULT, keep_loops=True):
    """builds the graph on the GPU and asserts it equals the oracle's; returns the oracle's result"""
    from gpu_util import gpu_graph_artifacts
    art, gr = gpu_graph_artifacts(reads, k, B, keep_loops=keep_loops, early_tc=early_tc, early_at=early_at, at_params=at_params)
    r = O.full_graph(reads, k, B, early_tc=early_tc, early_at=early_at, keep_loops=keep_loops, at_params=at_params)
    tc = (r["tc"]["removed"], r["tc"]["tipped"], r["tc"]["clipped"]) if early_tc else (0, 0, 0)
    assert gr.tip_clipper_stats() == tc
    assert gr.at_clipper_stats() == (r["at"] if early_at else [0, 0, 0, 0])
    assert np.array_equal(art["masks"], r["masks"])
    assert art["unitigs"] == r["unitigs"].seqs
    assert art["gfa"] == r["gfa"]
    gr.free()
    return r


def _outcome(r):
    """what a clipper option can change: the clipper statistics and the mask array"""
    return r["tc"], r["at"], r["masks"].tobytes()


# ---- early tip clipper: the length bound -------------------------------------------------------------------------------------
TC_READS = {21: (100, 3000, 2500, 0.02, 81, 8), 77: (150, 1500, 2500, 0.01, 82, 5), 127: (250, 800, 3000, 0.005, 83, 6)}   # L, n, glen, err, seed, B
BIG = 2 ** 32 + 3


def _tc_case(k):
    L, n, glen, err, seed, B = TC_READS[k]
    return synthetic_reads(n, L, glen, err, seed=seed), L, B


@functools.lru_cache(maxsize=None)
def _tc_oracle(k, bound):
    reads, _, B = _tc_case(k)
    return _outcome(O.full_graph(reads, k, B, early_tc=bound))


@pytest.mark.parametrize("bound", ["1", "2", "5", "L-k", "10L", "2^32+3"])
@pytest.mark.parametrize("k", sorted(TC_READS))
def test_early_tip_clipper_length_bound(k, bound):
    """bounds 1, 2 and 5 bind (the oracle's result differs from the one at 10 L); 2^32 + 3 gives the unbounded result, which a bound
    truncated to 32 bits (3) would not"""
    reads, L, B = _tc_case(k)
    b = {"1": 1, "2": 2, "5": 5, "L-k": L - k, "10L": 10 * L, "2^32+3": BIG}[bound]
    r = _gpu_vs_oracle(reads, k, B, early_tc=b)
    assert r["tc"]["removed"] > 0
    if b < 10:
        assert _tc_oracle(k, b) != _tc_oracle(k, 10 * L)
    if b == BIG:
        assert _tc_oracle(k, BIG) == _tc_oracle(k, 10 * L) != _tc_oracle(k, BIG & 0xffffffff)


# ---- early A/T clipper: ratio, min_length, max_length ------------------------------------------------------------------------
AT_READS = {21: (100, 2000, 2000, 0.01, 91, 8), 97: (250, 150, 1000, 0.002, 92, 6)}     # L, n, glen, err, seed, B


def _at_case(k):
    """A-rich reads plus a 350-vertex A-rich dead-end arm (longer than the default max_length)"""
    L, n, glen, err, seed, B = AT_READS[k]
    return at_reads(n, L, glen, err, seed) + at_arm_reads(350, L, seed), L, B


def _at_sets(k):
    return {"default": AT_DEFAULT, "max1": (0.8, 10, 1), "min0": (0.8, 0, 200), "mink": (0.8, k, 200), "ratio0.5": (0.5, 10, 200),
            "ratio1": (1.0, 10, 200), "max1e6": (0.8, 10, 10 ** 6)}


@functools.lru_cache(maxsize=None)
def _at_oracle(k, params):
    reads, L, B = _at_case(k)
    return _outcome(O.full_graph(reads, k, B, early_tc=L - k, early_at=True, at_params=params))


@pytest.mark.parametrize("which", list(_at_sets(0)))
@pytest.mark.parametrize("k", sorted(AT_READS))
def test_early_at_clipper_parameters(k, which):
    """every parameter set differs from the default in the oracle's result, so each parameter reaches the clipper; on the 250-bp case
    max_length 10^6 clips the arm that max_length 200 gives up on (at k = 21 the A-rich arm repeats its k-mers, so no dead-end chain
    outlasts 200 vertices and max_length 10^6 changes nothing there)"""
    reads, L, B = _at_case(k)
    params = _at_sets(k)[which]
    r = _gpu_vs_oracle(reads, k, B, early_tc=L - k, early_at=True, at_params=params)
    assert r["at"][0] > 0
    if which != "default" and (which, k) != ("max1e6", 21):
        assert _at_oracle(k, params) != _at_oracle(k, AT_DEFAULT)
    if which == "max1e6" and k == 97:
        assert r["at"][2] - _at_oracle(k, AT_DEFAULT)[1][2] > 200


@pytest.mark.parametrize("params", [(0.8, 22, 200), (0.0, 10, 200), (1.0000001, 10, 200), (0.8, 10, 0)],
                         ids=["min_length=k+1", "ratio=0", "ratio>1", "max_length=0"])
def test_early_at_clipper_refuses_bad_parameters(params):
    """min_length > k, a ratio outside (0, 1] and max_length 0 are refused with SGPU_EINVAL; the context stays usable"""
    from gpu_util import ctx, gpu_graph_artifacts
    reads, L, B = _at_case(21)
    with pytest.raises(SpadesGpuError, match=r"^\[2\] "):
        gpu_graph_artifacts(reads, 21, B, early_tc=L - 21, early_at=True, at_params=params)
    assert ctx().h
    _gpu_vs_oracle(reads[:200], 21, B, early_at=True)


# ---- keep_perfect_loops = false ----------------------------------------------------------------------------------------------
def _loop_case(k, seed):
    """the circle and hairpin-circle windows plus noisy reads"""
    return loops_reads(250, 250) + synthetic_reads(600, 150, 1500, 0.01, seed=seed)


@pytest.mark.parametrize("k,B,seed", [(21, 6, 101), (33, 4, 102), (127, 5, 103)])
def test_no_loops_matches_oracle(k, B, seed):
    """without the loop sweeps the graph holds the unbranching paths only: fewer unitigs than with the perfect loops"""
    reads = _loop_case(k, seed)
    r = _gpu_vs_oracle(reads, k, B, keep_loops=False)
    assert len(O.full_graph(reads, k, B)["unitigs"].seqs) > len(r["unitigs"].seqs)


def test_no_loops_with_both_clippers():
    k, B, L = 55, 7, 150
    reads = _loop_case(k, 104) + at_reads(1500, L, 2000, 0.01, 105)
    r = _gpu_vs_oracle(reads, k, B, early_tc=L - k, early_at=True, keep_loops=False)
    assert r["tc"]["removed"] > 0 and r["at"][2] > 0
    kept = O.full_graph(reads, k, B, early_tc=L - k, early_at=True)
    assert len(kept["unitigs"].seqs) > len(r["unitigs"].seqs)


@pytest.mark.parametrize("name", G.names("nlgraph"))
def test_no_loops_matches_reference_golden(name):
    """keep_perfect_loops = false against the unmodified reference's ExtractUnbranchingPaths"""
    from gpu_util import gpu_graph_artifacts
    g = G.load(name)
    art, gr = gpu_graph_artifacts(g["reads"], g["k"], g["B"], keep_loops=False)
    assert G.check_graph(g, art) == []
    gr.free()
