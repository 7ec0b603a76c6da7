"""The coverage pre-filter in key-range passes (sgpu_reads_cov_filter_ex, sgpu_cov_pass_plan_host, reads_io.CovFilteringWrap(passes=)).
CPU: the pass plan, the composition of the pass hash with the rank owner, the exported symbols. GPU: forced P against the oracle
and the reference fixtures, P planned from a small HBM budget, a pass that owns ~90 % of its capacity, and degenerate read sets.
Every GPU case asserts the passes taken, so a case that stops reaching its path fails."""
import ctypes as C

import numpy as np
import pytest

import golden_util as G
import oracle as O
from spades_b200.packing import pack_reads, revcomp, synthetic_reads

MAX_PASSES = 256


def _block(b):
    return (max(b, 1) + 511) // 512 * 512


def _resident(n):
    """what the filter holds next to its table (cov_plan.h): four per-read arrays of n + 1 entries and two small flags"""
    m = n + 1
    return _block(m) + 3 * _block(4 * m) + _block(8) + _block(4)


def _single_cap(bound):
    return max(1024, bound + bound // 2)


def _pass_cap(bound, passes):
    from spades_b200.distributed import cov_layout_host
    return _single_cap(bound) if passes == 1 else cov_layout_host(passes, bound, np.zeros(0, np.uint64))[1]


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_library_exports_the_pass_entry_points():
    from spades_b200 import _lib
    L = C.CDLL(_lib.LIB_PATH)
    for s in ("sgpu_reads_cov_filter_ex", "sgpu_cov_pass_plan_host"):
        assert s in _lib.SYMBOLS and hasattr(L, s), s
    assert [f[0] for f in _lib.SgpuTimes._fields_[-2:]] == ["cov_filter_passes", "cov_filter_table_bytes"]


@pytest.mark.parametrize("bound,n", [(0, 0), (1000, 10), (3300, 3000), (25_301_174, 1_000_000), (863_686_382, 20_000_000),
                                     (6_900_000_000, 160_000_000)])
def test_pass_plan(bound, n):
    """P = 1 exactly when today's table fits next to the per-read arrays; P never falls as the budget shrinks; a pass table holds
    cov_slice_capacity(bound, P) entries and the P tables together at least 1.5 x the bound; past 256 passes the plan refuses"""
    from spades_b200.distributed import cov_pass_plan_host
    one = _resident(n) + _block(8 * _single_cap(bound))
    floor = _resident(n) + _block(8 * _pass_cap(bound, MAX_PASSES))
    assert cov_pass_plan_host(bound, n, one) == (1, _single_cap(bound))
    assert cov_pass_plan_host(bound, n, one + 12345) == (1, _single_cap(bound))
    if floor < one:
        assert cov_pass_plan_host(bound, n, one - 1)[0] >= 2
    last = 1
    for budget in np.linspace(one, floor, 300).astype(np.int64).tolist():          # shrinking
        p, cap = cov_pass_plan_host(bound, n, budget)
        assert p >= last
        last = p
        assert cap == _pass_cap(bound, p)
        assert _resident(n) + _block(8 * cap) <= budget
        if p > 1:
            assert p * cap >= bound + bound // 2
            assert _resident(n) + _block(8 * _pass_cap(bound, p - 1)) > budget      # the smallest P that fits
    assert cov_pass_plan_host(bound, n, floor)[1] == _pass_cap(bound, MAX_PASSES)
    with pytest.raises(MemoryError):
        cov_pass_plan_host(bound, n, floor - 1)
    with pytest.raises(ValueError):
        cov_pass_plan_host(bound, -1, floor)


def test_pass_hash_composes_with_the_owner():
    """pass p of rank w is id = owner(key, W * P): id // P == owner(key, W), so passes can split a rank's slice without moving keys
    between ranks"""
    from spades_b200.distributed import cov_layout_host
    rng = np.random.default_rng(5)
    keys = rng.integers(0, 1 << 47, 50000, dtype=np.uint64)
    keys[:3] = [0, 1, (1 << 47) - 1]
    for W in range(1, 9):
        owner = cov_layout_host(W, 0, keys)[0].astype(np.int64)
        for P in range(1, 17):
            assert np.array_equal(cov_layout_host(W * P, 0, keys)[0].astype(np.int64) // P, owner), (W, P)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
def _kept_reads(c):
    from spades_b200.packing import unpack_reads
    from spades_b200.reads_io import download_reads
    return unpack_reads(*download_reads(c))


def _filter(c, reads, K, thr, passes):
    """filter `reads` with forced passes and apply; checks the passes and table size the context reports -> (keep, stats list)"""
    from spades_b200.reads_io import CovFilteringWrap
    c.set_reads(*pack_reads(reads))
    keep, st = CovFilteringWrap(c, K, thr, apply=True, passes=passes)
    t = c.times()
    assert t["cov_filter_passes"] == passes
    assert t["cov_filter_table_bytes"] == 8 * _pass_cap(st["cardinality_upper_bound"], passes)
    return keep, [st["cardinality_upper_bound"], st["key_bits"], st["distinct_keys"], st["kept"]]


def _check_against_oracle(c, reads, K, thr, passes_list):
    want_keep, want = O.cov_filter(*pack_reads(reads), K, thr)
    survivors = [r for r, f in zip(reads, want_keep) if f]
    for P in passes_list:
        keep, st = _filter(c, reads, K, thr, P)
        assert st == want, P
        assert np.array_equal(keep, want_keep), P
        assert _kept_reads(c) == survivors, P
    return want_keep, want


def _random_reads(K, seed):
    """ragged, short, poly-A, low-complexity and palindromic reads (the shapes of the single-table oracle test)"""
    rng = np.random.default_rng(seed)
    reads = synthetic_reads(1500, 120, 3000, 0.01, seed=seed) + synthetic_reads(300, 90, 40000, 0.02, seed=seed + 100)
    x = "".join("ACGT"[i] for i in rng.integers(0, 4, 80))
    reads += [x + revcomp(x)] * 3 + ["A" * 150, "T" * 97, "AC" * 40, "ACGT", x[:K - 1], x[:K]]
    reads = [r[: int(rng.integers(K - 2, len(r) + 1))] if rng.random() < 0.2 and len(r) > K else r for r in reads]
    return [r for r in reads if r]


@pytest.mark.gpu
@pytest.mark.parametrize("thr", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("K", [12, 22, 33, 56, 64, 70])
def test_forced_passes_match_oracle_random(K, thr):
    from gpu_util import ctx
    _check_against_oracle(ctx(), _random_reads(K, 1000 + 10 * K + thr), K, thr, (1, 2, 3, 8, 64))


@pytest.mark.gpu
@pytest.mark.parametrize("passes", [2, 7])
@pytest.mark.parametrize("name", G.names("covfilter"))
def test_forced_passes_match_reference_golden(name, passes):
    from gpu_util import ctx
    g = G.load(name)
    K, thr = g["k"] + 1, int(g["thr"][0])
    want_keep, want = _check_against_oracle(ctx(), list(g["reads"]), K, thr, (passes,))
    assert want[:2] == [int(g["card"][0]), int(g["key_bits"][0])] and np.array_equal(want_keep, g["keep"])


def _million_reads():
    import json
    import os
    from spades_b200.packing import pack_fixed
    r = json.load(open(os.path.join(G.GOLDEN_DIR, "syn1M_sha256.json")))["reads"]
    codes = synthetic_reads(r["n"], r["len"], r["genome_len"], r["err"], seed=r["seed"], as_codes=True)
    return codes, pack_fixed


def _million_case(case):
    import json
    import os
    return json.load(open(os.path.join(G.GOLDEN_DIR, "syn1M_covfilter.json")))["cases"][case]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["k21", "k55"])
def test_million_reads_three_passes(case):
    """the 1 M-read fixture of the unmodified reference in three key-range passes: bound, key width, survivors, SHA-256 of the
    verdicts; then the count of the survivors against a count of the same reads handed over directly"""
    import hashlib
    from gpu_util import ctx
    from spades_b200.kmer_index import DeBruijnReadKMerSplitter, KMerDiskCounter
    from spades_b200.reads_io import CovFilteringWrap
    codes, pack_fixed = _million_reads()
    cs = _million_case(case)
    c = ctx()
    c.set_reads(*pack_fixed(codes))
    keep, st = CovFilteringWrap(c, cs["k"] + 1, cs["threshold"], apply=True, passes=3)
    assert c.times()["cov_filter_passes"] == 3
    assert st["cardinality_upper_bound"] == cs["cardinality_upper_bound"] and st["key_bits"] == cs["key_bits"] and st["kept"] == cs["kept"]
    assert hashlib.sha256(keep.tobytes()).hexdigest() == cs["sha256_keep"]
    a = KMerDiskCounter(c, DeBruijnReadKMerSplitter(cs["k"] + 1)).Count(16)
    ka, ca = a.kmers().copy(), a.counts().copy(); a.free()
    c.set_reads(*pack_fixed(codes[keep.astype(bool)]))
    b = KMerDiskCounter(c, DeBruijnReadKMerSplitter(cs["k"] + 1)).Count(16)
    assert np.array_equal(ka, b.kmers()) and np.array_equal(ca, b.counts()); b.free()


@pytest.mark.gpu
def test_planned_passes_within_an_hbm_budget():
    """a context whose HBM budget holds the 1 M reads but not the single table (12 bytes per key of the 25 M-key bound) plans
    P >= 2 by itself and stays within the budget; the verdicts are the reference's, the statistics those of the single table, which
    the default context takes for the same reads"""
    import hashlib
    import gpu_util
    from spades_b200.kmer_index import Context
    from spades_b200.reads_io import CovFilteringWrap
    codes, pack_fixed = _million_reads()
    cs = _million_case("k21")
    budget = 256 << 20
    assert 12 * cs["cardinality_upper_bound"] > budget
    gpu_util.release()
    small = Context(0, hbm_budget_bytes=budget)
    small.set_reads(*pack_fixed(codes))
    keep, st = CovFilteringWrap(small, cs["k"] + 1, cs["threshold"], apply=False)
    t = small.times()
    small.close()
    assert t["cov_filter_passes"] >= 2
    assert t["cov_filter_table_bytes"] == 8 * _pass_cap(st["cardinality_upper_bound"], t["cov_filter_passes"])
    assert t["cov_filter_table_bytes"] <= budget and t["peak_bytes"] <= budget
    assert st["cardinality_upper_bound"] == cs["cardinality_upper_bound"] and st["key_bits"] == cs["key_bits"] and st["kept"] == cs["kept"]
    assert hashlib.sha256(keep.tobytes()).hexdigest() == cs["sha256_keep"]
    c = gpu_util.ctx()
    c.set_reads(*pack_fixed(codes))
    keep1, st1 = CovFilteringWrap(c, cs["k"] + 1, cs["threshold"], apply=False)
    t1 = c.times()
    assert t1["cov_filter_passes"] == 1
    assert t1["cov_filter_table_bytes"] == 8 * _single_cap(cs["cardinality_upper_bound"])
    assert st1 == st and np.array_equal(keep1, keep)


@pytest.mark.gpu
@pytest.mark.parametrize("passes", [2, 3, 4])
def test_pass_owning_most_of_its_capacity(passes):
    """pass 0 owns ~90 % of its table's capacity (more than 1.5 x its even share): no overflow, the oracle's result"""
    from dist_cov_worker import owner_skew
    from gpu_util import ctx
    shards, owned0 = owner_skew(passes)
    reads = [r for s in shards for r in s]
    _, want = _check_against_oracle(ctx(), reads, 32, 1, (passes,))
    cap = _pass_cap(want[0], passes)
    assert cap > owned0 >= 0.85 * cap


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["empty", "one_read", "all_short"])
def test_degenerate_read_sets_in_four_passes(kind):
    from gpu_util import ctx
    rng = np.random.default_rng(9)
    K = 33
    reads = {"empty": [], "one_read": ["".join("ACGT"[i] for i in rng.integers(0, 4, 150))],
             "all_short": ["".join("ACGT"[i] for i in rng.integers(0, 4, int(m))) for m in rng.integers(1, K, 200)]}[kind]
    for thr in (0, 2):
        _check_against_oracle(ctx(), reads, K, thr, (4,))
