"""CPU: the host arithmetic of the distributed EdgeIndex refill (spades_b200.distributed.DistributedEdgeIndex) -- the union edge
numbering against assemble_graph's order, the single-index decision from truncated vertex lists against brute force, the slot
ranges -- and the null refusals of the new C entries."""
import ctypes as C

import numpy as np
import pytest


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fake_pieces(rng, world, B, k):
    """per-rank edges as DistributedGraph.edges() gives them: every edge's text is unique, and every bucket's edges come from its owner"""
    owners = rng.integers(0, world, B).astype(np.int32)
    pieces, tag = [], 0
    uc = np.zeros((world, B), np.uint64)
    lc = np.zeros((world, B), np.uint64)
    for r in range(world):
        for b in range(B):
            if owners[b] == r:
                uc[r, b] = rng.integers(0, 4)
                lc[r, b] = rng.integers(0, 2)
    for r in range(world):
        n_u, n_l = int(uc[r].sum()), int(lc[r].sum())
        texts = []
        for _ in range(n_u + n_l):
            texts.append("".join("ACGT"[(tag >> (2 * i)) & 3] for i in range(k + 1)))
            tag += 1
        n = n_u + n_l
        pieces.append(dict(text="".join(texts).encode(), lens=np.full(n, k + 1, np.uint32), link_start=np.arange(n, dtype=np.uint64) << 2,
                           link_end=np.arange(n, dtype=np.uint64) << 2, raw_cov=np.zeros(n, np.uint32), unitig_edges=n_u,
                           unitig_counts=uc[r], loop_counts=lc[r], texts=texts))
    return owners, uc, lc, pieces


@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_edge_numbers_follow_assemble_graph(world, monkeypatch):
    """every rank's union numbers put its edges exactly where assemble_graph puts them"""
    import torch.distributed as dist
    from spades_b200 import distributed as D
    rng = np.random.default_rng(world)
    k, B = 9, 13
    owners, uc, lc, pieces = _fake_pieces(rng, world, B, k)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)
    monkeypatch.setattr(dist, "get_global_rank", lambda group, r: r, raising=False)

    def gather(obj, out, dst=0, group=None):
        out[:] = [{key: v for key, v in p.items() if key != "texts"} for p in pieces]
    monkeypatch.setattr(dist, "gather_object", gather)

    class FakeGraph:
        num_buckets = B

        def edges(self):
            return pieces[0]
    fg = FakeGraph()
    fg.k, fg.owners = k, owners
    ag = D.assemble_graph(fg)
    union = ag.unitigs()
    ag.free()
    for r in range(world):
        p = pieces[r]
        ids = D.dist_edge_numbers(world, r, owners, uc, lc, p["unitig_edges"], len(p["lens"]))
        for i, t in enumerate(p["texts"]):
            assert union[int(ids[i])] == t
    assert sum(len(p["lens"]) for p in pieces) == len(union)


def test_edge_numbers_refuse_inconsistent_counts():
    from spades_b200 import distributed as D
    owners = np.array([0, 1], np.int32)
    uc = np.array([[2, 0], [0, 1]], np.uint64)
    lc = np.zeros((2, 2), np.uint64)
    assert list(D.dist_edge_numbers(2, 1, owners, uc, lc, 1, 1)) == [2]
    with pytest.raises(ValueError):
        D.dist_edge_numbers(2, 0, owners, uc, lc, 1, 1)                     # counts do not cover the rank's edges
    bad = uc.copy(); bad[1, 0] = 1
    with pytest.raises(ValueError):
        D.dist_edge_numbers(2, 0, owners, bad, lc, 2, 2)                    # a rank counting a bucket it does not own
    with pytest.raises(ValueError):
        D.dist_edge_numbers(2, 0, np.array([0, 2], np.int32), uc, lc, 2, 2)  # an owner outside the world


def _brute_single(ls_all, le_all, B):
    v = set()
    for ls, le in zip(ls_all, le_all):
        v.update(int(x) >> 2 for x in ls)
        v.update(int(x) >> 2 for x in le if int(x) != (1 << 64) - 1)
    return B > 1 and (2 * len(v)) // B > 0


@pytest.mark.parametrize("seed", range(6))
def test_single_flag_from_truncated_lists_matches_brute_force(seed):
    """the truncated per-rank lists decide the flag as the whole vertex set does, on both sides of the boundary"""
    from spades_b200.distributed import edge_index_single, edge_index_vertex_prefix
    rng = np.random.default_rng(seed)
    for world in (1, 2, 3, 4):
        for nv in (0, 1, 3, 7, 10, 11, 40):
            verts = rng.choice(10 ** 6, nv, replace=False).astype(np.uint64) if nv else np.zeros(0, np.uint64)
            ls_all, le_all = [], []
            for r in range(world):
                n = int(rng.integers(0, 6))
                pick = lambda: (verts[rng.integers(0, nv, n)] << 2 | rng.integers(0, 4, n).astype(np.uint64)) if nv else np.zeros(0, np.uint64)  # noqa: E731
                ls = pick() if nv else np.zeros(0, np.uint64)
                le = pick() if nv else np.zeros(0, np.uint64)
                if n and nv:
                    le[rng.random(n) < 0.3] = np.uint64((1 << 64) - 1)     # self-conjugate ends
                ls_all.append(ls); le_all.append(le)
            for B in (1, 2, 3, 7, 2 * nv - 1, 2 * nv, 2 * nv + 1, 2 * nv + 2, 200):
                if B < 1:
                    continue
                prefixes = [edge_index_vertex_prefix(ls, le, B) for ls, le in zip(ls_all, le_all)]
                assert all(len(p) <= (B + 1) // 2 for p in prefixes)
                assert edge_index_single(prefixes, B) == _brute_single(ls_all, le_all, B), (world, nv, B)


def test_vertex_prefix_is_sorted_distinct_and_truncated():
    from spades_b200.distributed import edge_index_vertex_prefix
    ls = np.array([9 << 2, 3 << 2 | 1, 9 << 2 | 2, 5 << 2], np.uint64)
    le = np.array([(1 << 64) - 1, 7 << 2, 1 << 2, 3 << 2], np.uint64)
    assert list(edge_index_vertex_prefix(ls, le, 100)) == [1, 3, 5, 7, 9]
    assert list(edge_index_vertex_prefix(ls, le, 5)) == [1, 3, 5]
    assert list(edge_index_vertex_prefix(ls, le, 1)) == [1]
    with pytest.raises(ValueError):
        edge_index_vertex_prefix(ls, le[:2], 4)


@pytest.mark.parametrize("n", [0, 1, 2, 7, 10, 1000, 2 ** 40 + 3])
def test_slot_ranges_tile_the_index(n):
    from spades_b200.distributed import slot_range_host
    for world in (1, 2, 3, 4, 7):
        ranges = [slot_range_host(n, world, r) for r in range(world)]
        assert ranges[0][0] == 0 and ranges[-1][1] == n
        for (a, b), (c, d) in zip(ranges, ranges[1:]):
            assert b == c and a <= b
        assert max(b - a for a, b in ranges) - min(b - a for a, b in ranges) <= 1
    with pytest.raises(ValueError):
        slot_range_host(n, 2, 2)


def test_new_entries_refuse_null_arguments_without_a_device():
    from spades_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    z = np.zeros(8, np.uint64)
    assert L.sgpu_dist_edge_index_begin(None, None, 0, 1, _p(z), _p(z), C.byref(h)) == 2
    assert L.sgpu_dist_edge_index_count_begin(None, 1, 0, C.byref(h)) == 2
    assert L.sgpu_dist_edge_index_keys(None, None, None, 0) == 2
    assert L.sgpu_dist_edge_index_ipc_handle(None, None) == 2
    assert L.sgpu_dist_edge_index_open_peers(None, None) == 2
    assert L.sgpu_dist_edge_index_merge(None) == 2
    assert L.sgpu_dist_edge_index_advance(None, None) == 2
    assert L.sgpu_dist_edge_index_level_done(None, 0, None) == 2
    assert L.sgpu_dist_edge_index_ranks(None) == 2
    assert L.sgpu_dist_edge_index_fill(None) == 2
    assert L.sgpu_dist_edge_index_values(None, None, None, 0) == 2
    assert L.sgpu_dist_edge_index_k(None) == -1
    assert L.sgpu_dist_edge_index_size(None) == -1
    assert L.sgpu_dist_edge_index_slot_range(None, None, None) == 2
    assert L.sgpu_dist_edge_index_serialized_size(None) == -1
    assert L.sgpu_dist_edge_index_serialize(None, None, 0) == 2
    assert L.sgpu_dist_edge_index_lookup(None, None, 0, None) == 2
    assert L.sgpu_dist_edge_index_times(None, None) == 2
    L.sgpu_dist_edge_index_free(None)
    assert L.sgpu_dist_edge_numbers_host(1, 0, 1, None, None, None, 0, 0, None) == 2
    assert L.sgpu_edge_index_vertex_prefix_host(None, None, 1, 4, None) == -1
    assert L.sgpu_dist_slot_range_host(10, 0, 0, None, None) == 2
