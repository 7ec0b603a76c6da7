"""Multi-GPU k-mer counting: one process per GPU, torch.distributed for the small tables and the barriers,
the record exchange itself is one kernel over NVLink peer memory (sgpu_dist_exchange: pull + merge).

Mirrors what hpcspades distributes with MPI tasks + a shared filesystem (projects/hpcspades/mpi/stages/construction_mpi.cpp:222-300):
every rank reads its own slice of the reads; afterwards every bucket lives on exactly one rank.
"""
import ctypes as C

import numpy as np

from .kmer_index import KMerDiskStorage, SGPU_CANONICAL, SGPU_RESULT_ON_HOST, _p

SGPU_IPC_BYTES = 96
SGPU_DIST_GRAPH_IPC_BYTES = 256
SGPU_DIST_EDGE_INDEX_IPC_BYTES = 128


def _backend_device(group):
    import torch.distributed as dist
    return "cuda" if dist.get_backend(group) == "nccl" else "cpu"


def _pass_budget(ctx, group, free_bytes, budget_bytes):
    """the budget of the next pass: 90 % of the least any rank of `group` can allocate now (free_bytes(c_uint64 pointer) reads this
    rank's), or a fixed budget_bytes (tests)"""
    import torch
    import torch.distributed as dist
    if budget_bytes is not None:
        return int(budget_bytes)
    fb = C.c_uint64()
    ctx.check(free_bytes(C.byref(fb)))
    tb = torch.tensor([fb.value], dtype=torch.int64, device=_backend_device(group))
    dist.all_reduce(tb, op=dist.ReduceOp.MIN, group=group)
    return int(int(tb.item()) * 0.90)


def _open_peers(ctx, group, ipc_handle, open_peers, nbytes=SGPU_IPC_BYTES):
    """all_gather of the ranks' nbytes descriptors (ipc_handle(out) writes this rank's), handed to open_peers(descriptors)"""
    import torch
    import torch.distributed as dist
    desc = np.zeros(nbytes, np.uint8)
    ctx.check(ipc_handle(desc.ctypes.data_as(C.c_void_p)))
    t_h = torch.from_numpy(desc).to(_backend_device(group))
    hs = [torch.empty_like(t_h) for _ in range(dist.get_world_size(group))]
    dist.all_gather(hs, t_h, group=group)
    descs = np.ascontiguousarray(torch.stack(hs).cpu().numpy())
    ctx.check(open_peers(descs.ctypes.data_as(C.c_void_p)))


def _all_gather_u64(local, group):
    """world x len(local) table of every rank's u64 row"""
    import torch
    import torch.distributed as dist
    t = torch.from_numpy(np.ascontiguousarray(local, np.uint64).view(np.int64)).to(_backend_device(group))
    rows = [torch.empty_like(t) for _ in range(dist.get_world_size(group))]
    dist.all_gather(rows, t, group=group)
    return np.ascontiguousarray(torch.stack(rows).cpu().numpy().view(np.uint64))


def _ownership(storage, group):
    """(world x B bucket sizes, world x B owned flags) of the ranks' sets"""
    import torch
    import torch.distributed as dist
    B = storage.num_buckets()
    mine = torch.from_numpy(np.concatenate([storage.bucket_sizes(), storage.owned_buckets().astype(np.int64)])).to(_backend_device(group))
    allv = [torch.empty_like(mine) for _ in range(dist.get_world_size(group))]
    dist.all_gather(allv, mine, group=group)
    allv = torch.stack(allv).cpu().numpy()
    return allv[:, :B], allv[:, B:].astype(bool)


def _check_owned_once(bsz_all, owned_all, what="k-mer"):
    if not (owned_all.sum(axis=0) == 1).all():
        raise ValueError("every %s bucket must be owned by exactly one rank (sets from one distributed count)" % what)
    if (bsz_all[~owned_all] != 0).any():
        raise ValueError("a rank holds %ss of a bucket it does not own" % what)


def _distributed_count(ctx, group, begin, budget_bytes):
    """the pass loop of a distributed count over the ranks of `group`: begin(world, rank, handle pointer) starts it (sgpu_dist_begin
    or sgpu_dist_begin_kpomers); returns (this rank's KMerDiskStorage, passes)"""
    import torch.distributed as dist
    L = ctx.L
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    h = C.c_void_p()
    ctx.check(begin(world, rank, C.byref(h)))
    try:
        npart = L.sgpu_dist_num_partitions(h)
        local = np.zeros(npart, np.uint64)
        ctx.check(L.sgpu_dist_local_counts(h, local.ctypes.data_as(C.c_void_p)))
        all_counts = _all_gather_u64(local, group)     # the per-partition record counts (world x npart x 8 bytes: small)
        total = C.c_uint64()
        ctx.check(L.sgpu_dist_plan(h, all_counts.ctypes.data_as(C.c_void_p), C.byref(total)))
        npass = 0
        while True:
            # every pass is planned against what ALL ranks can allocate right now (earlier passes' outputs are resident)
            budget = _pass_budget(ctx, group, lambda fb: L.sgpu_dist_free_bytes(h, fb), budget_bytes)
            p = C.c_int()
            ctx.check(L.sgpu_dist_next_pass(h, budget, C.byref(p)))
            if p.value < 0:
                break
            # peers' arenas are mapped once per process
            _open_peers(ctx, group, lambda out: L.sgpu_dist_ipc_handle(h, out), lambda descs: L.sgpu_dist_open_peers(h, descs))
            ctx.check(L.sgpu_dist_scatter(h, p.value))    # local partition into the staging buffer
            dist.barrier(group=group)                     # every rank's staging buffer is complete
            ctx.check(L.sgpu_dist_exchange(h, p.value))   # one kernel: pull my pieces from all peers over NVLink + merge
            dist.barrier(group=group)                     # nobody reads my staging buffer any more (it becomes the sort's partner)
            ctx.check(L.sgpu_dist_sort(h, p.value))
            npass += 1
        dist.barrier(group=group)
        ks = C.c_void_p()
        ctx.check(L.sgpu_dist_end(h, C.byref(ks)))
        return KMerDiskStorage(ctx, ks), npass
    finally:
        L.sgpu_dist_free(h)


class DistributedKMerCounter:
    """KMerDiskCounter over a read set sharded across the ranks of a torch.distributed process group. result_on_host: each rank's
    set goes to its pinned host memory, pass by pass behind the next one."""

    def __init__(self, ctx, K, mode=SGPU_CANONICAL, group=None, result_on_host=False):
        self.ctx, self.K, self.mode, self.group, self.result_on_host = ctx, K, mode, group, result_on_host
        self.npass = 0

    def close(self):
        pass

    def Count(self, num_buckets, budget_bytes=None):
        mode = self.mode | (SGPU_RESULT_ON_HOST if self.result_on_host else 0)
        st, self.npass = _distributed_count(self.ctx, self.group, lambda world, rank, out: self.ctx.L.sgpu_dist_begin(
            self.ctx.h, self.K, num_buckets, mode, world, rank, out), budget_bytes)
        return st


class DistributedKmersFromKpomers:
    """KMerDiskCounter over a DeBruijnKMerKMerSplitter across the ranks of a torch.distributed process group: every rank brings a
    (k+1)-mer set (its shard of a DistributedKMerCounter count, or any other; the sets may overlap), and every rank gets the buckets
    it owns of the k-mers of the union of the sets, as sgpu_kmers_from_kpomers_ex gives them on one GPU. The source may live in HBM
    or in host memory; result_on_host: this rank's k-mers go to its pinned host memory, pass by pass behind the next one."""

    def __init__(self, ctx, kpomer_storage, group=None, result_on_host=False):
        self.ctx, self.kpomers, self.group, self.result_on_host = ctx, kpomer_storage, group, result_on_host
        self.npass = 0

    def close(self):
        pass

    def Count(self, num_buckets, budget_bytes=None):
        import torch.distributed as dist
        if not self.kpomers.h:
            raise ValueError("the (k+1)-mer set has been freed")
        # the ranks' level-A geometries and bucket functions only agree for one B and one k
        shape = (self.kpomers.k(), int(num_buckets))
        shapes = [None] * dist.get_world_size(self.group)
        dist.all_gather_object(shapes, shape, group=self.group)
        if any(tuple(x) != shape for x in shapes):
            raise ValueError("the ranks' (k+1, num_buckets) differ: %s" % (shapes,))
        mode = SGPU_RESULT_ON_HOST if self.result_on_host else 0
        st, self.npass = _distributed_count(self.ctx, self.group, lambda world, rank, out: self.ctx.L.sgpu_dist_begin_kpomers(
            self.ctx.h, self.kpomers.h, num_buckets, mode, world, rank, out), budget_bytes)
        return st


def assemble_kmer_index(ctx, storage, mphf, group=None):
    """KMerIndex::serialize of the union of the ranks' bucket-owned k-mer sets, from each rank's set (`storage`, from a distributed
    count) and its index (`mphf`, KMerIndexBuilder.BuildIndex of it). A bucket's bytes depend on its own keys only, so each owner
    sends the serialized bytes of the buckets it owns; rank 0 writes num_segments, every bucket's bytes in bucket order and the
    segment_starts of the union's bucket sizes. Returns the bytes on rank 0, None elsewhere."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    B = storage.num_buckets()
    bsz_all, owned_all = _ownership(storage, group)
    _check_owned_once(bsz_all, owned_all)
    own = owned_all[rank]
    runs, b = [], 0
    while b < B:                     # the serialized bytes of every maximal run of owned buckets
        if own[b]:
            e = b
            while e < B and own[e]:
                e += 1
            runs.append((b, mphf.serialize_buckets(b, e)))
            b = e
        else:
            b += 1
    pieces = [None] * world if rank == 0 else None
    dist.gather_object(runs, pieces, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    if rank != 0:
        return None
    # segment_starts as the single-GPU index computes them (mphf.cu): the running sum stops before the last entry
    bsz = bsz_all.sum(axis=0).astype(np.uint64)
    starts = np.zeros(B + 1, np.uint64)
    starts[1:B] = np.cumsum(bsz[:B - 1])
    starts[B] = bsz[B - 1]
    body = [blob for _, blob in sorted((r for rr in pieces for r in rr), key=lambda r: r[0])]
    return np.uint64(B).tobytes() + b"".join(body) + starts.tobytes()


class DistributedExtensionIndex:
    """this rank's share of the union's extension masks and coverage (DistributedExtensionIndexBuilder.Build)"""

    def __init__(self, ctx, h, kpomers, kmers, with_coverage):
        self.ctx, self.h, self.kpomers, self.kmers, self.with_coverage = ctx, h, kpomers, kmers, with_coverage
        self.npass = 0
        self.local_counts = None          # this rank's mask contributions per destination k-mer bucket
        self._hist = np.zeros(0, np.uint64)

    def masks(self):
        """the masks of this rank's k-mers, in the slot order of its k-mer index"""
        n = self.kmers.total_kmers()
        out = np.zeros(max(n, 1), np.uint8)
        self.ctx.check(self.ctx.L.sgpu_dist_ext_masks(self.h, _p(out), n))
        return out[:n]

    def coverage(self):
        """the multiplicities of this rank's (k+1)-mers, in the slot order of its (k+1)-mer index"""
        n = self.kpomers.total_kmers()
        out = np.zeros(max(n, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_dist_ext_coverage(self.h, _p(out), n))
        return out[:n]

    def histogram(self):
        """the union's coverage histogram (DeBruijnGraph.histogram of one GPU over the union)"""
        if not self.with_coverage:
            raise ValueError("built without a (k+1)-mer index: no coverage")
        return self._hist.copy()

    def times(self):
        """milliseconds of this rank's contribution histogram, scatters, applies, coverage fill and coverage histogram"""
        out = np.zeros(5, np.float32)
        self.ctx.check(self.ctx.L.sgpu_dist_ext_times(self.h, _p(out)))
        return dict(zip(("histogram", "scatter", "apply", "coverage", "coverage_histogram"), (float(x) for x in out)))

    def free(self):
        if self.h:
            self.ctx.L.sgpu_dist_ext_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DistributedExtensionIndexBuilder:
    """DeBruijnExtensionIndexBuilder and the coverage fill across the ranks of a torch.distributed process group. Every rank brings
    its bucket-owned (k+1)-mer set with multiplicities (its shard of a DistributedKMerCounter count) and that set's index, and its
    bucket-owned k-mer set (DistributedKmersFromKpomers) and that set's index. Build gives every rank the masks of the k-mers it
    owns and the coverage of the (k+1)-mers it owns, each in its own indexes' slot order, and the union's histogram: what one GPU
    computes over the union (assemble_masks / assemble_coverage lay the slices out in the union's order). kpomer_index=None builds
    the masks only; the (k+1)-mer sets may then overlap. The sets and indexes must not be freed before the result."""

    def __init__(self, ctx, kpomers, kpomer_index, kmers, kmer_index, group=None):
        self.ctx, self.kpomers, self.kpomer_index, self.kmers, self.kmer_index, self.group = ctx, kpomers, kpomer_index, kmers, kmer_index, group

    def Build(self, budget_bytes=None):
        """budget_bytes: a fixed budget of every mask pass (tests); None plans each pass against the memory every rank has free"""
        import torch
        import torch.distributed as dist
        ctx, L, group = self.ctx, self.ctx.L, self.group
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        kp, km = self.kpomers, self.kmers
        if not kp.h or not km.h:
            raise ValueError("a k-mer set has been freed")
        with_cov = self.kpomer_index is not None
        # every rank takes part in the same collectives only for one k, one B and one choice of coverage
        shape = (km.k(), km.num_buckets(), with_cov)
        shapes = [None] * world
        dist.all_gather_object(shapes, shape, group=group)
        if any(tuple(x) != shape for x in shapes):
            raise ValueError("the ranks' (k, num_buckets, coverage) differ: %s" % (shapes,))
        if with_cov:
            _check_owned_once(*_ownership(kp, group), what="(k+1)-mer")     # overlapping sources would count a (k+1)-mer twice
        bsz_all, owned_all = _ownership(km, group)
        _check_owned_once(bsz_all, owned_all)
        owners = np.ascontiguousarray(owned_all.argmax(axis=0), np.int32)
        h = C.c_void_p()
        ctx.check(L.sgpu_dist_ext_begin(ctx.h, kp.h, self.kpomer_index.h if with_cov else None, km.h, self.kmer_index.h, _p(owners), world, rank,
                                        C.byref(h)))
        ext = DistributedExtensionIndex(ctx, h, kp, km, with_cov)
        try:
            local = np.zeros(km.num_buckets(), np.uint64)
            ctx.check(L.sgpu_dist_ext_local_counts(h, _p(local)))
            ext.local_counts = local
            all_counts = _all_gather_u64(local, group)
            total = C.c_uint64()
            ctx.check(L.sgpu_dist_ext_plan(h, _p(all_counts), C.byref(total)))
            while True:
                budget = _pass_budget(ctx, group, lambda fb: L.sgpu_dist_ext_free_bytes(h, fb), budget_bytes)
                p = C.c_int()
                ctx.check(L.sgpu_dist_ext_next_pass(h, budget, C.byref(p)))
                if p.value < 0:
                    break
                _open_peers(ctx, group, lambda out: L.sgpu_dist_ext_ipc_handle(h, out), lambda descs: L.sgpu_dist_ext_open_peers(h, descs))
                ctx.check(L.sgpu_dist_ext_scatter(h, p.value))     # this rank's contributions to the pass, grouped by owner
                dist.barrier(group=group)                          # every rank's staging buffer is complete
                ctx.check(L.sgpu_dist_ext_apply(h, p.value))       # my pieces out of every peer's staging buffer, into my slice
                dist.barrier(group=group)                          # nobody reads my staging buffer any more
                ext.npass += 1
            if with_cov:
                # the union's histogram: the ranks' histograms summed, as long as the longest
                n = L.sgpu_dist_ext_histogram(h, None, 0)
                mine = np.zeros(max(n, 1), np.uint64)
                L.sgpu_dist_ext_histogram(h, _p(mine), n)
                dev = _backend_device(group)
                t = torch.tensor([n], dtype=torch.int64, device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
                m = int(t.item())
                hist = np.zeros(max(m, 1), np.uint64)
                hist[:n] = mine[:n]
                th = torch.from_numpy(hist.view(np.int64)).to(dev)
                dist.all_reduce(th, group=group)
                ext._hist = th.cpu().numpy().view(np.uint64)[:m].copy()
        except BaseException:
            ext.free()
            raise
        return ext


def _assemble_slices(piece, storage, group, what):
    """the union's array from the owners' slices (`piece`: this rank's, in the slot order of its index over `storage`): bucket b's
    run of its owner's slice goes to the union's position of bucket b. Rank 0 gets the array, the others None."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    bsz_all, owned_all = _ownership(storage, group)
    _check_owned_once(bsz_all, owned_all, what)
    pieces = [None] * world if rank == 0 else None
    dist.gather_object(piece, pieces, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    if rank != 0:
        return None
    bsz = bsz_all.sum(axis=0)
    ustart = np.concatenate(([0], np.cumsum(bsz))).astype(np.int64)
    lstart = np.concatenate((np.zeros((world, 1), np.int64), np.cumsum(bsz_all, axis=1)), axis=1)
    out = np.zeros(int(ustart[-1]), piece.dtype)
    for b in np.flatnonzero(bsz):
        r = int(np.flatnonzero(owned_all[:, b])[0])
        out[ustart[b]:ustart[b + 1]] = pieces[r][lstart[r, b]:lstart[r, b] + bsz[b]]
    return out


def assemble_masks(ext, group=None):
    """DeBruijnGraph.masks of one GPU over the union, from the ranks' slices of a DistributedExtensionIndex (the masks before any
    clipper) or of a DistributedGraph (after its early clippers): on rank 0, None elsewhere"""
    return _assemble_slices(ext.masks(), ext.kmers, group, "k-mer")


def assemble_coverage(ext, group=None):
    """DeBruijnGraph.coverage of one GPU over the union, from the ranks' slices: on rank 0, None elsewhere"""
    return _assemble_slices(ext.coverage(), ext.kpomers, group, "(k+1)-mer")


class DistributedGraph:
    """this rank's share of the union's condensed graph (DistributedGraphConstructor.ConstructGraph): the unitigs that start at a
    junction it owns, in its final_kmers x out-edge order, then the perfect loops whose leader it owns; with per-bucket counts of
    both, so that assemble_graph can interleave the ranks' edges into one GPU's order. masks() is this rank's slice of the masks
    after the early clippers (assemble_masks lays the slices out on rank 0), and the clipper statistics are the union's."""

    def __init__(self, ctx, h, k, num_buckets, owners, kmers):
        self.ctx, self.h, self.k, self.num_buckets, self.owners, self.kmers = ctx, h, k, num_buckets, owners, kmers
        self._tc, self._at = (0, 0, 0), [0, 0, 0, 0]

    def masks(self):
        """the masks of this rank's k-mers after the early clippers (the extension index's when they were off), in the slot order of
        its k-mer index"""
        n = self.kmers.total_kmers()
        out = np.zeros(max(n, 1), np.uint8)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_masks(self.h, _p(out), n))
        return out[:n]

    def tip_clipper_stats(self):
        """the union's (removed k-mers, tipped junctions, clipped links) of the early tip clipper, as DeBruijnGraph has them"""
        return self._tc

    def at_clipper_stats(self):
        """the union's (edges collected, links removed, k-mers removed, clipped tips) of the early A/T clipper, as DeBruijnGraph has them"""
        return list(self._at)

    def _clipper_counters(self):
        at, tc, remote = np.zeros(4, np.uint64), np.zeros(3, np.uint64), np.zeros(3, np.uint64)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_clipper_stats(self.h, _p(at), _p(tc), _p(remote)))
        return at, tc, remote

    def remote_clipper_stores(self):
        """this rank's clipper stores that landed in another rank's slice: {"marks", "roots", "clears"}"""
        return dict(zip(("marks", "roots", "clears"), (int(x) for x in self._clipper_counters()[2])))

    def stats(self):
        """(edges, unitig edges, bases, junction batches) of this rank"""
        out = np.zeros(4, np.uint64)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_stats(self.h, _p(out)))
        return tuple(int(x) for x in out)

    def edges(self):
        """this rank's edges: dict of text (bytes), lens, link_start, link_end, raw_cov, unitig_edges, unitig_counts, loop_counts"""
        n, nu, nb, _ = self.stats()
        seq = np.zeros(max(nb, 1), np.uint8)
        lens = np.zeros(max(n, 1), np.uint32)
        ls, le = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64)
        rc = np.zeros(max(n, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_edges(self.h, _p(seq), _p(lens), _p(ls), _p(le), _p(rc)))
        uc, lc = np.zeros(self.num_buckets, np.uint64), np.zeros(self.num_buckets, np.uint64)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_bucket_counts(self.h, _p(uc), _p(lc)))
        return dict(text=seq[:nb].tobytes(), lens=lens[:n], link_start=ls[:n], link_end=le[:n], raw_cov=rc[:n], unitig_edges=nu,
                    unitig_counts=uc, loop_counts=lc)

    def times(self):
        """milliseconds of this rank's mask copy + junction list, unitigs, visited clear and loops"""
        out = np.zeros(4, np.float32)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_times(self.h, _p(out)))
        return dict(zip(("junctions", "unitigs", "clear_visited", "loops"), (float(x) for x in out)))

    def clipper_times(self):
        """milliseconds of this rank's early clipper phases (isolate and unlink summed over both clippers)"""
        out = np.zeros(6, np.float32)
        self.ctx.check(self.ctx.L.sgpu_dist_graph_clipper_times(self.h, _p(out)))
        return dict(zip(("at_edges_probe", "at_edges_apply", "at_tips_probe", "tip_probe", "isolate", "unlink"), (float(x) for x in out)))

    def free(self):
        if self.h:
            self.ctx.L.sgpu_dist_graph_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DistributedGraphConstructor:
    """The Construction stage's early clippers and UnbranchingPathExtractor over the ranks of a torch.distributed process group,
    from each rank's DistributedExtensionIndex (its Build has run) and the indexes that built it: ConstructGraph gives every rank its
    share of the edges one GPU's DeBruijnGraphConstructor.ConstructGraph gives over the union with the same options;
    assemble_graph puts them together. The clippers and the walks read the other ranks' indexes, masks and coverage in place; no
    rank holds more than its own slices and per-bucket tables. The extension index is not changed (its masks stay the unclipped
    slice). The extension index, sets and indexes must not be freed before the result."""

    def __init__(self, ctx, ext, kpomer_index, kmer_index, group=None):
        self.ctx, self.ext, self.kpomer_index, self.kmer_index, self.group = ctx, ext, kpomer_index, kmer_index, group

    def ConstructGraph(self, keep_perfect_loops=True, early_tip_clipper_length=0, early_at_clipper=False, at_ratio=0.8, at_min_length=10,
                       at_max_length=200, budget_bytes=None):
        """the options of DeBruijnGraphConstructor.ConstructGraph (every rank passes the same ones); budget_bytes: a fixed budget of
        the junction batches (tests); None sizes them from the memory left"""
        import torch
        import torch.distributed as dist
        ctx, L, group, ext = self.ctx, self.ctx.L, self.group, self.ext
        world = dist.get_world_size(group)
        if not ext.h or not ext.kmers.h or not ext.kpomers.h:
            raise ValueError("the extension index or one of its sets has been freed")
        km, kp = ext.kmers, ext.kpomers
        with_cov = self.kpomer_index is not None
        if with_cov != ext.with_coverage:
            raise ValueError("the (k+1)-mer index must be given exactly when the extension index has coverage")
        from ._lib import SgpuGraphOptions
        opts = SgpuGraphOptions(1 if keep_perfect_loops else 0, int(early_tip_clipper_length), 1 if early_at_clipper else 0, float(at_ratio),
                                int(at_min_length), int(at_max_length))
        # the same checks as DistributedExtensionIndexBuilder: every rank takes part in the same collectives, so the options agree too
        shape = (km.k(), km.num_buckets(), with_cov) + tuple(getattr(opts, f) for f, _ in opts._fields_)
        shapes = [None] * world
        dist.all_gather_object(shapes, shape, group=group)
        if any(tuple(x) != shape for x in shapes):
            raise ValueError("the ranks' (k, num_buckets, coverage, graph options) differ: %s" % (shapes,))
        bsz_all, owned_all = _ownership(km, group)
        _check_owned_once(bsz_all, owned_all)
        owners = np.ascontiguousarray(owned_all.argmax(axis=0), np.int32)
        powners = None
        if with_cov:
            pbsz, powned = _ownership(kp, group)
            _check_owned_once(pbsz, powned, what="(k+1)-mer")
            powners = np.ascontiguousarray(powned.argmax(axis=0), np.int32)
        ubsz = np.ascontiguousarray(bsz_all.sum(axis=0), np.uint64)
        h = C.c_void_p()
        ctx.check(L.sgpu_dist_graph_begin_opts(ctx.h, ext.h, _p(owners), _p(powners) if with_cov else None, _p(ubsz), int(budget_bytes or 0),
                                               C.byref(opts), C.byref(h)))
        g = DistributedGraph(ctx, h, km.k(), km.num_buckets(), owners, km)
        try:
            def open_peers():
                _open_peers(ctx, group, lambda out: L.sgpu_dist_graph_ipc_handle(h, out), lambda descs: L.sgpu_dist_graph_open_peers(h, descs),
                            SGPU_DIST_GRAPH_IPC_BYTES)
            open_peers()
            # the clippers' phases: every rank's probe is over before any rank changes a mask (the snapshot of one GPU's build)
            phases = []
            if early_at_clipper:
                phases += ["at_edges_probe", "at_edges_apply", "at_tips_probe", "isolate", "unlink"]
            if early_tip_clipper_length:
                phases += ["tip_probe", "isolate", "unlink"]
            if phases:
                for name in phases + ["junctions"]:
                    ctx.check(getattr(L, "sgpu_dist_graph_" + name)(h))
                    dist.barrier(group=group)
                at, tc, _ = g._clipper_counters()            # the union's counters: the sums of the ranks'
                t = torch.from_numpy(np.concatenate((at, tc)).view(np.int64)).to(_backend_device(group))
                dist.all_reduce(t, group=group)
                tot = t.cpu().numpy().view(np.uint64)
                g._at, g._tc = [int(x) for x in tot[:4]], tuple(int(x) for x in tot[4:])
            ctx.check(L.sgpu_dist_graph_unitigs(h))          # walks through every rank's masks; marks visited k-mers wherever they live
            dist.barrier(group=group)                         # every rank's visited flags are final
            if keep_perfect_loops:
                ctx.check(L.sgpu_dist_graph_clear_visited(h))
                dist.barrier(group=group)                     # every rank's masks are cleared and its remaining slots ranked
                open_peers()                                  # the remaining slots' positions now exist
                ctx.check(L.sgpu_dist_graph_loops(h))
            dist.barrier(group=group)                         # nobody reads my arrays any more
        except BaseException:
            g.free()
            raise
        return g


class AssembledGraph:
    """the union's graph from the ranks' edges (assemble_graph): unitigs(), gfa() and write_gfa() as DeBruijnGraph has them"""

    def __init__(self, ctx_lib, h):
        self.L, self.h = ctx_lib, h

    def _err(self):
        from .kmer_index import SpadesGpuError
        return SpadesGpuError("host-only graph call failed")

    def unitigs(self):
        ne, nb = self.L.sgpu_graph_num_unitigs(self.h), self.L.sgpu_graph_unitig_bases(self.h)
        buf = np.zeros(max(nb, 1), np.uint8); lens = np.zeros(max(ne, 1), np.uint32)
        if self.L.sgpu_graph_unitigs(self.h, _p(buf), _p(lens)):
            raise self._err()
        s = buf[:nb].tobytes().decode()
        out, o = [], 0
        for ln in lens[:ne]:
            out.append(s[o:o + int(ln)]); o += int(ln)
        return out

    def gfa(self, version="SPAdes-4.3.0-dev"):
        n = self.L.sgpu_graph_gfa(self.h, version.encode(), None, 0)
        if n < 0:
            raise self._err()
        buf = np.zeros(max(n, 1), np.uint8)
        self.L.sgpu_graph_gfa(self.h, version.encode(), _p(buf), n)
        return buf[:n].tobytes().decode()

    def write_gfa(self, path, version="SPAdes-4.3.0-dev"):
        if self.L.sgpu_graph_write_gfa(self.h, version.encode(), str(path).encode()):
            raise self._err()

    def free(self):
        if self.h:
            self.L.sgpu_graph_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def graph_from_edges(k, text, lens, link_start, link_end, raw_cov):
    """a host-only graph (AssembledGraph) from edges laid end to end in `text`; refuses inconsistent edges with ValueError"""
    from . import _lib
    L = _lib.load()
    lens = np.ascontiguousarray(lens, np.uint32)
    ls, le = np.ascontiguousarray(link_start, np.uint64), np.ascontiguousarray(link_end, np.uint64)
    rc = np.ascontiguousarray(raw_cov, np.uint32)
    n = len(lens)
    if not (len(ls) == len(le) == len(rc) == n):
        raise ValueError("the edge arrays have different lengths")
    buf = np.frombuffer(bytes(text) + b"\0", np.uint8)
    h = C.c_void_p()
    if L.sgpu_graph_from_edges(int(k), _p(buf), len(text), _p(lens), _p(ls), _p(le), _p(rc), n, C.byref(h)):
        raise ValueError("inconsistent edges: a length below k + 1, or lengths that do not add up to the text")
    return AssembledGraph(L, h)


def assemble_graph(dg, group=None):
    """the union's graph on rank 0 (None elsewhere): the ranks' edges interleaved into one GPU's order -- the unitig edges bucket by
    bucket (each bucket's from its owner, in its order), then the loop edges bucket by bucket"""
    import torch.distributed as dist
    rank = dist.get_rank(group)
    mine = dg.edges()
    pieces = [None] * dist.get_world_size(group) if rank == 0 else None
    dist.gather_object(mine, pieces, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    if rank != 0:
        return None
    texts, lens, ls, le, rc = [], [], [], [], []
    offs = [np.concatenate(([0], np.cumsum(p["lens"], dtype=np.uint64))).astype(np.int64) for p in pieces]
    cur_u = [0] * len(pieces)
    cur_l = [p["unitig_edges"] for p in pieces]

    def take(r, a, n):
        p = pieces[r]
        texts.append(p["text"][offs[r][a]:offs[r][a + n]])
        for dst, key in ((lens, "lens"), (ls, "link_start"), (le, "link_end"), (rc, "raw_cov")):
            dst.append(p[key][a:a + n])
    for counts, cur in (("unitig_counts", cur_u), ("loop_counts", cur_l)):
        for b in range(dg.num_buckets):
            r = int(dg.owners[b])
            n = int(pieces[r][counts][b])
            if n:
                take(r, cur[r], n)
                cur[r] += n
    for r, p in enumerate(pieces):
        if cur_u[r] != p["unitig_edges"] or cur_l[r] != len(p["lens"]):
            raise ValueError("rank %d's bucket counts do not cover its edges" % r)
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)     # noqa: E731
    return graph_from_edges(dg.k, b"".join(texts), cat(lens, np.uint32), cat(ls, np.uint64), cat(le, np.uint64), cat(rc, np.uint32))


def edge_index_vertex_prefix(link_start, link_end, num_buckets):
    """the sorted distinct vertex slots of edges with these link records, the first ceil(num_buckets / 2) of them (pure host
    arithmetic): a rank's part of the single-index decision of a DistributedEdgeIndex"""
    from . import _lib
    L = _lib.load()
    ls, le = np.ascontiguousarray(link_start, np.uint64), np.ascontiguousarray(link_end, np.uint64)
    if len(ls) != len(le) or int(num_buckets) < 1:
        raise ValueError("link arrays of different lengths, or num_buckets < 1")
    out = np.zeros((int(num_buckets) + 1) // 2 + 1, np.uint64)
    n = L.sgpu_edge_index_vertex_prefix_host(_p(ls), _p(le), len(ls), int(num_buckets), _p(out))
    if n < 0:
        raise ValueError("bad arguments")
    return out[:n].copy()


def edge_index_single(prefixes, num_buckets):
    """the single-index flag of the (k+1)-mer EdgeIndex over the union (num_buckets > 1 and 2 x distinct vertex slots >= num_buckets),
    from every rank's edge_index_vertex_prefix: a rank holding ceil(B / 2) vertices decides it alone, otherwise the lists are whole"""
    B = int(num_buckets)
    union = np.unique(np.concatenate([np.asarray(p, np.uint64) for p in prefixes])) if len(prefixes) else np.zeros(0, np.uint64)
    return B > 1 and len(union) >= (B + 1) // 2


def dist_edge_numbers(world, rank, owners, unitig_counts_all, loop_counts_all, unitig_edges, edges):
    """the union number of each of a rank's edges in assemble_graph's order (pure host arithmetic)"""
    from . import _lib
    L = _lib.load()
    owners = np.ascontiguousarray(owners, np.int32)
    uc, lc = np.ascontiguousarray(unitig_counts_all, np.uint64), np.ascontiguousarray(loop_counts_all, np.uint64)
    out = np.zeros(max(int(edges), 1), np.uint64)
    rc = L.sgpu_dist_edge_numbers_host(int(world), int(rank), len(owners), _p(owners), _p(uc), _p(lc), int(unitig_edges), int(edges), _p(out))
    if rc:
        raise ValueError("inconsistent bucket counts (code %d)" % rc)
    return out[:int(edges)]


def slot_range_host(n, world, rank):
    """[lo, hi): the slots of rank `rank` of a DistributedEdgeIndex over n slots (pure host arithmetic)"""
    from . import _lib
    L = _lib.load()
    lo, hi = C.c_uint64(), C.c_uint64()
    if L.sgpu_dist_slot_range_host(int(n), int(world), int(rank), C.byref(lo), C.byref(hi)):
        raise ValueError("bad world size or rank")
    return int(lo.value), int(hi.value)


class DistributedEdgeIndex:
    """EdgeIndex (graph.EdgeIndex) over the union of the ranks' edges of a DistributedGraph, built across the ranks of a
    torch.distributed process group. Every rank holds the union's index: K, size(), serialize() and seq_idx() are one GPU's over the
    union (assembled graph); values() are the (edge id, offset) of this rank's slots, slot_range() = [n r / W, n (r+1) / W), with
    the union's edge ids (assemble_edge_index_values gathers them). k and num_buckets as graph.EdgeIndex; every rank passes the same
    arguments. budget_bytes: a fixed budget of every pass of the key count (tests); None plans each pass against the memory every
    rank has free. The graph may be freed afterwards."""
    REMOVED, TOMBSTONE = (1 << 64) - 2, 0x7FFFFFFE

    def __init__(self, dg, k=None, num_buckets=None, group=None, budget_bytes=None):
        import torch
        import torch.distributed as dist
        ctx, L = dg.ctx, dg.ctx.L
        self.ctx, self.h, self.group = ctx, None, group
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        K = 0 if k is None else int(k)
        B = 1 if num_buckets is None else int(num_buckets)
        # every rank takes part in the same collectives only for one K and one B
        shape = (K, B, dg.k, dg.num_buckets)
        shapes = [None] * world
        dist.all_gather_object(shapes, shape, group=group)
        if any(tuple(x) != shape for x in shapes):
            raise ValueError("the ranks' (k, num_buckets) differ: %s" % ([x[:2] for x in shapes],))
        if not dg.h:
            raise ValueError("the distributed graph has been freed")
        e = dg.edges()
        uc, lc = _all_gather_u64(e["unitig_counts"], group), _all_gather_u64(e["loop_counts"], group)
        h = C.c_void_p()
        ctx.check(L.sgpu_dist_edge_index_begin(ctx.h, dg.h, K, B, _p(uc), _p(lc), C.byref(h)))
        self.h = h
        self.K = L.sgpu_dist_edge_index_k(h)
        self.nw = (self.K + 31) // 32
        self.count_ms = 0.0
        try:
            import time
            t0 = time.perf_counter()
            keys, self.npass = _distributed_count(ctx, group, lambda w, r, out: L.sgpu_dist_edge_index_count_begin(h, w, r, out), budget_bytes)
            self.count_ms = (time.perf_counter() - t0) * 1e3
            try:
                single = False
                if self.K == dg.k + 1:
                    prefixes = [None] * world
                    dist.all_gather_object(prefixes, edge_index_vertex_prefix(e["link_start"], e["link_end"], B), group=group)
                    single = edge_index_single(prefixes, B)
                ubsz = np.ascontiguousarray(_all_gather_u64(keys.bucket_sizes().astype(np.uint64), group).sum(axis=0), np.uint64)
                ctx.check(L.sgpu_dist_edge_index_keys(h, keys.h, _p(ubsz), 1 if single else 0))
                _open_peers(ctx, group, lambda out: L.sgpu_dist_edge_index_ipc_handle(h, out), lambda descs: L.sgpu_dist_edge_index_open_peers(h, descs),
                            SGPU_DIST_EDGE_INDEX_IPC_BYTES)
                dev = _backend_device(group)
                self.levels = 0
                while True:
                    dist.barrier(group=group)                  # every rank's copy of the level is complete
                    ctx.check(L.sgpu_dist_edge_index_merge(h))
                    dist.barrier(group=group)                  # nobody reads my level or collision words any more
                    live = C.c_uint64()
                    ctx.check(L.sgpu_dist_edge_index_advance(h, C.byref(live)))
                    t = torch.tensor([live.value], dtype=torch.int64, device=dev)
                    dist.all_reduce(t, group=group)
                    more = C.c_int()
                    ctx.check(L.sgpu_dist_edge_index_level_done(h, int(t.item()), C.byref(more)))
                    self.levels += 1
                    if not more.value:
                        break
                ctx.check(L.sgpu_dist_edge_index_ranks(h))
            finally:
                keys.free()
            dist.barrier(group=group)                          # every rank's slice is cleared and its copy of the index complete
            ctx.check(L.sgpu_dist_edge_index_fill(h))
            dist.barrier(group=group)                          # every put has landed
        except BaseException:
            self.free()
            raise

    def size(self):
        return int(self.ctx.L.sgpu_dist_edge_index_size(self.h))

    def slot_range(self):
        lo, hi = C.c_int64(), C.c_int64()
        self.ctx.check(self.ctx.L.sgpu_dist_edge_index_slot_range(self.h, C.byref(lo), C.byref(hi)))
        return int(lo.value), int(hi.value)

    def serialize(self) -> bytes:
        n = self.ctx.L.sgpu_dist_edge_index_serialized_size(self.h)
        buf = np.zeros(max(n, 1), np.uint8)
        self.ctx.check(self.ctx.L.sgpu_dist_edge_index_serialize(self.h, _p(buf), n))
        return buf[:n].tobytes()

    def values(self):
        """(edge ids u64, offsets u32) of this rank's slots, slot_range() in slot order"""
        lo, hi = self.slot_range()
        n = hi - lo
        ids = np.zeros(max(n, 1), np.uint64); offs = np.zeros(max(n, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_dist_edge_index_values(self.h, _p(ids), _p(offs), n))
        return ids[:n], offs[:n]

    def seq_idx(self, keys):
        keys = np.ascontiguousarray(keys, np.uint64).reshape(-1, self.nw)
        out = np.zeros(max(len(keys), 1), np.uint64)
        self.ctx.check(self.ctx.L.sgpu_dist_edge_index_lookup(self.h, _p(keys), len(keys), _p(out)))
        return out[: len(keys)]

    def times(self):
        """milliseconds of this rank's begin (edge numbers, packing), key count, keys, levels, ranks, fill and values"""
        out = np.zeros(6, np.float32)
        self.ctx.check(self.ctx.L.sgpu_dist_edge_index_times(self.h, _p(out)))
        t = dict(zip(("pack", "keys", "levels", "ranks", "fill", "values"), (float(x) for x in out)))
        t["count"] = self.count_ms
        return t

    def free(self):
        if self.h:
            self.ctx.L.sgpu_dist_edge_index_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def assemble_edge_index_values(dei, group=None):
    """graph.EdgeIndex.values of one GPU over the union, from the ranks' slot ranges of a DistributedEdgeIndex: (ids, offsets) on
    rank 0, None elsewhere"""
    import torch.distributed as dist
    rank = dist.get_rank(group)
    mine = dei.values()
    pieces = [None] * dist.get_world_size(group) if rank == 0 else None
    dist.gather_object((dei.slot_range(), mine), pieces, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    if rank != 0:
        return None
    n = dei.size()
    ids, offs = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    at = 0
    for (lo, hi), (i, o) in pieces:
        if lo != at:
            raise ValueError("the ranks' slot ranges do not tile the index")
        ids[lo:hi], offs[lo:hi] = i, o
        at = hi
    if at != n:
        raise ValueError("the ranks' slot ranges do not tile the index")
    return ids, offs


def distributed_cov_filter(ctx, k_plus_one, threshold, group=None, apply=True, phase_done=None):
    """reads_io.CovFilteringWrap over a read set sharded across the ranks of a torch.distributed process group: the verdicts, bound
    and key width are those of one GPU over the union of the shards (in rank order). Returns (keep flags of this rank's reads as
    they were, {"cardinality_upper_bound", "key_bits", "distinct_keys" (the union's), "distinct_keys_rank" (this rank's slice),
    "kept" (this rank's reads)}); with apply the survivors become this rank's read set, ready for DistributedKMerCounter.
    phase_done(name), if given, is called as each of "hll", "merge", "fill", "filter" ends (scripts/bench_dist_covfilter.py)."""
    done = phase_done or (lambda name: None)
    import torch
    import torch.distributed as dist
    L = ctx.L
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    backend_dev = _backend_device(group)
    n, nw = C.c_int64(), C.c_uint64()
    ctx.check(L.sgpu_reads_info(ctx.h, C.byref(n), C.byref(nw)))
    keep = np.zeros(max(n.value, 1), np.uint8)
    stats = np.zeros(4, np.uint64)
    h = C.c_void_p()
    ctx.check(L.sgpu_dist_cov_begin(ctx.h, int(k_plus_one), int(threshold), world, rank, C.byref(h)))
    try:
        done("hll")
        for name, step in (("merge", L.sgpu_dist_cov_bound), ("fill", L.sgpu_dist_cov_fill)):
            # descriptors of the registers, then of the table slices; the all_gather also orders the steps across the ranks
            _open_peers(ctx, group, lambda out: L.sgpu_dist_cov_ipc_handle(h, out), lambda descs: L.sgpu_dist_cov_open_peers(h, descs))
            ctx.check(step(h))
            done(name)
        dist.barrier(group=group)                     # every rank's windows are in the owners' slices
        ctx.check(L.sgpu_dist_cov_filter(h, 1 if apply else 0, keep.ctypes.data_as(C.c_void_p), stats.ctypes.data_as(C.c_void_p)))
        done("filter")
        dist.barrier(group=group)                     # nobody reads my slice any more
    finally:
        L.sgpu_dist_cov_free(h)
    tot = torch.tensor([int(stats[2])], dtype=torch.int64, device=backend_dev)
    dist.all_reduce(tot, group=group)
    return keep[: n.value], {"cardinality_upper_bound": int(stats[0]), "key_bits": int(stats[1]), "distinct_keys": int(tot.item()),
                             "distinct_keys_rank": int(stats[2]), "kept": int(stats[3])}


def cov_layout_host(world, cardinality_bound, keys):
    """the distributed filter's layout alone (pure host arithmetic): (owner rank of each masked key, entries of a rank's slice)"""
    from . import _lib
    L = _lib.load()
    keys = np.ascontiguousarray(keys, np.uint64)
    owners = np.zeros(max(len(keys), 1), np.uint32)
    cap = C.c_uint64()
    if L.sgpu_dist_cov_layout_host(world, cardinality_bound, keys.ctypes.data_as(C.c_void_p), len(keys), owners.ctypes.data_as(C.c_void_p), C.byref(cap)):
        raise ValueError("bad world size or arguments")
    return owners[: len(keys)], int(cap.value)


def cov_pass_plan_host(cardinality_bound, nreads, budget_bytes):
    """the single-GPU filter's key-range pass plan alone (pure host arithmetic): (passes, entries of one pass's table) for the device
    bytes left after the cardinality bound; raises MemoryError when 256 passes do not fit"""
    from . import _lib
    L = _lib.load()
    passes, cap = C.c_int(), C.c_uint64()
    rc = L.sgpu_cov_pass_plan_host(cardinality_bound, nreads, budget_bytes, C.byref(passes), C.byref(cap))
    if rc == 4:
        raise MemoryError("the coverage filter's table does not fit %d bytes in 256 key-range passes" % budget_bytes)
    if rc:
        raise ValueError("bad arguments")
    return passes.value, int(cap.value)


def ext_plan_host(world, owners, all_counts, budget_bytes, record_bytes):
    """the mask passes' plan alone (pure host arithmetic): (passes, bucket boundaries, the most records any rank sends or any owner
    receives in one pass) for owners[b] = the rank owning k-mer bucket b and all_counts = world x B contributions"""
    from . import _lib
    L = _lib.load()
    owners = np.ascontiguousarray(owners, np.int32)
    all_counts = np.ascontiguousarray(all_counts, np.uint64)
    B = len(owners)
    bounds = np.zeros(B + 1, np.int32)
    mx = C.c_uint64()
    n = L.sgpu_dist_ext_plan_host(world, B, _p(owners), _p(all_counts), budget_bytes, record_bytes, _p(bounds), C.byref(mx))
    if n < 0:
        raise ValueError("bad world size, owner table or arguments")
    return n, bounds[: n + 1].copy(), int(mx.value)


def plan_host(world, num_buckets, key_bits, all_counts, budget_bytes, record_bytes):
    """The pass / ownership planning alone (pure host arithmetic; used by the CPU gloo tests)."""
    from . import _lib
    L = _lib.load()
    all_counts = np.ascontiguousarray(all_counts, np.uint64)
    bounds = np.zeros(num_buckets + 2, np.int32)
    mx = C.c_uint64()
    n = L.sgpu_dist_plan_host(world, num_buckets, key_bits, all_counts.ctypes.data_as(C.c_void_p), budget_bytes, record_bytes,
                              bounds.ctypes.data_as(C.c_void_p), C.byref(mx))
    if n < 0:
        raise RuntimeError("sgpu_dist_plan_host failed")
    return n, bounds[: n + 1].copy(), int(mx.value)


def owner_bounds(pass_lo, pass_hi, world):
    """contiguous ownership split of a pass's bucket range (same formula as DistPlan::own_lo)."""
    nb = pass_hi - pass_lo
    return [pass_lo + (nb * g) // world for g in range(world + 1)]
