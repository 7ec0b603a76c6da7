"""Multi-GPU k-mer counting: one process per GPU, torch.distributed for the small tables and the barriers,
the record exchange itself is one kernel over NVLink peer memory (sgpu_dist_exchange: pull + merge).

Mirrors what hpcspades distributes with MPI tasks + a shared filesystem (projects/hpcspades/mpi/stages/construction_mpi.cpp:222-300):
every rank reads its own slice of the reads; afterwards every bucket lives on exactly one rank.
"""
import ctypes as C

import numpy as np

from .kmer_index import KMerDiskStorage, SGPU_CANONICAL, SGPU_RESULT_ON_HOST

SGPU_IPC_BYTES = 96


def _backend_device(group):
    import torch.distributed as dist
    return "cuda" if dist.get_backend(group) == "nccl" else "cpu"


def _distributed_count(ctx, group, begin, budget_bytes):
    """the pass loop of a distributed count over the ranks of `group`: begin(world, rank, handle pointer) starts it (sgpu_dist_begin
    or sgpu_dist_begin_kpomers); returns (this rank's KMerDiskStorage, passes)"""
    import torch
    import torch.distributed as dist
    L = ctx.L
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    backend_dev = _backend_device(group)
    h = C.c_void_p()
    ctx.check(begin(world, rank, C.byref(h)))
    try:
        npart = L.sgpu_dist_num_partitions(h)
        local = np.zeros(npart, np.uint64)
        ctx.check(L.sgpu_dist_local_counts(h, local.ctypes.data_as(C.c_void_p)))
        # all_gather of the per-partition record counts (world x npart x 8 bytes: small)
        t_local = torch.from_numpy(local.view(np.int64)).to(backend_dev)
        gathered = [torch.empty_like(t_local) for _ in range(world)]
        dist.all_gather(gathered, t_local, group=group)
        all_counts = np.ascontiguousarray(torch.stack(gathered).cpu().numpy().view(np.uint64))
        total = C.c_uint64()
        ctx.check(L.sgpu_dist_plan(h, all_counts.ctypes.data_as(C.c_void_p), C.byref(total)))
        npass = 0
        while True:
            # every pass is planned against what ALL ranks can allocate right now (earlier passes' outputs are resident)
            if budget_bytes is None:
                fb = C.c_uint64()
                ctx.check(L.sgpu_dist_free_bytes(h, C.byref(fb)))
                tb = torch.tensor([fb.value], dtype=torch.int64, device=backend_dev)
                dist.all_reduce(tb, op=dist.ReduceOp.MIN, group=group)
                budget = int(int(tb.item()) * 0.90)
            else:
                budget = int(budget_bytes)                 # tests: a fixed per-pass budget
            p = C.c_int()
            ctx.check(L.sgpu_dist_next_pass(h, budget, C.byref(p)))
            if p.value < 0:
                break
            desc = np.zeros(SGPU_IPC_BYTES, np.uint8)
            ctx.check(L.sgpu_dist_ipc_handle(h, desc.ctypes.data_as(C.c_void_p)))
            t_h = torch.from_numpy(desc).to(backend_dev)
            hs = [torch.empty_like(t_h) for _ in range(world)]
            dist.all_gather(hs, t_h, group=group)
            descs = np.ascontiguousarray(torch.stack(hs).cpu().numpy())
            ctx.check(L.sgpu_dist_open_peers(h, descs.ctypes.data_as(C.c_void_p)))     # peers' arenas are mapped once per process
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
    import torch
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    backend_dev = _backend_device(group)
    B = storage.num_buckets()
    mine = torch.from_numpy(np.concatenate([storage.bucket_sizes(), storage.owned_buckets().astype(np.int64)])).to(backend_dev)
    allv = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(allv, mine, group=group)
    allv = torch.stack(allv).cpu().numpy()
    bsz_all, owned_all = allv[:, :B], allv[:, B:].astype(bool)
    if not (owned_all.sum(axis=0) == 1).all():
        raise ValueError("every bucket must be owned by exactly one rank (sets from one distributed count)")
    if (bsz_all[~owned_all] != 0).any():
        raise ValueError("a rank holds records of a bucket it does not own")
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
        desc = np.zeros(SGPU_IPC_BYTES, np.uint8)
        for name, step in (("merge", L.sgpu_dist_cov_bound), ("fill", L.sgpu_dist_cov_fill)):
            # descriptors of the registers, then of the table slices; the all_gather also orders the steps across the ranks
            ctx.check(L.sgpu_dist_cov_ipc_handle(h, desc.ctypes.data_as(C.c_void_p)))
            t_h = torch.from_numpy(desc).to(backend_dev)
            hs = [torch.empty_like(t_h) for _ in range(world)]
            dist.all_gather(hs, t_h, group=group)
            descs = np.ascontiguousarray(torch.stack(hs).cpu().numpy())
            ctx.check(L.sgpu_dist_cov_open_peers(h, descs.ctypes.data_as(C.c_void_p)))
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
