"""Multi-GPU k-mer counting: one process per GPU, torch.distributed for the small tables and the barriers,
the record exchange itself is one kernel over NVLink peer memory (sgpu_dist_exchange: pull + merge).

Mirrors what hpcspades distributes with MPI tasks + a shared filesystem (projects/hpcspades/mpi/stages/construction_mpi.cpp:222-300):
every rank reads its own slice of the reads; afterwards every bucket lives on exactly one rank.
"""
import ctypes as C

import numpy as np

from .kmer_index import KMerDiskStorage, SGPU_CANONICAL, SGPU_RESULT_ON_HOST

SGPU_IPC_BYTES = 96


class DistributedKMerCounter:
    """KMerDiskCounter over a read set sharded across the ranks of a torch.distributed process group. result_on_host: each rank's
    set goes to its pinned host memory, pass by pass behind the next one."""

    def __init__(self, ctx, K, mode=SGPU_CANONICAL, group=None, result_on_host=False):
        self.ctx, self.K, self.mode, self.group, self.result_on_host = ctx, K, mode, group, result_on_host
        self.npass = 0

    def close(self):
        pass

    def Count(self, num_buckets, budget_bytes=None):
        import torch
        import torch.distributed as dist
        ctx, L = self.ctx, self.ctx.L
        world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        backend_dev = "cuda" if dist.get_backend(self.group) == "nccl" else "cpu"
        h = C.c_void_p()
        mode = self.mode | (SGPU_RESULT_ON_HOST if self.result_on_host else 0)
        ctx.check(L.sgpu_dist_begin(ctx.h, self.K, num_buckets, mode, world, rank, C.byref(h)))
        try:
            npart = L.sgpu_dist_num_partitions(h)
            local = np.zeros(npart, np.uint64)
            ctx.check(L.sgpu_dist_local_counts(h, local.ctypes.data_as(C.c_void_p)))
            # all_gather of the per-partition record counts (world x npart x 8 bytes: small)
            t_local = torch.from_numpy(local.view(np.int64)).to(backend_dev)
            gathered = [torch.empty_like(t_local) for _ in range(world)]
            dist.all_gather(gathered, t_local, group=self.group)
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
                    dist.all_reduce(tb, op=dist.ReduceOp.MIN, group=self.group)
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
                dist.all_gather(hs, t_h, group=self.group)
                descs = np.ascontiguousarray(torch.stack(hs).cpu().numpy())
                ctx.check(L.sgpu_dist_open_peers(h, descs.ctypes.data_as(C.c_void_p)))     # peers' arenas are mapped once per process
                ctx.check(L.sgpu_dist_scatter(h, p.value))    # local partition into the staging buffer
                dist.barrier(group=self.group)                # every rank's staging buffer is complete
                ctx.check(L.sgpu_dist_exchange(h, p.value))   # one kernel: pull my pieces from all peers over NVLink + merge
                dist.barrier(group=self.group)                # nobody reads my staging buffer any more (it becomes the sort's partner)
                ctx.check(L.sgpu_dist_sort(h, p.value))
                npass += 1
            dist.barrier(group=self.group)
            ks = C.c_void_p()
            ctx.check(L.sgpu_dist_end(h, C.byref(ks)))
            self.npass = npass
            return KMerDiskStorage(ctx, ks)
        finally:
            L.sgpu_dist_free(h)


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
    backend_dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
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
