"""The k-mers of a distributed (k+1)-mer set, the union's index assembled from the owners' buckets, and the owned bucket files.
GPU: every case of dist_kmers_worker.CASES with W ranks sharing device 0 (gloo), and with one GPU per rank over NCCL when two or
more GPUs are visible. CPU: the new C entries refuse bad arguments without a device."""
import ctypes as C
import gc
import os
import subprocess
import sys
import time

import pytest

from test_distributed import CUDA_PROCESS_BYTES, _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check_lines(lines, world):
    from dist_kmers_worker import CASES, expected_lines
    assert len(lines) == expected_lines(CASES), "%d result lines for %d counts" % (len(lines), expected_lines(CASES))
    names = [c["name"] for c in CASES for _ in range(1 + ("Bk2" in c))]
    for name, line in zip(names, lines):
        assert (" W=%d %s " % (world, name)) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_kmers_one_device(world, tmp_path):
    """W processes with their own context and arena on device 0, joined by gloo: the distributed (k+1)-mer count of the read
    shards, then the distributed k-mers of its shards (or of overlapping whole sets), checked on rank 0 against the oracle and the
    single-GPU path over the union of the reads"""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_kmers_worker import ARENA_BYTES, CASES, run_spawned
    gpu_util.release()
    gc.collect()
    free, total = torch.cuda.mem_get_info(0)
    need = world * (ARENA_BYTES + CUDA_PROCESS_BYTES)
    if free < need:
        pytest.skip("device 0 has %.2f GiB free of %.2f GiB; %d ranks need %.2f GiB (%.2f GiB arena + %.2f GiB process overhead each)"
                    % (free / 2**30, total / 2**30, world, need / 2**30, ARENA_BYTES / 2**30, CUDA_PROCESS_BYTES / 2**30))
    out = tmp_path / "lines.txt"
    t0 = time.time()
    mp.spawn(run_spawned, args=(world, _free_port(), str(out), CASES), nprocs=world, join=True)
    lines = out.read_text().splitlines()
    print("W=%d: %d counts in %.1f s" % (world, len(lines), time.time() - t0))
    if lines and lines[0].startswith("SKIP"):
        pytest.skip(lines[0][5:])
    _check_lines(lines, world)


@pytest.mark.gpu
def test_distributed_kmers_two_gpus():
    """the same cases with one GPU per rank over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "dist_kmers_worker.py")], capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-6000:]); sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0
    _check_lines([ln for ln in r.stdout.splitlines() if ln.startswith("dist kmers ")], 2)


def test_new_entries_refuse_bad_arguments_without_a_device():
    from spades_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    assert L.sgpu_dist_begin_kpomers(None, None, 16, 0, 1, 0, C.byref(h)) == 2          # SGPU_EINVAL
    assert L.sgpu_kset_owned_buckets(None, None) == 2
    assert L.sgpu_kset_write_owned_buckets(None, b"/nonexistent/prefix") == 2
    assert L.sgpu_mphf_serialized_size_buckets(None, 0, 1) == -1
    assert L.sgpu_mphf_serialize_buckets(None, 0, 1, None, 0) == 2


@pytest.mark.gpu
def test_source_freed_while_counting_is_released_at_the_end():
    """sgpu_kset_free of the (k+1)-mer set a distributed count reads defers the release to sgpu_dist_free: the count still reads the
    whole set and gives the single-GPU k-mers"""
    import numpy as np
    import torch.distributed as dist
    import gpu_util
    from dist_kmers_worker import ARENA_BYTES
    from spades_b200.distributed import _distributed_count
    from spades_b200.kmer_index import Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter
    from spades_b200.packing import pack_reads, synthetic_reads
    gpu_util.release()
    gc.collect()
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1)
    ctx = Context(0, hbm_budget_bytes=ARENA_BYTES)
    try:
        ctx.set_reads(*pack_reads(synthetic_reads(2000, 150, 3000, 0.01, seed=31)))
        kp_ref = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(56)).Count(8)
        want = KMerDiskCounter(ctx, DeBruijnKMerKMerSplitter(55, kp_ref)).Count(8)
        kp = KMerDiskCounter(ctx, DeBruijnReadKMerSplitter(56), result_on_host=True).Count(8)

        def begin(world, rank, out):
            rc = ctx.L.sgpu_dist_begin_kpomers(ctx.h, kp.h, 8, 0, world, rank, out)
            kp.free()
            return rc
        got, _ = _distributed_count(ctx, None, begin, None)
        assert np.array_equal(got.kmers(), want.kmers())
        assert np.array_equal(got.bucket_sizes(), want.bucket_sizes())
        got.free(); want.free(); kp_ref.free()
    finally:
        ctx.close()
        dist.destroy_process_group()
