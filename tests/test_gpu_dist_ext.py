"""The extension masks, coverage and histogram across ranks (DistributedExtensionIndexBuilder) against one GPU over the union.
GPU: every case of dist_ext_worker.CASES with W ranks sharing device 0 (gloo), and with one GPU per rank over NCCL when two or
more GPUs are visible. CPU: the new C entries refuse bad arguments without a device, and the pass plan of the masks."""
import ctypes as C
import gc
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from test_distributed import CUDA_PROCESS_BYTES, _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check_lines(lines, world):
    from dist_ext_worker import CASES
    assert len(lines) == len(CASES), "%d result lines for %d cases" % (len(lines), len(CASES))
    for case, line in zip(CASES, lines):
        assert (" W=%d %s " % (world, case["name"])) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_extension_index_one_device(world, tmp_path):
    """W processes with their own context and arena on device 0, joined by gloo: distributed (k+1)-mer count, distributed k-mers,
    both indexes and the distributed masks and coverage, checked on rank 0 against the single-GPU graph build over the union and
    the oracle"""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_ext_worker import ARENA_BYTES, CASES, run_spawned
    gpu_util.release()
    gc.collect()
    free, total = torch.cuda.mem_get_info(0)
    need = world * (ARENA_BYTES + CUDA_PROCESS_BYTES)
    if free < need:
        pytest.skip("device 0 has %.2f GiB free of %.2f GiB; %d ranks need %.2f GiB" % (free / 2**30, total / 2**30, world, need / 2**30))
    out = tmp_path / "lines.txt"
    t0 = time.time()
    mp.spawn(run_spawned, args=(world, _free_port(), str(out), CASES), nprocs=world, join=True)
    lines = out.read_text().splitlines()
    print("W=%d: %d cases in %.1f s" % (world, len(lines), time.time() - t0))
    _check_lines(lines, world)


@pytest.mark.gpu
def test_distributed_extension_index_two_gpus():
    """the same cases with one GPU per rank over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "dist_ext_worker.py")], capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-6000:]); sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0
    _check_lines([ln for ln in r.stdout.splitlines() if ln.startswith("dist ext ")], 2)


def test_new_entries_refuse_bad_arguments_without_a_device():
    from spades_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    owners = np.zeros(4, np.int32)
    assert L.sgpu_dist_ext_begin(None, None, None, None, None, owners.ctypes.data_as(C.c_void_p), 1, 0, C.byref(h)) == 2    # SGPU_EINVAL
    assert L.sgpu_dist_ext_local_counts(None, None) == 2
    assert L.sgpu_dist_ext_plan(None, None, None) == 2
    assert L.sgpu_dist_ext_free_bytes(None, None) == 2
    assert L.sgpu_dist_ext_next_pass(None, 0, None) == 2
    assert L.sgpu_dist_ext_ipc_handle(None, None) == 2
    assert L.sgpu_dist_ext_open_peers(None, None) == 2
    assert L.sgpu_dist_ext_scatter(None, 0) == 2
    assert L.sgpu_dist_ext_apply(None, 0) == 2
    assert L.sgpu_dist_ext_masks(None, None, 0) == 2
    assert L.sgpu_dist_ext_coverage(None, None, 0) == 2
    assert L.sgpu_dist_ext_histogram(None, None, 0) == -1
    assert L.sgpu_dist_ext_times(None, None) == 2
    L.sgpu_dist_ext_free(None)


def test_host_plan_refuses_bad_owner_tables():
    from spades_b200.distributed import ext_plan_host
    counts = np.ones((2, 4), np.uint64)
    with pytest.raises(ValueError):
        ext_plan_host(2, [0, 1, 2, 0], counts, 1 << 20, 17)       # owner 2 of a world of 2
    with pytest.raises(ValueError):
        ext_plan_host(2, [0, -1, 1, 0], counts, 1 << 20, 17)
    with pytest.raises(ValueError):
        ext_plan_host(0, [0, 0, 0, 0], counts, 1 << 20, 17)
    with pytest.raises(ValueError):
        ext_plan_host(2, np.zeros(8193, np.int32), np.ones((2, 8193), np.uint64), 1 << 20, 17)


def _priced(owners, counts, a, b):
    """the most records any rank sends or any owner receives if buckets [a, b) are one pass"""
    world = counts.shape[0]
    sent = counts[:, a:b].sum(axis=1)
    recv = [counts[:, a:b][:, owners[a:b] == g].sum() for g in range(world)]
    return int(max(sent.max(), max(recv)))


@pytest.mark.parametrize("world,B,seed", [(1, 1, 0), (1, 64, 1), (3, 100, 2), (4, 3, 3), (2, 8192, 4), (5, 700, 5)])
def test_host_plan_covers_every_bucket_once_within_the_budget(world, B, seed):
    from spades_b200.distributed import ext_plan_host
    rng = np.random.default_rng(seed)
    owners = rng.integers(0, world, B).astype(np.int32)
    counts = rng.integers(0, 5000, (world, B)).astype(np.uint64)
    counts[:, rng.integers(0, B, max(1, B // 10))] = 0
    rb = 17
    total = int(counts.sum())
    for budget in (10 * total * rb + 1, total * rb // 7 + 1, total * rb // 40 + 1, 1):
        n, bounds, most = ext_plan_host(world, owners, counts, budget, rb)
        # every destination bucket lies in exactly one pass
        assert bounds[0] == 0 and bounds[-1] == B and len(bounds) == n + 1
        assert (np.diff(bounds) > 0).all()
        priced = [_priced(owners, counts, int(bounds[p]), int(bounds[p + 1])) for p in range(n)]
        assert most == max(priced)
        if budget > total * rb:
            assert n == 1
        capped = n == min(B, 256) and any(p * rb > budget for p in priced)
        for p in range(n):
            a, b = int(bounds[p]), int(bounds[p + 1])
            if priced[p] * rb <= budget or b - a == 1:
                continue
            # over the budget: only when the budget needs more passes than the plan may make, and then an even split of the buckets
            assert capped, (budget, p, priced[p] * rb)
            left = min(B, 256) - p
            assert b - a <= -(-(B - a) // left), (a, b, left)


def test_host_plan_even_split_when_the_budget_is_too_small():
    from spades_b200.distributed import ext_plan_host
    rng = np.random.default_rng(9)
    B = 1000
    n, bounds, _ = ext_plan_host(2, rng.integers(0, 2, B), rng.integers(1, 100, (2, B)), 1, 17)
    assert n == 256
    assert set(np.diff(bounds).tolist()) <= {3, 4}
