"""N>1 path. CPU: the exchange planning under a real world_size-2 gloo group. GPU: the distributed count of every case of
dist_worker.CASES against the oracle, with W ranks sharing device 0 (always runs), and with one GPU per rank over NCCL
(when two or more GPUs are visible)."""
import gc
import os
import socket
import subprocess
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_PROCESS_BYTES = 3 << 29        # what one more process costs on the device next to its arena: CUDA context, modules, torch


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_exchange_plan_world2_gloo():
    import torch.multiprocessing as mp
    from dist_worker import run_plan
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(run_plan, args=(world, port, out), nprocs=world, join=True)
    assert all(out.get(r) for r in range(world)), dict(out)


def test_plan_keeps_a_set_within_128_chunks():
    """a budget that fits one bucket per pass: the distributed count still makes at most 128 passes (the chunks a set may hold),
    each an even split of the buckets"""
    import numpy as np
    from spades_b200.distributed import plan_host
    world, B, rA = 2, 300, 2
    counts = np.random.default_rng(3).integers(1, 5000, size=(world, B << rA)).astype(np.uint64)
    npass, bounds, _ = plan_host(world, B, rA, counts, 1, 16)
    assert npass == 128
    assert bounds[0] == 0 and bounds[-1] == B
    assert set(np.diff(bounds).tolist()) == {2, 3}


def _check_lines(lines, world):
    from dist_worker import CASES
    assert len(lines) == len(CASES), "%d result lines for %d cases" % (len(lines), len(CASES))
    for case, line in zip(CASES, lines):
        assert (" W=%d %s " % (world, case["name"])) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_count_one_device(world, tmp_path):
    """W processes with their own context and arena on device 0, joined by gloo: level-A histograms, all-gathered partition
    counts, per-pass planning, staging + IPC descriptor exchange, the pull kernel reading the other processes' staging buffers
    through mapped arenas, sort and compaction at the owner, per-rank MPHF. W = 1 is the branch without IPC, W = 3 an
    uneven ownership split."""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_worker import ARENA_BYTES, CASES, run_spawned
    gpu_util.release()               # the session's shared context holds most of the device memory
    gc.collect()
    free, total = torch.cuda.mem_get_info(0)
    need = world * (ARENA_BYTES + CUDA_PROCESS_BYTES)
    if free < need:
        pytest.skip("device 0 has %.2f GiB free of %.2f GiB; %d ranks need %.2f GiB (%.2f GiB arena + %.2f GiB process overhead each)"
                    % (free / 2**30, total / 2**30, world, need / 2**30, ARENA_BYTES / 2**30, CUDA_PROCESS_BYTES / 2**30))
    out = tmp_path / "lines.txt"
    t0 = time.time()
    mp.spawn(run_spawned, args=(world, _free_port(), str(out), CASES), nprocs=world, join=True)
    lines = out.read_text().splitlines()          # rank 0 has printed them as it went
    print("W=%d: %d cases in %.1f s" % (world, len(lines), time.time() - t0))
    if lines and lines[0].startswith("SKIP"):
        pytest.skip(lines[0][5:])
    _check_lines(lines, world)


@pytest.mark.gpu
def test_distributed_count_two_gpus():
    """the same cases with one GPU per rank over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "dist_worker.py")], capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-6000:]); sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0
    _check_lines([ln for ln in r.stdout.splitlines() if ln.startswith("dist case ")], 2)
