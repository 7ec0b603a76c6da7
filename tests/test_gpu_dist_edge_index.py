"""The EdgeIndex refill across ranks (DistributedEdgeIndex) against one GPU's EdgeIndex over the union and the oracle. GPU: every case
of dist_edge_index_worker.CASES with W ranks sharing device 0 (gloo), and with one GPU per rank over NCCL when two or more GPUs are
visible; every *_eigraph reference fixture at W = 2 and 3; arguments that differ between the ranks. CPU (test_dist_edge_index.py):
the edge numbering, the single-index decision, the slot ranges and the null refusals."""
import gc
import os
import subprocess
import sys
import time

import pytest

import golden_util as G
from test_distributed import CUDA_PROCESS_BYTES, _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spawn(world, what, tmp_path):
    """W processes with their own context and arena on device 0, joined by gloo; rank 0's result lines"""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_edge_index_worker import ARENA_BYTES, run_spawned
    gpu_util.release()
    gc.collect()
    free, total = torch.cuda.mem_get_info(0)
    need = world * (ARENA_BYTES + CUDA_PROCESS_BYTES)
    if free < need:
        pytest.skip("device 0 has %.2f GiB free of %.2f GiB; %d ranks need %.2f GiB" % (free / 2**30, total / 2**30, world, need / 2**30))
    out = tmp_path / "lines.txt"
    t0 = time.time()
    mp.spawn(run_spawned, args=(world, _free_port(), str(out), what), nprocs=world, join=True)
    lines = out.read_text().splitlines()
    print("W=%d: %d lines in %.1f s" % (world, len(lines), time.time() - t0))
    print("\n".join(lines))
    return lines


def _check_lines(lines, world):
    from dist_edge_index_worker import CASES
    assert len(lines) == len(CASES), "%d result lines for %d cases" % (len(lines), len(CASES))
    for case, line in zip(CASES, lines):
        assert (" W=%d %s " % (world, case["name"])) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_edge_index_one_device(world, tmp_path):
    """the whole distributed chain up to the EdgeIndex: every rank's serialized index and lookups equal one GPU's over the union,
    and the assembled values equal one GPU's and, for the small cases, the oracle's"""
    _check_lines(_spawn(world, "cases", tmp_path), world)


@pytest.mark.gpu
def test_distributed_edge_index_two_gpus():
    """the same cases with one GPU per rank over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "dist_edge_index_worker.py")], capture_output=True,
                       text=True, timeout=1800)
    sys.stdout.write(r.stdout[-6000:]); sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0
    _check_lines([ln for ln in r.stdout.splitlines() if ln.startswith("dist edge index W=")], 2)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_distributed_edge_index_reference_fixtures(world, tmp_path):
    """every *_eigraph fixture of the unmodified reference through the distributed path: serialized index, edge ids and offsets"""
    names = G.names("eigraph")
    lines = _spawn(world, names, tmp_path)
    assert len(lines) == len(names)
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2])
def test_distributed_edge_index_refusals(world, tmp_path):
    """K or num_buckets that differ between the ranks raise ValueError on every rank before any collective of the build, and the
    same context then builds an index that matches one GPU's"""
    lines = _spawn(world, "refusals", tmp_path)
    assert lines == ["dist edge index refusals W=%d OK" % world]
