"""The early tip and A/T clippers across ranks (DistributedGraphConstructor.ConstructGraph with the clippers on) against one GPU over
the union and the oracle. GPU: every case of dist_clip_worker.CASES with W ranks sharing device 0 (gloo), and with one GPU per rank
over NCCL when two or more GPUs are visible; every reference fixture of the clippers at W = 2 and 3; the refusals. CPU: the new C
entries refuse null arguments without a device."""
import ctypes as C
import gc
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import golden_util as G
from test_distributed import CUDA_PROCESS_BYTES, _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spawn(world, what, tmp_path):
    """W processes with their own context and arena on device 0, joined by gloo; rank 0's result lines"""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_clip_worker import ARENA_BYTES, run_spawned
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
    from dist_clip_worker import CASES
    assert len(lines) == len(CASES), "%d result lines for %d cases" % (len(lines), len(CASES))
    for case, line in zip(CASES, lines):
        assert (" W=%d %s " % (world, case["name"])) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_clippers_one_device(world, tmp_path):
    """the whole distributed chain with the clippers on: the union's clipper statistics, clipped masks, unitigs and GFA equal the
    single-GPU build's and the oracle's; at W >= 2 some marks, roots or bit clears land in another rank's slice"""
    _check_lines(_spawn(world, "cases", tmp_path), world)


@pytest.mark.gpu
def test_distributed_clippers_two_gpus():
    """the same cases with one GPU per rank over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "dist_clip_worker.py")], capture_output=True, text=True,
                       timeout=1800)
    sys.stdout.write(r.stdout[-6000:]); sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0
    _check_lines([ln for ln in r.stdout.splitlines() if ln.startswith("dist clip ")], 2)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_distributed_clippers_reference_fixtures(world, tmp_path):
    """every *_tcgraph and *_atgraph fixture of the unmodified reference through the distributed path: masks, removed k-mers,
    unitigs and GFA"""
    names = G.names("tcgraph") + G.names("atgraph")
    lines = _spawn(world, names, tmp_path)
    assert len(lines) == len(names)
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2])
def test_distributed_clippers_refusals(world, tmp_path):
    """bad A/T parameters (SGPU_EINVAL on every rank), options that differ between the ranks (ValueError) and phase entries called
    out of order are refused, and the context stays usable"""
    lines = _spawn(world, "refusals", tmp_path)
    assert lines == ["dist clip refusals W=%d OK" % world]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_new_entries_refuse_null_arguments_without_a_device():
    from spades_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    owners = np.zeros(4, np.int32)
    sizes = np.zeros(4, np.uint64)
    opts = _lib.SgpuGraphOptions(1, 79, 1, 0.8, 10, 200)
    assert L.sgpu_dist_graph_begin_opts(None, None, _p(owners), None, _p(sizes), 0, C.byref(opts), C.byref(h)) == 2    # SGPU_EINVAL
    assert L.sgpu_dist_graph_begin_opts(None, None, _p(owners), None, _p(sizes), 0, None, C.byref(h)) == 2
    for name in ("at_edges_probe", "at_edges_apply", "at_tips_probe", "tip_probe", "isolate", "unlink", "junctions"):
        assert getattr(L, "sgpu_dist_graph_" + name)(None) == 2, name
    out = np.zeros(4, np.uint64)
    assert L.sgpu_dist_graph_masks(None, None, 0) == 2
    assert L.sgpu_dist_graph_clipper_stats(None, _p(out), _p(out), _p(out)) == 2
    assert L.sgpu_dist_graph_clipper_times(None, _p(np.zeros(6, np.float32))) == 2
