"""The unitigs and perfect loops across ranks (DistributedGraphConstructor + assemble_graph) against one GPU over the union.
GPU: every case of dist_graph_worker.CASES with W ranks sharing device 0 (gloo), and with one GPU per rank over NCCL when two or
more GPUs are visible. CPU: the new C entries refuse bad arguments without a device, and a host-only graph refuses inconsistent
edges and the device accessors."""
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
    from dist_graph_worker import CASES
    assert len(lines) == len(CASES), "%d result lines for %d cases" % (len(lines), len(CASES))
    for case, line in zip(CASES, lines):
        assert (" W=%d %s " % (world, case["name"])) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_graph_one_device(world, tmp_path):
    """W processes with their own context and arena on device 0, joined by gloo: the whole distributed chain up to the assembled
    graph, checked on rank 0 against the single-GPU graph build over the union and the oracle"""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_graph_worker import ARENA_BYTES, CASES, run_spawned
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
def test_distributed_graph_two_gpus():
    """the same cases with one GPU per rank over NCCL"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "dist_graph_worker.py")], capture_output=True, text=True,
                       timeout=1800)
    sys.stdout.write(r.stdout[-6000:]); sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0
    _check_lines([ln for ln in r.stdout.splitlines() if ln.startswith("dist graph ")], 2)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_new_entries_refuse_bad_arguments_without_a_device():
    from spades_b200 import _lib
    L = _lib.load()
    h = C.c_void_p()
    owners = np.zeros(4, np.int32)
    sizes = np.zeros(4, np.uint64)
    assert L.sgpu_dist_graph_begin(None, None, _p(owners), None, _p(sizes), 0, C.byref(h)) == 2    # SGPU_EINVAL
    assert L.sgpu_dist_graph_ipc_handle(None, None) == 2
    assert L.sgpu_dist_graph_open_peers(None, None) == 2
    assert L.sgpu_dist_graph_unitigs(None) == 2
    assert L.sgpu_dist_graph_clear_visited(None) == 2
    assert L.sgpu_dist_graph_loops(None) == 2
    assert L.sgpu_dist_graph_stats(None, None) == 2
    assert L.sgpu_dist_graph_edges(None, None, None, None, None, None) == 2
    assert L.sgpu_dist_graph_bucket_counts(None, None, None) == 2
    assert L.sgpu_dist_graph_times(None, None) == 2
    L.sgpu_dist_graph_free(None)
    assert L.sgpu_graph_from_edges(21, None, 0, None, None, None, None, 0, None) == 2


def _edges(k, lens):
    rng = np.random.default_rng(3)
    text = "".join("ACGT"[c] for c in rng.integers(0, 4, int(sum(lens)))).encode()
    n = len(lens)
    return text, np.asarray(lens, np.uint32), np.arange(n, dtype=np.uint64) << 2 | 1, (np.arange(n, dtype=np.uint64) + 7) << 2, np.ones(n, np.uint32)


def test_graph_from_edges_refuses_inconsistent_edges():
    from spades_b200 import _lib
    L = _lib.load()
    k = 5
    text, lens, ls, le, rc = _edges(k, [6, 9, 12])
    buf = np.frombuffer(text, np.uint8)
    h = C.c_void_p()

    def make(nbases, lens_):
        return L.sgpu_graph_from_edges(k, _p(buf), nbases, _p(lens_), _p(ls), _p(le), _p(rc), len(lens_), C.byref(h))
    assert make(len(text) - 1, lens) == 2                                  # the last edge reaches past the text
    assert make(len(text), np.asarray([6, 9, 12 + 4], np.uint32)) == 2     # an offset past the text
    assert make(len(text), np.asarray([5, 10, 12], np.uint32)) == 2        # a length below k + 1
    assert make(len(text), np.asarray([6, 9, 11], np.uint32)) == 2         # lengths and text size disagree
    assert make(len(text), np.asarray([6, 9, 12], np.uint32)) == 0
    g = h
    assert L.sgpu_graph_num_unitigs(g) == 3 and L.sgpu_graph_unitig_bases(g) == len(text)
    assert L.sgpu_graph_gfa(g, b"v", None, 0) > 0
    out = np.zeros(len(text), np.uint8)
    assert L.sgpu_graph_masks(g, _p(out), 1) == 2
    assert L.sgpu_graph_coverage(g, _p(out), 1) == 2
    assert L.sgpu_graph_histogram(g, None, 0) == -1
    assert L.sgpu_graph_tip_clipper_stats(g, _p(np.zeros(3, np.uint64))) == 2
    assert L.sgpu_graph_at_clipper_stats(g, _p(np.zeros(4, np.uint64))) == 2
    L.sgpu_graph_free(g)


def test_graph_from_edges_python_refuses_array_sizes_that_disagree():
    from spades_b200.distributed import graph_from_edges
    text, lens, ls, le, rc = _edges(5, [6, 9, 12])
    with pytest.raises(ValueError):
        graph_from_edges(5, text, lens, ls[:2], le, rc)
    with pytest.raises(ValueError):
        graph_from_edges(5, text, lens, ls, le, rc[:1])
    with pytest.raises(ValueError):
        graph_from_edges(5, text[:-1], lens, ls, le, rc)
    g = graph_from_edges(5, text, lens, ls, le, rc)
    assert g.unitigs() == [text[:6].decode(), text[6:15].decode(), text[15:].decode()]
    assert g.gfa().startswith("H\tsp:Z:SPAdes-4.3.0-dev\nS\t3\t")
    g.free()
