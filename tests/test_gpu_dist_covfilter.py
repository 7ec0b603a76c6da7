"""The coverage pre-filter across ranks (sgpu_dist_cov_*, spades_b200.distributed.distributed_cov_filter). CPU: the owner and
slice-capacity arithmetic and the exported symbols. GPU: every case of dist_cov_worker.CASES with W = 1 .. 4 processes on device 0,
each with its own context and arena, joined by gloo, against sgpu_reads_cov_filter over the union and the oracle."""
import ctypes as C
import gc
import os
import socket
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_PROCESS_BYTES = 3 << 29        # what one more process costs on the device next to its arena: CUDA context, modules, torch


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_library_exports_the_distributed_filter():
    from spades_b200 import _lib
    L = C.CDLL(_lib.LIB_PATH)
    names = [s for s in _lib.SYMBOLS if s.startswith("sgpu_dist_cov_")]
    assert len(names) == 8
    for s in names:
        assert hasattr(L, s), s


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_owner_and_slice_capacity(world):
    """owner = high word of (key x 0xC2B2AE3D27D4EB4F mod 2^64) x world; a slice holds 1.5 x the even share of the bound plus
    8 x sqrt(share) entries (at least 1024), so the ranks' slices together exceed the single-GPU table"""
    from spades_b200.distributed import cov_layout_host
    rng = np.random.default_rng(world)
    keys = rng.integers(0, 1 << 47, 200000, dtype=np.uint64)
    keys[:4] = [0, 1, (1 << 47) - 1, 12345]
    owners, _ = cov_layout_host(world, 0, keys)
    want = [((int(k) * 0xC2B2AE3D27D4EB4F) % (1 << 64)) * world >> 64 for k in keys.tolist()]
    assert owners.tolist() == want
    share = np.bincount(owners, minlength=world) / len(keys)
    assert np.all(np.abs(share - 1 / world) < 0.01)
    for maxn in [0, 1, 1000, 3300, 864_000_000, 1 << 38]:
        _, cap = cov_layout_host(world, maxn, np.zeros(0, np.uint64))
        s = -(-maxn // world)
        assert cap == max(1024, s + s // 2 + 8 * int(np.ceil(np.sqrt(s))))
        assert cap * world >= maxn + maxn // 2
    with pytest.raises(ValueError):
        cov_layout_host(0, 10, keys)


def test_owner_skew_case_is_built_as_intended():
    """with two or more ranks the owner-skew reads put ~90 % of a slice's capacity on rank 0, above 1.5 x the even share, at a fixed
    key width"""
    import oracle as O
    from dist_cov_worker import owner_skew
    from spades_b200.distributed import cov_layout_host
    from spades_b200.packing import pack_reads
    for world in (1, 2, 3, 4):
        shards, owned0 = owner_skew(world)
        union = [r for s in shards for r in s]
        _, st = O.cov_filter(*pack_reads(union), 32, 1)
        assert st[1] == 21
        _, cap = cov_layout_host(world, st[0], np.zeros(0, np.uint64))
        assert owned0 < cap
        if world > 1:                # (one rank owns every key: 3 000 of a 5 412-entry slice)
            assert owned0 >= 0.85 * cap and owned0 > 3 * (-(-st[0] // world)) // 2


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_distributed_cov_filter_one_device(world, tmp_path):
    """W processes on device 0: register merge through the mapped arenas, owner slices filled with remote CAS, verdicts from the
    owners' slices, compaction; then the distributed count of the survivors for the cases that ask for it. W = 1 is the branch
    without IPC."""
    import torch
    import torch.multiprocessing as mp
    import gpu_util
    from dist_cov_worker import ARENA_BYTES, CASES, run_spawned
    gpu_util.release()               # the session's shared context holds most of the device memory
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
    if lines and lines[0].startswith("SKIP"):
        pytest.skip(lines[0][5:])
    assert len(lines) == len(CASES), "%d result lines for %d cases" % (len(lines), len(CASES))
    for case, line in zip(CASES, lines):
        assert (" W=%d %s " % (world, case["name"])) in line, line
    bad = [ln for ln in lines if not ln.endswith(" OK")]
    assert not bad, "\n".join(bad)
