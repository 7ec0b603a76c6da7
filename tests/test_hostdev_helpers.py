"""CPU: the __host__ __device__ arithmetic of spades_b200/csrc/kmer_dev.cuh (host compilation) against the oracle.
The same functions are re-checked on the device in test_gpu_parity.py::test_device_arithmetic."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
from spades_b200 import _lib


def run_selftest(ctx_h, on_device, op, K, arg, keys):
    L = _lib.load()
    keys = np.ascontiguousarray(keys, np.uint64)
    n = keys.shape[0]
    out = np.zeros(n, np.uint64)
    rc = L.sgpu_selftest(ctx_h, on_device, op, K, arg, keys.ctypes.data_as(C.c_void_p), n, out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out


def random_kmers(K, n, seed):
    rng = np.random.default_rng(seed)
    nw = (K + 31) // 32
    codes = rng.integers(0, 4, size=(n, nw * 32), dtype=np.uint64)
    codes[:, K:] = 0
    # a few palindromes / extremes
    codes[0, :K] = 0
    codes[1, :K] = 3
    if K % 2 == 0:
        half = codes[2, :K // 2].copy()
        codes[2, K // 2:K] = (3 - half)[::-1]
    sh = (np.arange(32, dtype=np.uint64) * np.uint64(2))
    return (codes.reshape(n, nw, 32) << sh).sum(axis=2, dtype=np.uint64)


def check_all(ctx_h, on_device):
    Lo = O.lib()
    for K in (1, 5, 21, 22, 31, 32, 33, 55, 56, 63, 64, 65, 77, 78, 96, 97, 127, 128):
        keys = random_kmers(K, 64, K)
        nw = keys.shape[1]
        h64 = run_selftest(ctx_h, on_device, 0, K, 0, keys)
        lo = run_selftest(ctx_h, on_device, 1, K, 0, keys)
        hi = run_selftest(ctx_h, on_device, 2, K, 0, keys)
        bk = run_selftest(ctx_h, on_device, 3, K, 1234, keys)
        mn = run_selftest(ctx_h, on_device, 4, K, 0, keys)
        rcw = [run_selftest(ctx_h, on_device, 5 + j, K, 0, keys) for j in range(nw)]
        for i, k in enumerate(keys):
            assert int(h64[i]) == O.xxh3_64(k)
            assert (int(lo[i]), int(hi[i])) == O.xxh3_128(k)
            assert int(bk[i]) == int(Lo.orc_bucket(k.ctypes.data_as(C.c_void_p), nw, 1234))
            assert int(mn[i]) == int(Lo.orc_is_minimal(k.ctypes.data_as(C.c_void_p), K))
            r = np.zeros(nw, np.uint64)
            Lo.orc_rc(k.ctypes.data_as(C.c_void_p), K, r.ctypes.data_as(C.c_void_p))
            assert [int(rcw[j][i]) for j in range(nw)] == [int(x) for x in r]
        # MSD digit extraction against a bit-string model
        total = 2 * K
        for pos, r_ in ((0, 8), (3, 11), (max(0, total - 5), 8), (60, 12), (64, 7), (120, 32), (total, 8)):
            if pos > total:
                continue
            got = run_selftest(ctx_h, on_device, 9, K, (pos << 8) | r_, keys)
            for i, k in enumerate(keys):
                bits = ""
                for j in range(nw):
                    wb = 64 if j < nw - 1 else total - 64 * (nw - 1)
                    bits += format(int(k[j]) & ((1 << wb) - 1), "0%db" % wb)
                want = int((bits[pos:pos + r_] + "0" * r_)[:r_], 2)
                assert int(got[i]) == want, (K, pos, r_, i)


def check_roll(ctx_h, on_device):
    """op 10: the rolling window + rolling reverse complement of the level-A kernels (kmer_dev.cuh roll_init/roll_next)
    against direct window extraction + FastRC, for every window of sequences whose lengths straddle word boundaries, in the
    chunks of both strand modes: 24 windows (canonical) and 12 windows (all windows, two records per window)."""
    rng = np.random.default_rng(99)
    for C_ in (24, 12):
        for K in (1, 2, 5, 21, 22, 31, 32, 33, 55, 56, 63, 64, 65, 77, 78, 96, 97, 127, 128):
            nw = (K + 31) // 32
            for L in (K, K + 1, K + C_ - 1, K + C_, K + C_ + 1, 150, 151, 192, 257, 1000):
                if L < K:
                    continue
                nwords = (L + 31) // 32
                nrec = max((nwords + nw - 1) // nw, (L - K + 1 + C_ - 1) // C_ + 1)
                codes = np.zeros(nrec * nw * 32, np.uint64)
                codes[:L] = rng.integers(0, 4, L, dtype=np.uint64)
                sh = (np.arange(32, dtype=np.uint64) * np.uint64(2))
                words = (codes.reshape(-1, 32) << sh).sum(axis=1, dtype=np.uint64).reshape(nrec, nw)
                out = run_selftest(ctx_h, on_device, 10, K, (C_ << 32) | L, words)
                nwin = L - K + 1
                for u in range(nrec):
                    cnt = min(C_, max(0, nwin - C_ * u))
                    assert int(out[u]) == (cnt << 32), (C_, K, L, u, hex(int(out[u])))


def test_host_roll_matches_direct_extraction():
    check_roll(None, 0)


def test_host_arithmetic_matches_oracle():
    check_all(None, 0)
